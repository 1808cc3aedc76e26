"""ctypes binding of libluminoth_b200.so (the C ABI in include/luminoth_b200.h).

Thin by design: torch tensors / numpy arrays are only the containers whose
pointers cross the boundary.  There is NO CPU fallback: if the library cannot
be loaded, or no CUDA device is visible, every entry point raises.
"""
import ctypes
import json
import os
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libluminoth_b200.so')

LUMI_OK, LUMI_EINVAL, LUMI_ECUDA, LUMI_ESTATE, LUMI_ENOWEIGHT, LUMI_EOVERFLOW = 0, -1, -2, -3, -4, -5

_lib = None
_lib_lock = threading.Lock()

_c_int_p = ctypes.POINTER(ctypes.c_int)
_c_f_p = ctypes.POINTER(ctypes.c_float)
_c_i64_p = ctypes.POINTER(ctypes.c_int64)
_c_i32_p = ctypes.POINTER(ctypes.c_int32)

# name -> (restype, argtypes); must list every symbol include/luminoth_b200.h declares
SIGNATURES = {
    'lumi_version': (ctypes.c_char_p, []),
    'lumi_device_count': (ctypes.c_int, []),
    'lumi_create': (ctypes.c_int, [ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                   ctypes.POINTER(ctypes.c_void_p)]),
    'lumi_set_weight': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_void_p, _c_i64_p, ctypes.c_int]),
    'lumi_num_weights': (ctypes.c_int, [ctypes.c_void_p]),
    'lumi_weight_info': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_char_p), _c_i64_p,
                                        _c_int_p]),
    'lumi_finalize': (ctypes.c_int, [ctypes.c_void_p]),
    'lumi_predict': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                    ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                    ctypes.c_int]),
    'lumi_predict_f32': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]),
    'lumi_max_detections': (ctypes.c_int, [ctypes.c_void_p]),
    'lumi_set_record_output': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    'lumi_stream': (ctypes.c_void_p, [ctypes.c_void_p]),
    'lumi_synchronize': (ctypes.c_int, [ctypes.c_void_p]),
    'lumi_last_launch_count': (ctypes.c_int, [ctypes.c_void_p]),
    'lumi_set_conv_impl': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    'lumi_set_conv_streamk': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    'lumi_set_debug_taps': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    'lumi_set_pipeline': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    'lumi_set_graphs': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    'lumi_last_graph_replays': (ctypes.c_int, [ctypes.c_void_p]),
    'lumi_profile_enable': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    'lumi_profile_read': (ctypes.c_char_p, [ctypes.c_void_p]),
    'lumi_profile_read_layers': (ctypes.c_char_p, [ctypes.c_void_p]),
    'lumi_get_tensor': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_void_p, ctypes.c_int64, _c_i64_p,
                                       _c_i64_p]),
    'lumi_last_error': (ctypes.c_char_p, [ctypes.c_void_p]),
    'lumi_destroy': (None, [ctypes.c_void_p]),
    'lumi_decode_jpeg': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                        ctypes.c_int, _c_int_p, _c_int_p]),
    'lumi_jpeg_last_error': (ctypes.c_char_p, []),
    'lumi_op_last_error': (ctypes.c_char_p, []),
    'lumi_op_trywait_probe': (ctypes.c_int, [ctypes.c_int] + [ctypes.POINTER(ctypes.c_uint)] * 3),
    'lumi_op_conv2d': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p] + [ctypes.c_int] * 6 +
                       [ctypes.c_void_p] * 3 + [ctypes.c_int] * 2 + [ctypes.c_void_p, _c_int_p, _c_int_p,
                                                                      ctypes.c_void_p]),
    'lumi_op_resize_bilinear': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                               ctypes.c_int, ctypes.c_int, ctypes.c_void_p]),
    'lumi_op_conv2d_preact': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p] +
                              [ctypes.c_int] * 6 + [ctypes.c_void_p] * 3 + [ctypes.c_int] * 2 +
                              [ctypes.c_void_p] * 4 + [_c_int_p, _c_int_p, ctypes.c_void_p]),
    'lumi_op_conv2d_io': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p] +
                          [ctypes.c_int] * 6 + [ctypes.c_void_p] * 3 + [ctypes.c_int] * 5 +
                          [ctypes.c_void_p] * 4 + [_c_int_p, _c_int_p, ctypes.c_void_p]),
    'lumi_pack_conv_weights': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 4),
    'lumi_op_max_pool': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 7 + [ctypes.c_void_p, ctypes.c_void_p]),
    'lumi_op_max_pool_preact': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 7 + [ctypes.c_void_p] * 4),
    'lumi_op_roi_pool': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p, ctypes.c_void_p,
                                                                                ctypes.c_int, ctypes.c_float,
                                                                                ctypes.c_float, ctypes.c_int,
                                                                                ctypes.c_int, ctypes.c_void_p,
                                                                                ctypes.c_void_p]),
    'lumi_roi_kernel': (ctypes.c_int, [ctypes.c_int] * 3),
    'lumi_op_roi_pool_batched': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p] * 2 +
                                 [ctypes.c_int, ctypes.c_float, ctypes.c_float] + [ctypes.c_int] * 3 +
                                 [ctypes.c_void_p] * 3),
    'lumi_op_spatial_mean': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p] * 2),
    'lumi_op_softmax_rows': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 2),
    'lumi_op_sort_desc': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    'lumi_op_nms_sorted': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_void_p]),
    'lumi_nms_path': (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.c_float]),
    'lumi_op_nms_batched': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                           ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    'lumi_op_rpn_proposals_batched': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64,
                                                     ctypes.c_int, ctypes.c_void_p] + [ctypes.c_int] * 3 +
                                      [ctypes.c_float] * 2 + [ctypes.c_int] * 2 + [ctypes.c_float] * 2 +
                                      [ctypes.c_int] * 8 + [ctypes.c_void_p] * 4),
    'lumi_op_class_detections_batched': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int64] + [ctypes.c_void_p] * 3 +
                                         [ctypes.c_int] * 3 + [ctypes.c_float] * 6 + [ctypes.c_int] * 5 +
                                         [ctypes.c_void_p] * 6),
    'lumi_op_rpn_proposals': (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_float, ctypes.c_float,
                                                                     ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                                                     ctypes.c_float, ctypes.c_int, ctypes.c_int] +
                              [ctypes.c_void_p] * 4),
    'lumi_op_class_detections': (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_int] +
                                 [ctypes.c_float] * 6 + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 5),
}


def load_library():
    """Load (once) and type the C ABI.  Raises RuntimeError when the library is
    missing -- it is never silently replaced by a CPU path."""
    global _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                'luminoth_b200: %s is not built (run `python -c "import __graft_entry__ as g; g.build()"`); '
                'there is no CPU fallback' % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)          # AttributeError if the symbol is missing
            fn.restype = res
            fn.argtypes = args
        _lib = lib
        return lib


def decode_jpeg(data, device=0):
    """JPEG bytes -> (H, W, 3) uint8 RGB numpy array, decoded on the GPU by nvJPEG (``lumi_decode_jpeg``).
    RuntimeError when nvJPEG / a CUDA device is unavailable or the stream is not a decodable JPEG."""
    lib = load_library()
    buf = (ctypes.c_ubyte * len(data)).from_buffer_copy(data)
    h, w = ctypes.c_int(), ctypes.c_int()
    rc = lib.lumi_decode_jpeg(buf, len(data), int(device), None, 0, 0, ctypes.byref(h), ctypes.byref(w))
    if rc != LUMI_OK:
        raise RuntimeError('lumi_decode_jpeg: ' + lib.lumi_jpeg_last_error().decode())
    out = np.empty((h.value, w.value, 3), np.uint8)
    rc = lib.lumi_decode_jpeg(buf, len(data), int(device), out.ctypes.data_as(ctypes.c_void_p), out.nbytes, 0,
                              ctypes.byref(h), ctypes.byref(w))
    if rc != LUMI_OK:
        raise RuntimeError('lumi_decode_jpeg: ' + lib.lumi_jpeg_last_error().decode())
    return out


def _raise(code, msg):
    msg = msg.decode() if isinstance(msg, bytes) else str(msg)
    if code in (LUMI_EINVAL, LUMI_ENOWEIGHT):
        raise ValueError(msg)
    raise RuntimeError('luminoth_b200 (code %d): %s' % (code, msg))


def _to_plain(config):
    if isinstance(config, dict):
        return {k: _to_plain(v) for k, v in config.items()}
    if isinstance(config, (list, tuple)):
        return [_to_plain(v) for v in config]
    if isinstance(config, np.generic):
        return config.item()
    return config


class Engine(object):
    """One engine handle = one GPU, one stream, one workspace.  Not re-entrant:
    calls are serialised by a lock (the reference has a single tf.Session)."""

    def __init__(self, config, device=0, max_batch=1, max_h=None, max_w=None):
        self._lib = load_library()
        self._h = ctypes.c_void_p()
        self._lock = threading.Lock()
        mtype = config['model']['type']
        if max_h is None or max_w is None:
            ip = config['dataset']['image_preprocessing']
            if mtype == 'ssd':
                max_h, max_w = ip['fixed_height'], ip['fixed_width']
            else:
                side = max(int(ip.get('max_size') or 1024), int(ip.get('min_size') or 600))
                max_h = max_w = side
        cfg_json = json.dumps(_to_plain(config)).encode()
        rc = self._lib.lumi_create(cfg_json, int(device), int(max_batch), int(max_h), int(max_w),
                                   ctypes.byref(self._h))
        if rc != LUMI_OK:
            _raise(rc, self._lib.lumi_last_error(None))
        self.device = int(device)
        self.max_batch = int(max_batch)
        self.max_detections = self._lib.lumi_max_detections(self._h)
        self._finalized = False

    # ---- weights
    def weight_specs(self):
        out = []
        name = ctypes.c_char_p()
        shape = (ctypes.c_int64 * 4)()
        ndim = ctypes.c_int()
        for i in range(self._lib.lumi_num_weights(self._h)):
            self._lib.lumi_weight_info(self._h, i, ctypes.byref(name), shape, ctypes.byref(ndim))
            out.append((name.value.decode(), tuple(int(shape[j]) for j in range(ndim.value))))
        return out

    def set_weight(self, name, array):
        a = np.ascontiguousarray(array, dtype=np.float32)
        shape = (ctypes.c_int64 * a.ndim)(*a.shape)
        rc = self._lib.lumi_set_weight(self._h, name.encode(), a.ctypes.data_as(ctypes.c_void_p), shape, a.ndim)
        if rc != LUMI_OK:
            _raise(rc, self._lib.lumi_last_error(self._h))

    def load_weights(self, weights):
        for name, shape in self.weight_specs():
            if name not in weights:
                raise ValueError("variable '%s' missing from the weight dict" % name)
            self.set_weight(name, weights[name])
        return self

    def finalize(self):
        rc = self._lib.lumi_finalize(self._h)
        if rc != LUMI_OK:
            _raise(rc, self._lib.lumi_last_error(self._h))
        self._finalized = True
        return self

    def set_conv_impl(self, impl):
        rc = self._lib.lumi_set_conv_impl(self._h, {'simt': 0, 'tc': 1}.get(impl, impl))
        if rc != LUMI_OK:
            raise ValueError('conv impl must be "simt" or "tc"')

    def set_conv_streamk(self, mode):
        """Tensor-core conv scheduling: 'off' (whole tiles), 'auto' (default), 'always' (stream-K wherever applicable)."""
        rc = self._lib.lumi_set_conv_streamk(self._h, {'off': 0, 'auto': 1, 'always': 2}.get(mode, mode))
        if rc != LUMI_OK:
            raise ValueError('stream-K mode must be "off", "auto" or "always"')

    # ---- forward
    def predict_raw(self, images):
        """images: [n,h,w,3] uint8 (``lumi_predict``) or float32 (``lumi_predict_f32``: resized images keep their
        non-integer pixel values, like the reference's feed); numpy array -> host path, H2D inside the call;
        CUDA torch tensor -> device path.  Returns numpy
        (boxes [n,K,4], scores [n,K], labels [n,K], counts [n])."""
        on_dev = False
        if isinstance(images, np.ndarray):
            is_f32 = images.dtype != np.uint8
            imgs = np.ascontiguousarray(images, dtype=np.float32 if is_f32 else np.uint8)
            n, h, w, c = imgs.shape
            ptr = imgs.ctypes.data
        else:                       # torch tensor
            import torch
            assert images.dtype in (torch.uint8, torch.float32) and images.is_contiguous()
            is_f32 = images.dtype == torch.float32
            n, h, w, c = images.shape
            on_dev = images.is_cuda
            ptr = images.data_ptr()
        if c != 3:
            raise ValueError('images must be [n,h,w,3] RGB')
        k = self.max_detections
        boxes = np.empty((n, k, 4), np.float32)
        scores = np.empty((n, k), np.float32)
        labels = np.empty((n, k), np.int32)
        counts = np.empty((n,), np.int32)
        fn = self._lib.lumi_predict_f32 if is_f32 else self._lib.lumi_predict
        with self._lock:
            rc = fn(self._h, ctypes.c_void_p(ptr), int(on_dev), n, h, w,
                    boxes.ctypes.data_as(ctypes.c_void_p), scores.ctypes.data_as(ctypes.c_void_p),
                    labels.ctypes.data_as(ctypes.c_void_p), counts.ctypes.data_as(ctypes.c_void_p), 0)
            if rc != LUMI_OK:
                _raise(rc, self._lib.lumi_last_error(self._h))
        return boxes, scores, labels, counts

    def predict_device(self, images, boxes, scores, labels, counts):
        """Fully asynchronous device-resident call (CUDA torch tensors in and out)."""
        n, h, w, _ = images.shape
        with self._lock:
            rc = self._lib.lumi_predict(self._h, ctypes.c_void_p(images.data_ptr()), 1, n, h, w,
                                        ctypes.c_void_p(boxes.data_ptr()), ctypes.c_void_p(scores.data_ptr()),
                                        ctypes.c_void_p(labels.data_ptr()), ctypes.c_void_p(counts.data_ptr()), 1)
            if rc != LUMI_OK:
                _raise(rc, self._lib.lumi_last_error(self._h))

    def set_record_output(self, records):
        """CUDA float32 tensor [max_batch, 1 + 6*K] (or None): every following predict also writes one packed
        {count, boxes, scores, labels} row per image there -- the send buffer of the detection all-gather."""
        if records is not None:
            assert records.is_cuda and records.is_contiguous() and records.numel() >= self.max_batch * (1 + 6 * self.max_detections)
        self._records = records          # keep the buffer alive
        self._lib.lumi_set_record_output(self._h, ctypes.c_void_p(records.data_ptr() if records is not None else 0))

    def set_pipeline(self, enable=True):
        self._lib.lumi_set_pipeline(self._h, int(bool(enable)))

    def set_graphs(self, enable=True):
        """CUDA-graph replay of the forward (default on): bit-identical results, one launch per (half-)batch."""
        self._lib.lumi_set_graphs(self._h, int(bool(enable)))

    @property
    def last_graph_replays(self):
        return self._lib.lumi_last_graph_replays(self._h)

    def set_debug_taps(self, enable=True):
        self._lib.lumi_set_debug_taps(self._h, int(bool(enable)))

    def profile(self, enable=True):
        self._lib.lumi_profile_enable(self._h, int(bool(enable)))

    def profile_read(self):
        """{category: (spans, total_ms, work)} accumulated since the last read
        (work = algorithmic FLOPs for conv_*, algorithmic bytes for roi_pool)."""
        txt = self._lib.lumi_profile_read(self._h).decode()
        out = {}
        for part in txt.split(';'):
            if part:
                name, cnt, ms, work = part.split(':')
                out[name] = (int(cnt), float(ms), float(work))
        return out

    def profile_read_layers(self):
        """[(conv layer, spans, total_ms, flops)] of the spans drained by the last profile_read()."""
        txt = self._lib.lumi_profile_read_layers(self._h).decode()
        out = []
        for part in txt.split(';'):
            if part:
                name, cnt, ms, work = part.rsplit(':', 3)
                out.append((name, int(cnt), float(ms), float(work)))
        return out

    def synchronize(self):
        rc = self._lib.lumi_synchronize(self._h)
        if rc != LUMI_OK:
            _raise(rc, self._lib.lumi_last_error(self._h))

    @property
    def stream(self):
        return self._lib.lumi_stream(self._h)

    @property
    def last_launch_count(self):
        return self._lib.lumi_last_launch_count(self._h)

    def get_tensor(self, name):
        numel = ctypes.c_int64()
        shape = (ctypes.c_int64 * 4)()
        with self._lock:
            rc = self._lib.lumi_get_tensor(self._h, name.encode(), None, 0, ctypes.byref(numel), shape)
            if rc != LUMI_OK:
                _raise(rc, self._lib.lumi_last_error(self._h))
            out = np.empty((numel.value,), np.float32)
            rc = self._lib.lumi_get_tensor(self._h, name.encode(), out.ctypes.data_as(ctypes.c_void_p), numel.value,
                                           ctypes.byref(numel), shape)
            if rc != LUMI_OK:
                _raise(rc, self._lib.lumi_last_error(self._h))
        shp = [int(s) for s in shape]
        while len(shp) > 1 and shp[-1] == 1:
            shp.pop()
        return out.reshape(shp)

    def close(self):
        if getattr(self, '_h', None) is not None and self._h:
            self._lib.lumi_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
