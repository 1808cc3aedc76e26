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
    'lumi_set_pixel_format': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    'lumi_predict': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                    ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p,
                                    ctypes.c_int]),
    'lumi_predict_f32': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]),
    'lumi_predict_resize': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 5 +
                            [ctypes.c_void_p] * 4 + [ctypes.c_int]),
    'lumi_predict_sizes': (ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 4 +
                           [ctypes.c_int]),
    'lumi_predict_windows': (ctypes.c_int, [ctypes.c_void_p] * 3 + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 2 +
                             [ctypes.c_int, ctypes.c_float] + [ctypes.c_void_p] * 4 + [ctypes.c_int]),
    'lumi_last_window_detections': (ctypes.c_int, [ctypes.c_void_p] * 5 + [_c_i64_p]),
    'lumi_max_detections': (ctypes.c_int, [ctypes.c_void_p]),
    'lumi_set_record_output': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    'lumi_stream': (ctypes.c_void_p, [ctypes.c_void_p]),
    'lumi_synchronize': (ctypes.c_int, [ctypes.c_void_p]),
    'lumi_last_launch_count': (ctypes.c_int, [ctypes.c_void_p]),
    'lumi_set_conv_impl': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    'lumi_set_conv_streamk': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
    'lumi_set_sm_limit': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int]),
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
    'lumi_op_pixels_to_rgb': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p] * 2),
    'lumi_op_conv2d_preact': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p] +
                              [ctypes.c_int] * 6 + [ctypes.c_void_p] * 3 + [ctypes.c_int] * 2 +
                              [ctypes.c_void_p] * 4 + [_c_int_p, _c_int_p, ctypes.c_void_p]),
    'lumi_op_conv2d_io': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p] +
                          [ctypes.c_int] * 6 + [ctypes.c_void_p] * 3 + [ctypes.c_int] * 5 +
                          [ctypes.c_void_p] * 4 + [_c_int_p, _c_int_p, ctypes.c_void_p]),
    'lumi_op_conv2d_sched': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p] +
                             [ctypes.c_int] * 6 + [ctypes.c_void_p] * 3 + [ctypes.c_int] * 5 +
                             [ctypes.c_void_p] * 2 + [ctypes.c_int] * 2 + [ctypes.c_void_p] * 2 +
                             [_c_int_p, _c_int_p, ctypes.c_void_p]),
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
    'lumi_op_l2norm_scale': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p, ctypes.c_float] +
                             [ctypes.c_void_p] * 2),
    'lumi_op_softmax_rows': (ctypes.c_int, [ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 2),
    'lumi_op_sort_desc': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]),
    'lumi_op_nms_sorted': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_void_p,
                                          ctypes.c_void_p, ctypes.c_void_p]),
    'lumi_nms_path': (ctypes.c_int, [ctypes.c_int, ctypes.c_int, ctypes.c_float]),
    'lumi_op_nms_batched': (ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_float,
                                           ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]),
    'lumi_op_window_merge': (ctypes.c_int, [ctypes.c_void_p] * 4 + [ctypes.c_int] * 2 + [ctypes.c_void_p] * 2 +
                             [ctypes.c_int] * 4 + [ctypes.c_float, ctypes.c_int] + [ctypes.c_void_p] * 4 +
                             [_c_i64_p, ctypes.c_void_p]),
    'lumi_op_rpn_proposals_batched':(ctypes.c_int, [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64,
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


# LUMI_PIXELS_* of include/luminoth_b200.h
PIXEL_FORMATS = {'rgb': 0, 'bgr': 1, 'nv12': 2, 'i420': 3}


def pixel_format_code(pixel_format):
    """The LUMI_PIXELS_* code of 'rgb', 'bgr', 'nv12' or 'i420'; ValueError for any other name."""
    try:
        return PIXEL_FORMATS[pixel_format]
    except (KeyError, TypeError):
        raise ValueError("pixel_format must be one of 'rgb', 'bgr', 'nv12', 'i420', got %r" % (pixel_format,))


def pixel_size(shape, pixel_format='rgb', uint8=True):
    """The (h, w) pixel size of one image array of ``shape`` in ``pixel_format``: RGB and BGR images are (h, w, 3);
    NV12 and I420 images are the 2-D (3h/2, w) uint8 arrays OpenCV and video decoders give (Y plane, then chroma),
    with h and w even.  ValueError for any other shape, and for an NV12 or I420 image that is not uint8."""
    code = pixel_format_code(pixel_format)
    shape = tuple(int(d) for d in shape)
    name = pixel_format.upper()
    if code < 2:
        if len(shape) != 3 or shape[2] != 3:
            raise ValueError('images must be (h, w, 3) %s, got shape %s' % (name, shape))
        return shape[0], shape[1]
    if not uint8:
        raise ValueError('%s images must be uint8' % name)
    if len(shape) != 2 or shape[0] % 3 or shape[1] % 2:
        raise ValueError('%s images must be (3h/2, w) uint8 arrays with an even height h and width w, got shape %s'
                         % (name, shape))
    return shape[0] * 2 // 3, shape[1]


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
        self._last_nwin = 0
        self._pixel_format = PIXEL_FORMATS['rgb']

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

    def set_sm_limit(self, sms):
        """SMs the launch decisions count on (persistent conv grids, stream-K, the wide-tile rule, the NMS grid):
        0 (default) the device's count; larger values are capped at it.  Runs what a GPU with fewer SMs would."""
        rc = self._lib.lumi_set_sm_limit(self._h, int(sms))
        if rc != LUMI_OK:
            _raise(rc, self._lib.lumi_last_error(self._h))

    def _use_pixel_format(self, code):
        """Sets the engine's pixel format to ``code`` when it differs (the caller holds the lock)."""
        if code != self._pixel_format:
            rc = self._lib.lumi_set_pixel_format(self._h, code)
            if rc != LUMI_OK:
                _raise(rc, self._lib.lumi_last_error(self._h))
            self._pixel_format = code

    # ---- forward
    def predict_raw(self, images, pixel_format='rgb'):
        """images: [n,h,w,3] uint8 (``lumi_predict``) or float32 (``lumi_predict_f32``: resized images keep their
        non-integer pixel values, like the reference's feed); numpy array -> host path, H2D inside the call;
        CUDA torch tensor -> device path.  ``pixel_format`` 'bgr' reads [n,h,w,3] BGR images, 'nv12' and 'i420'
        [n,3h/2,w] uint8 frames (``pixel_size``); the results equal those of their RGB conversions.  Returns numpy
        (boxes [n,K,4], scores [n,K], labels [n,K], counts [n])."""
        code = pixel_format_code(pixel_format)
        on_dev = False
        if isinstance(images, np.ndarray):
            is_f32 = images.dtype != np.uint8
        else:                       # torch tensor
            import torch
            assert images.dtype in (torch.uint8, torch.float32) and images.is_contiguous()
            is_f32 = images.dtype == torch.float32
            on_dev = images.is_cuda
        shape = tuple(images.shape)
        if code == 0:
            n, h, w, c = shape
            if c != 3:
                raise ValueError('images must be [n,h,w,3] RGB')
        else:                       # refuses float32 and odd-sized YUV before any conversion
            n = shape[0]
            h, w = pixel_size(shape[1:], pixel_format, not is_f32)
        if isinstance(images, np.ndarray):
            imgs = np.ascontiguousarray(images, dtype=np.float32 if is_f32 else np.uint8)
            ptr = imgs.ctypes.data
        else:
            ptr = images.data_ptr()
        k = self.max_detections
        boxes = np.empty((n, k, 4), np.float32)
        scores = np.empty((n, k), np.float32)
        labels = np.empty((n, k), np.int32)
        counts = np.empty((n,), np.int32)
        fn = self._lib.lumi_predict_f32 if is_f32 else self._lib.lumi_predict
        with self._lock:
            self._use_pixel_format(code)
            rc = fn(self._h, ctypes.c_void_p(ptr), int(on_dev), n, h, w,
                    boxes.ctypes.data_as(ctypes.c_void_p), scores.ctypes.data_as(ctypes.c_void_p),
                    labels.ctypes.data_as(ctypes.c_void_p), counts.ctypes.data_as(ctypes.c_void_p), 0)
            if rc != LUMI_OK:
                _raise(rc, self._lib.lumi_last_error(self._h))
        return boxes, scores, labels, counts

    def predict_resize(self, images, h, w, pixel_format='rgb'):
        """Like ``predict_raw`` for a list of (h0, w0, 3) images of any sizes, resized to h x w inside the forward
        (``lumi_predict_resize``): bit-identical to ``lumi_op_resize_bilinear`` per image followed by ``predict_raw``
        on the float32 batch.  The images are all numpy arrays (host path) or all CUDA torch tensors (device path),
        and all uint8 or all float32 (numpy arrays of other dtypes are read as float32).  CUDA tensors must be on the
        engine's device and may be non-contiguous (they are copied); the engine reads them after the work queued so far
        on torch's current stream of that device, which is what wrote them.  ``pixel_format`` as in ``predict_raw``:
        'bgr' images are (h0, w0, 3), 'nv12' and 'i420' images (3 h0 / 2, w0) uint8.  Returns numpy (boxes [n,K,4] in
        h x w pixels, scores [n,K], labels [n,K], counts [n])."""
        return self._predict_sources('predict_resize', images, None, int(h), int(w), pixel_format=pixel_format)

    def predict_sizes(self, images, targets, pixel_format='rgb'):
        """``predict_resize`` with one target size per image (``lumi_predict_sizes``): images[i] is resized to
        targets[i] = (h_i, w_i), every image runs in one forward at the top left of a canvas of the largest target
        height and width, and its results equal those of ``predict_resize([images[i]], h_i, w_i)``.  Same argument
        rules as ``predict_resize``; boxes come back in each image's own target pixels.  Faster R-CNN only (SSD takes
        only its fixed size)."""
        targets = np.array(targets, np.int32).reshape(-1, 2) if len(targets) else np.zeros((0, 2), np.int32)
        return self._predict_sources('predict_sizes', images, targets, 0, 0, pixel_format=pixel_format)

    def predict_windows(self, images, windows, scales, iou_threshold, pixel_format='rgb'):
        """Sliced prediction (``lumi_predict_windows``): windows[k] = (src, y0, x0, h, w, th, tw) is the h x w region
        of images[src] at (y0, x0), resized to th x tw and predicted like ``predict_resize``; scales[k] = (s_y, s_x) is
        its scale factor.  The windows' detections are mapped to source pixels and merged per source image on the GPU
        (per-label greedy NMS at ``iou_threshold``, then the top ``max_detections`` by score).  Same image rules as
        ``predict_resize``, ``pixel_format`` included (windows are in pixels, and may start at odd rows and columns of
        NV12 and I420 sources).  Returns numpy (boxes [n,K,4] in source pixels, scores [n,K], labels [n,K], counts [n])
        for the n source images."""
        windows = np.ascontiguousarray(np.asarray(windows, np.int32).reshape(-1, 7))
        scales = np.ascontiguousarray(np.asarray(scales, np.float32).reshape(-1, 2))
        if len(scales) != len(windows):
            raise ValueError('predict_windows: %d windows but %d scale pairs' % (len(windows), len(scales)))
        return self._predict_sources('predict_windows', images, None, 0, 0,
                                     windows=(windows, scales, float(iou_threshold)), pixel_format=pixel_format)

    def last_window_detections(self):
        """The per-window detections of the last ``predict_windows`` call, in window pixels (boxes [nwin,K,4], scores
        [nwin,K], labels [nwin,K], counts [nwin]), and its merge statistics {'workspace_bytes', 'candidates',
        'longest_list', 'groups'}."""
        stats = (ctypes.c_int64 * 4)()
        nwin = self._last_nwin
        k = self.max_detections
        boxes = np.empty((nwin, k, 4), np.float32)
        scores = np.empty((nwin, k), np.float32)
        labels = np.empty((nwin, k), np.int32)
        counts = np.empty((nwin,), np.int32)
        with self._lock:
            rc = self._lib.lumi_last_window_detections(self._h, *[a.ctypes.data_as(ctypes.c_void_p)
                                                                  for a in (boxes, scores, labels, counts)], stats)
            if rc != LUMI_OK:
                _raise(rc, self._lib.lumi_last_error(self._h))
        names = ('workspace_bytes', 'candidates', 'longest_list', 'groups')
        return boxes, scores, labels, counts, dict(zip(names, (int(v) for v in stats)))

    def _predict_sources(self, name, images, targets, h, w, windows=None, pixel_format='rgb'):
        code = pixel_format_code(pixel_format)
        images = list(images)
        n = len(images)
        if n == 0:
            raise ValueError('%s: no images' % name)
        if targets is not None and len(targets) != n:
            raise ValueError('%s: %d images but %d targets' % (name, n, len(targets)))
        on_dev = [not isinstance(im, np.ndarray) for im in images]
        if any(on_dev) != all(on_dev):
            raise ValueError('%s: the images must be all numpy arrays or all CUDA tensors' % name)
        if on_dev[0]:
            import torch
            for im in images:
                if not im.is_cuda or im.dtype not in (torch.uint8, torch.float32):
                    raise ValueError('%s: device images must be CUDA uint8 or float32 tensors' % name)
                if im.device.index != self.device:
                    raise ValueError('%s: image on %s, the engine runs on cuda:%d' % (name, im.device, self.device))
            f32 = [im.dtype == torch.float32 for im in images]
            srcs = [im.contiguous() for im in images]
            ptrs = [s.data_ptr() for s in srcs]
        else:
            f32 = [im.dtype != np.uint8 for im in images]
            srcs = [np.ascontiguousarray(im, dtype=np.float32 if f else np.uint8) for im, f in zip(images, f32)]
            ptrs = [s.ctypes.data for s in srcs]
        if any(f32) != all(f32):
            raise ValueError('%s: the images of one call must share a dtype (uint8 or float32)' % name)
        if code == 0:
            for s in srcs:
                if len(s.shape) != 3 or s.shape[2] != 3:
                    raise ValueError('%s: images must be (h0, w0, 3) RGB' % name)
            sizes = np.array([s.shape[:2] for s in srcs], np.int32)
        else:
            try:
                sizes = np.array([pixel_size(s.shape, pixel_format, not f) for s, f in zip(srcs, f32)], np.int32)
            except ValueError as ex:
                raise ValueError('%s: %s' % (name, ex))
        ptr_arr = (ctypes.c_void_p * n)(*ptrs)
        k = self.max_detections
        boxes = np.empty((n, k, 4), np.float32)
        scores = np.empty((n, k), np.float32)
        labels = np.empty((n, k), np.int32)
        counts = np.empty((n,), np.int32)
        outs = [a.ctypes.data_as(ctypes.c_void_p) for a in (boxes, scores, labels, counts)]
        with self._lock:
            self._use_pixel_format(code)
            if on_dev[0]:
                # the engine's streams do not follow torch's: make its stream wait for the work torch has queued on
                # the device's current stream (the caller's writes of the images, the copies of .contiguous()); the
                # call returns synchronised, so srcs outlive the engine's reads
                dev = torch.device('cuda', self.device)
                ready = torch.cuda.Event()
                ready.record(torch.cuda.current_stream(dev))
                torch.cuda.ExternalStream(self.stream, device=dev).wait_event(ready)
            sz = sizes.ctypes.data_as(ctypes.c_void_p)
            if windows is not None:
                wins, scl, thr = windows
                rc = self._lib.lumi_predict_windows(self._h, ptr_arr, sz, int(f32[0]), int(on_dev[0]), n,
                                                    wins.ctypes.data_as(ctypes.c_void_p),
                                                    scl.ctypes.data_as(ctypes.c_void_p), len(wins), thr, *outs, 0)
                if rc == LUMI_OK:
                    self._last_nwin = len(wins)
            elif targets is None:
                rc = self._lib.lumi_predict_resize(self._h, ptr_arr, sz, int(f32[0]), int(on_dev[0]), n, h, w, *outs, 0)
            else:
                rc = self._lib.lumi_predict_sizes(self._h, ptr_arr, sz, targets.ctypes.data_as(ctypes.c_void_p),
                                                  int(f32[0]), int(on_dev[0]), n, *outs, 0)
            if rc != LUMI_OK:
                _raise(rc, self._lib.lumi_last_error(self._h))
        return boxes, scores, labels, counts

    def predict_device(self, images, boxes, scores, labels, counts):
        """Fully asynchronous device-resident call (CUDA torch tensors in and out)."""
        n, h, w, _ = images.shape
        with self._lock:
            self._use_pixel_format(PIXEL_FORMATS['rgb'])
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
