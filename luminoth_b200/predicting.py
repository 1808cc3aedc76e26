"""``PredictorNetwork`` -- drop-in for ``luminoth/utils/predicting.py:10-148``.

Same constructor and ``predict_image(image) -> [{'bbox', 'label', 'prob'}]``
(sorted by probability, integer pixel boxes in the ORIGINAL image, probs
rounded to 4 decimals).  ``predict_batch(images)`` is the batched extension
(the reference is hard-wired to batch 1, ``fasterrcnn.py:101-103``).

What changed underneath: graph build + ``session.run`` is one call into the
sm_90a engine (``lumi_predict`` / ``lumi_predict_f32``).  The aspect-preserving
resize of ``datasets/object_detection_dataset.py:71-83`` / ``utils/image.py:38-147``
runs on the GPU (``lumi_op_resize_bilinear``, bit-identical to the TF1 legacy
bilinear kernel); only its size arithmetic (float32, like the reference) stays on
the host.  Images of different sizes in one ``predict_batch`` call are bucketed by
their preprocessed size, each bucket runs as one batched engine call, and the
results come back in the caller's order.
"""
import json
import math
import os
import warnings

import numpy as np

from .config import get_model_type
from .engine import Engine


def _resize_bilinear_legacy(image, new_h, new_w):
    """tf.image.resize_images(BILINEAR), TF1 legacy kernel (align_corners=False,
    src = dst * in/out, no half-pixel offset) -- ``utils/image.py:94-97``."""
    image = np.asarray(image, np.float32)
    H, W = image.shape[:2]
    if (H, W) == (new_h, new_w):
        return image
    hs = np.float32(H) / np.float32(new_h)
    ws = np.float32(W) / np.float32(new_w)
    ys = np.arange(new_h, dtype=np.float32) * hs
    xs = np.arange(new_w, dtype=np.float32) * ws
    y0 = np.floor(ys).astype(np.int64); x0 = np.floor(xs).astype(np.int64)
    y1 = np.minimum(y0 + 1, H - 1); x1 = np.minimum(x0 + 1, W - 1)
    yl = (ys - y0.astype(np.float32))[:, None, None]
    xl = (xs - x0.astype(np.float32))[None, :, None]
    top = image[y0][:, x0] + (image[y0][:, x1] - image[y0][:, x0]) * xl
    bot = image[y1][:, x0] + (image[y1][:, x1] - image[y1][:, x0]) * xl
    return (top + (bot - top) * yl).astype(np.float32)


def target_size(shape, config):
    """(new_h, new_w, scale_factor) of the inference preprocessing for an image of ``shape`` --
    ``utils/image.py:38-114`` (aspect-preserving, float32 arithmetic, ``tf.to_int32`` truncation) and
    ``:117-147`` (fixed size; scale_factor is then the tuple (s_h, s_w))."""
    ip = config['dataset']['image_preprocessing']
    f32 = np.float32
    h, w = f32(shape[0]), f32(shape[1])
    if ip.get('fixed_height') and ip.get('fixed_width'):
        nh, nw = int(ip['fixed_height']), int(ip['fixed_width'])
        return nh, nw, (f32(nh) / h, f32(nw) / w)
    mn, mx = ip.get('min_size'), ip.get('max_size')
    up = max(f32(mn) / min(h, w), f32(1.)) if mn is not None else f32(1.)
    down = min(f32(mx) / max(h, w), f32(1.)) if mx is not None else f32(1.)
    scale = f32(up * down)
    return int(math.trunc(float(h * scale))), int(math.trunc(float(w * scale))), scale


def preprocess_image(image, config):
    """Inference preprocessing on the host (numpy); returns (float32 image, scale_factor).  The product path
    resizes on the GPU (``PredictorNetwork._resize_on_device``); this restatement is its cross-check."""
    image = np.asarray(image)
    if image.ndim != 3 or image.shape[2] != 3:
        raise ValueError('expected an (H, W, 3) RGB image')
    nh, nw, scale = target_size(image.shape, config)
    return _resize_bilinear_legacy(image, nh, nw), scale


def format_predictions(objects, labels, probs, scale_factor, class_labels=None):
    """``predicting.py:114-148``: rescale, int(round()), round(prob, 4), sort desc."""
    objects = np.array(objects, np.float32, copy=True)
    labels = np.asarray(labels).tolist()
    probs = np.asarray(probs, np.float32).tolist()
    if class_labels is not None:
        labels = [class_labels[label] for label in labels]
    if isinstance(scale_factor, tuple):
        objects /= np.array([scale_factor[1], scale_factor[0], scale_factor[1], scale_factor[0]], np.float32)
    else:
        objects /= np.float32(scale_factor)
    objects = [[int(round(coord)) for coord in obj] for obj in objects.tolist()]
    return sorted([{'bbox': obj, 'label': label, 'prob': round(prob, 4)}
                   for obj, label, prob in zip(objects, labels, probs)],
                  key=lambda x: x['prob'], reverse=True)


def load_checkpoint_weights(engine, job_dir, prefix=None):
    """The ``Saver.restore`` of ``predicting.py:51-63`` without TensorFlow: reads the latest Saver-V2 bundle under
    ``job_dir`` and returns {tf variable name: array} for exactly the variables the engine's plan uses (optimizer
    slots, ``global_step`` and never-executed layers such as ResNet-50's block4 are ignored, like a Saver built from
    the inference graph would).  Raises ``ValueError`` when the directory holds no checkpoint, a variable is
    missing or a shape differs."""
    from . import tf_checkpoint as tfc
    if prefix is None:
        prefix = tfc.latest_checkpoint(job_dir)            # ValueError('Could not find checkpoint in ...')
    reader = tfc.BundleReader(prefix)
    weights, missing = {}, []
    for name, shape in engine.weight_specs():
        if not reader.has_tensor(name):
            missing.append(name)
            continue
        if tuple(reader.shape(name)) != tuple(shape):
            raise ValueError("checkpoint variable '%s' has shape %s, the model expects %s"
                             % (name, tuple(reader.shape(name)), tuple(shape)))
        weights[name] = reader.get_tensor(name, verify=True).astype(np.float32, copy=False)   # per-tensor crc32c checked
    if missing:
        raise ValueError('checkpoint %s lacks %d model variables, e.g. %s' % (prefix, len(missing), missing[:3]))
    return weights


class PredictorNetwork(object):
    """Instantiates a network in order to get predictions from it.

    ``weights``: optional dict {tf variable name: array} (TF layouts).  Without
    it, and without a checkpoint, the model is randomly initialised with a
    warning -- exactly the reference's "prediction without checkpoint is just
    used for testing" branch (``predicting.py:64-72``).
    """

    def __init__(self, config, weights=None, device=0, max_batch=1):
        self.class_labels = None
        if config.dataset.dir:
            classes_file = os.path.join(config.dataset.dir, 'classes.json')
            if os.path.exists(classes_file):
                with open(classes_file) as f:
                    self.class_labels = json.load(f)
        config.dataset.data_augmentation = None
        get_model_type(config.model.type)                 # ValueError on unknown model types
        self.config = config
        self.engine = Engine(config, device=device, max_batch=max_batch)
        if callable(weights):                             # e.g. lumi eval: one specific checkpoint of the run
            weights = weights(self.engine)
        if weights is None:
            if config.train.job_dir:
                job_dir = config.train.job_dir
                if config.train.run_name:
                    job_dir = os.path.join(job_dir, config.train.run_name)
                # predicting.py:51-63: latest checkpoint of <job_dir>/<run_name>, restored by variable name
                weights = load_checkpoint_weights(self.engine, job_dir)
            else:
                warnings.warn('Could not load checkpoint. Using initialized model.')
                from .synth import make_weights
                weights = make_weights(config, seed=config.train.seed or 0, profile='reference')
        self.engine.load_weights(weights).finalize()

    # -- reference API
    def predict_image(self, image):
        return self.predict_batch([image])[0]

    # -- batched extension
    def predict_batch(self, images):
        """Predictions for a list of (H, W, 3) images of ANY mix of sizes, in the caller's order.  Images are grouped
        by the size the preprocessing gives them (``target_size``); each group runs through the engine in chunks of
        ``max_batch`` -- a directory of equally sized frames (``predict.py:69-97``, video frames ``:100-171``) is
        one batched call per chunk instead of one call per image."""
        return [format_predictions(boxes, labels, probs, scale, self.class_labels)
                for boxes, labels, probs, scale in self.predict_batch_raw(images)]

    def predict_batch_raw(self, images):
        """The network's fetches per image, before the Python post-step of ``predicting.py:114-148``:
        [(objects (K,4) float32 in PREPROCESSED-image pixels, labels (K,) int32, probs (K,) float32, scale_factor)]
        in the caller's order (``lumi eval`` compares these with the scaled ground truth, ``eval.py:330-347``)."""
        images = [np.asarray(im) for im in images]
        if not images:
            return []
        for im in images:
            if im.ndim != 3 or im.shape[2] != 3:
                raise ValueError('expected an (H, W, 3) RGB image')
        sizes = [target_size(im.shape, self.config) for im in images]
        buckets = {}                                     # (nh, nw) -> indices, first-seen order
        for i, (nh, nw, _) in enumerate(sizes):
            buckets.setdefault((nh, nw), []).append(i)
        out = [None] * len(images)
        for (nh, nw), idxs in buckets.items():
            untouched = all(images[i].dtype == np.uint8 and images[i].shape[:2] == (nh, nw) for i in idxs)
            for s in range(0, len(idxs), self.engine.max_batch):
                chunk = idxs[s:s + self.engine.max_batch]
                if untouched:   # integer pixels, no resize: the uint8 entry point (the benchmark shapes)
                    batch = np.stack([images[i] for i in chunk])
                else:           # the reference feeds the resized FLOAT image (predicting.py:110-112)
                    batch = self._resize_on_device([images[i] for i in chunk], nh, nw)
                boxes, scores, labels, counts = self.engine.predict_raw(batch)
                for j, i in enumerate(chunk):
                    k = int(counts[j])
                    out[i] = (boxes[j, :k].copy(), labels[j, :k].copy(), scores[j, :k].copy(), sizes[i][2])
        return out

    def _resize_on_device(self, images, nh, nw):
        """``resize_image`` / ``resize_image_fixed`` (utils/image.py:38-147) on the GPU: legacy TF bilinear kernel,
        bit-identical to the float32 host restatement; returns a CUDA float32 tensor [n, nh, nw, 3]."""
        import ctypes
        import torch
        lib = self.engine._lib
        dev = torch.device('cuda', self.engine.device)
        batch = torch.empty((len(images), nh, nw, 3), dtype=torch.float32, device=dev)
        for i, im in enumerate(images):
            is_f32 = im.dtype != np.uint8
            src = torch.from_numpy(np.ascontiguousarray(im, dtype=np.float32 if is_f32 else np.uint8)).to(dev)
            rc = lib.lumi_op_resize_bilinear(ctypes.c_void_p(src.data_ptr()), int(is_f32), im.shape[0], im.shape[1],
                                             ctypes.c_void_p(batch[i].data_ptr()), nh, nw, None)
            if rc != 0:
                raise RuntimeError(lib.lumi_op_last_error().decode())
        torch.cuda.synchronize(dev)
        return batch
