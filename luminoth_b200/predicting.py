"""``PredictorNetwork`` -- drop-in for ``luminoth/utils/predicting.py:10-148``.

Same constructor and ``predict_image(image) -> [{'bbox', 'label', 'prob'}]``
(sorted by probability, integer pixel boxes in the ORIGINAL image, probs
rounded to 4 decimals).  ``predict_batch(images)`` is the batched extension
(the reference is hard-wired to batch 1, ``fasterrcnn.py:101-103``).

What changed underneath: graph build + ``session.run`` is one call into the
sm_90a engine (``lumi_predict`` / ``lumi_predict_resize``).  The aspect-preserving
resize of ``datasets/object_detection_dataset.py:71-83`` / ``utils/image.py:38-147``
runs inside the engine's forward (``lumi_predict_resize`` samples the TF1 legacy
bilinear kernel, bit-identically, in the kernels that stage the first conv's input);
only its size arithmetic (float32, like the reference) stays on the host.  Images
of different sizes in one ``predict_batch`` call are bucketed by their
preprocessed size, each bucket runs as one batched engine call, and the results
come back in the caller's order.  With ``pack_sizes=True``, images of different
preprocessed sizes share an engine call (``lumi_predict_sizes``), each at the top
left of a common canvas, with the results of separate calls.
"""
import json
import math
import os
import warnings

import numpy as np

from .config import get_model_type
from .engine import Engine, pixel_format_code, pixel_size


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
    resizes inside the engine (``Engine.predict_resize``); this restatement is its cross-check."""
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


# Packing (``pack_sizes=True``) starts a new engine call when the images of the current one would cover less than this
# share of their canvas (n x largest height x largest width): the canvas positions outside the images cost conv time.
PACK_FILL = 0.75


def _pixel_sizes(images, pixel_format):
    """The (h, w) pixel size of each image (``engine.pixel_size``); RGB images keep their old error message."""
    if pixel_format_code(pixel_format) == 0:
        for im in images:
            if im.ndim != 3 or im.shape[2] != 3:
                raise ValueError('expected an (H, W, 3) RGB image')
        return [im.shape[:2] for im in images]
    return [pixel_size(im.shape, pixel_format, im.dtype == np.uint8) for im in images]


def _format_kw(pixel_format):
    """The engine calls' pixel_format keyword: none for RGB, the engine's default (engines stood in for by callers may
    not take the keyword)."""
    return {} if pixel_format_code(pixel_format) == 0 else {'pixel_format': pixel_format}


def size_groups(targets, max_batch):
    """Today's grouping: indices bucketed by identical target (h, w) in first-seen order, each bucket cut into
    chunks of ``max_batch``."""
    buckets = {}
    for i, t in enumerate(targets):
        buckets.setdefault(tuple(t), []).append(i)
    return [idxs[s:s + max_batch] for idxs in buckets.values() for s in range(0, len(idxs), max_batch)]


def pack_groups(targets, max_batch, fill=PACK_FILL):
    """Groups for packed calls: indices sorted by orientation (landscape or square first, then portrait), then by
    height and width, cut into groups of at most ``max_batch`` that end where adding the next image would bring the
    group's fill (sum of image areas over n x canvas height x canvas width) below ``fill``."""
    order = sorted(range(len(targets)), key=lambda i: (targets[i][0] > targets[i][1], targets[i][0], targets[i][1], i))
    groups, cur, area, hc, wc = [], [], 0, 0, 0
    for i in order:
        h, w = targets[i]
        nh, nw, na = max(hc, h), max(wc, w), area + h * w
        if cur and (len(cur) == max_batch or na < fill * (len(cur) + 1) * nh * nw):
            groups.append(cur)
            cur, area, nh, nw, na = [], 0, h, w, h * w
        cur.append(i)
        area, hc, wc = na, nh, nw
    if cur:
        groups.append(cur)
    return groups


def _tile_starts(size, tile, step):
    if size <= tile:
        return [0]
    return list(range(0, size - tile, step)) + [size - tile]      # the last one shifted inward, flush with the border


def tile_grid(h, w, tile_h, tile_w, overlap):
    """Overlapping windows covering an h x w image: [(y0, x0, wh, ww)] row by row.  Windows are tile_h x tile_w
    (clipped to the image on a side no longer than a tile) and step by int(tile * (1 - overlap)), at least 1; the
    last row and column are shifted inward so every window lies inside the image.  An image no larger than a tile
    gives one whole-image window.  Windows are unique."""
    h, w, tile_h, tile_w = int(h), int(w), int(tile_h), int(tile_w)
    if h < 1 or w < 1:
        raise ValueError('tile_grid: image is %d x %d, sides must be >= 1' % (h, w))
    if tile_h < 1 or tile_w < 1:
        raise ValueError('tile_grid: tile is %d x %d, sides must be >= 1' % (tile_h, tile_w))
    if not 0.0 <= overlap < 1.0:
        raise ValueError('tile_grid: overlap must be in [0, 1), got %r' % (overlap,))
    step_h = max(1, int(tile_h * (1.0 - overlap)))
    step_w = max(1, int(tile_w * (1.0 - overlap)))
    wh, ww = min(tile_h, h), min(tile_w, w)
    return [(y0, x0, wh, ww) for y0 in _tile_starts(h, tile_h, step_h) for x0 in _tile_starts(w, tile_w, step_w)]


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

    def __init__(self, config, weights=None, device=0, max_batch=1, pack_sizes=False):
        self.class_labels = None
        self.pack_sizes = bool(pack_sizes)
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
    def predict_image(self, image, pixel_format='rgb'):
        return self.predict_batch([image], pixel_format=pixel_format)[0]

    # -- batched extension
    def predict_batch(self, images, pixel_format='rgb'):
        """Predictions for a list of (H, W, 3) images of ANY mix of sizes, in the caller's order.  Images are grouped
        by the size the preprocessing gives them (``target_size``); each group runs through the engine in chunks of
        ``max_batch`` -- a directory of equally sized frames (``predict.py:69-97``, video frames ``:100-171``) is
        one batched call per chunk instead of one call per image.  ``pixel_format`` 'bgr' takes (H, W, 3) BGR images
        (OpenCV's), 'nv12' and 'i420' (3H/2, W) uint8 frames (decoders'); they are converted to RGB in the engine's
        input staging, with the results of their RGB conversions."""
        return [format_predictions(boxes, labels, probs, scale, self.class_labels)
                for boxes, labels, probs, scale in self.predict_batch_raw(images, pixel_format=pixel_format)]

    def predict_batch_raw(self, images, pixel_format='rgb'):
        """The network's fetches per image, before the Python post-step of ``predicting.py:114-148``:
        [(objects (K,4) float32 in PREPROCESSED-image pixels, labels (K,) int32, probs (K,) float32, scale_factor)]
        in the caller's order (``lumi eval`` compares these with the scaled ground truth, ``eval.py:330-347``).
        ``pixel_format`` as in ``predict_batch``."""
        images = [np.asarray(im) for im in images]
        if not images:
            return []
        psizes = _pixel_sizes(images, pixel_format)
        fmt = _format_kw(pixel_format)
        sizes = [target_size(p, self.config) for p in psizes]
        targets = [(nh, nw) for nh, nw, _ in sizes]
        if self.pack_sizes:
            groups = pack_groups(targets, self.engine.max_batch)
        else:
            groups = size_groups(targets, self.engine.max_batch)
        touched = set(t for t, im, p in zip(targets, images, psizes) if im.dtype != np.uint8 or tuple(p) != t)
        out = [None] * len(images)
        for chunk in groups:
            shapes = set(targets[i] for i in chunk)
            srcs = [images[i] for i in chunk]
            if len(shapes) == 1 and not shapes & touched:
                # integer pixels, no resize: the uint8 entry point (the benchmark shapes)
                res = self.engine.predict_raw(np.stack(srcs), **fmt)
            else:       # the reference feeds the resized FLOAT image (predicting.py:110-112): resized in the engine's
                if any(im.dtype != np.uint8 for im in srcs):    # input staging, one call per group
                    srcs = [im.astype(np.float32, copy=False) for im in srcs]   # uint8 -> float32 is exact
                if len(shapes) == 1:
                    res = self.engine.predict_resize(srcs, *targets[chunk[0]], **fmt)
                else:
                    res = self.engine.predict_sizes(srcs, [targets[i] for i in chunk], **fmt)
            boxes, scores, labels, counts = res
            for j, i in enumerate(chunk):
                k = int(counts[j])
                out[i] = (boxes[j, :k].copy(), labels[j, :k].copy(), scores[j, :k].copy(), sizes[i][2])
        return out

    def merge_iou_threshold(self):
        """The IoU threshold ``predict_tiled`` merges windows at by default: the model's class NMS threshold, or the
        RPN's NMS threshold when Faster R-CNN runs without its RCNN."""
        m = self.config.model
        if m.type == 'ssd':
            return float(m.proposals.class_nms_threshold)
        if m.network.get('with_rcnn', False):
            return float(m.rcnn.proposals.class_nms_threshold)
        return float(m.rpn.proposals.nms_threshold)

    def tile_windows(self, shape, tile, overlap=0.2, full_image=True):
        """The windows ``predict_tiled`` runs for an image of pixel size ``shape`` (h, w, ...):
        ([(y0, x0, h, w, th, tw)], [(s_y, s_x)]), the ``tile_grid`` windows with their targets and scale factors from
        ``target_size``, and with ``full_image`` the whole image last (unless the grid already is the whole image)."""
        th_, tw_ = (tile, tile) if np.isscalar(tile) else tuple(tile)
        h, w = int(shape[0]), int(shape[1])
        grid = tile_grid(h, w, th_, tw_, overlap)
        if full_image and (0, 0, h, w) not in grid:
            grid.append((0, 0, h, w))
        wins, scales = [], []
        for y0, x0, wh, ww in grid:
            nh, nw, s = target_size((wh, ww), self.config)
            wins.append((y0, x0, wh, ww, nh, nw))
            scales.append(tuple(s) if isinstance(s, tuple) else (s, s))
        return wins, scales

    def predict_tiled(self, images, tile, overlap=0.2, full_image=True, iou_threshold=None, pixel_format='rgb'):
        """Sliced prediction of large images: each image is cut into overlapping ``tile`` x ``tile`` windows
        (``tile_grid``; ``tile`` may be an (h, w) pair), each window runs at the model's resolution
        (``target_size``), and the windows' boxes are mapped back into the image and merged across the seams by
        per-label NMS at ``iou_threshold`` (default ``merge_iou_threshold()``), all in one engine call
        (``Engine.predict_windows``).  With ``full_image`` the whole image is also predicted at its own target size,
        so objects larger than a tile are not lost at the seams.  ``pixel_format`` as in ``predict_batch``.  Returns,
        per image, the ``predict_image`` format with boxes in the image's own pixels."""
        images = [np.asarray(im) for im in images]
        psizes = _pixel_sizes(images, pixel_format)
        if not images:
            return []
        if iou_threshold is None:
            iou_threshold = self.merge_iou_threshold()
        windows, scales = [], []
        for i, p in enumerate(psizes):
            wins, scl = self.tile_windows(p, tile, overlap, full_image)
            windows += [(i,) + wdw for wdw in wins]
            scales += scl
        if any(im.dtype != np.uint8 for im in images):
            images = [im.astype(np.float32, copy=False) for im in images]     # uint8 -> float32 is exact
        boxes, scores, labels, counts = self.engine.predict_windows(images, windows, scales, iou_threshold,
                                                                    **_format_kw(pixel_format))
        return [format_predictions(boxes[i, :counts[i]], labels[i, :counts[i]], scores[i, :counts[i]], 1.0,
                                   self.class_labels) for i in range(len(images))]
