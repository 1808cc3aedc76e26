"""SSD inference forward at the configured fixed size (oracle only).

``luminoth/models/ssd/ssd.py:37-195`` (heads, softmax, anchors) and
``luminoth/models/ssd/proposal.py:41-171`` (per-class filter -> decode ->
clip -> area filter -> NMS -> concat -> top_k).  The reference has NO tests
for SSD: parity unpinned (see package docstring).
"""
import numpy as np

from . import tf_ops as T
from .anchors import ssd_anchors
from .bbox import decode, clip_boxes, change_order
from .vgg import ssd_feature_maps


def ssd_heads(fmaps, wts, num_classes, anchors_per_point, scope='ssd'):
    """``ssd.py:73-109``: per feature map two 3x3 SAME convs (+bias)."""
    offs, scores = [], []
    for i, fm in enumerate(fmaps.values()):
        n = 'MultiBox_%d' % i
        o = T.conv2d(fm, wts['%s/%s_offsets_conv/w' % (scope, n)], 1, 'SAME',
                     bias=wts['%s/%s_offsets_conv/b' % (scope, n)])
        c = T.conv2d(fm, wts['%s/%s_classes_conv/w' % (scope, n)], 1, 'SAME',
                     bias=wts['%s/%s_classes_conv/b' % (scope, n)])
        offs.append(o.reshape(-1, 4))
        scores.append(c.reshape(-1, num_classes + 1))
    bbox_offsets = np.concatenate(offs, axis=0)
    class_scores = np.concatenate(scores, axis=0)
    return bbox_offsets, class_scores, T.softmax(class_scores)


def ssd_proposal(cls_prob, loc_pred, all_anchors, im_shape, num_classes, pcfg, variances):
    """``proposal.py:41-171``."""
    f32 = np.float32
    cls_prob = np.asarray(cls_prob, f32); loc_pred = np.asarray(loc_pred, f32)
    all_anchors = np.asarray(all_anchors, f32)
    min_prob = f32(pcfg.get('min_prob_threshold') or 0.0)
    sel_boxes, sel_probs, sel_labels = [], [], []
    for c in range(num_classes):
        p = cls_prob[:, c + 1]
        keep = p >= min_prob
        p = p[keep]
        raw = decode(all_anchors[keep], loc_pred[keep], variances)
        clipped = clip_boxes(raw, im_shape)
        ok = (np.maximum(clipped[:, 2] - clipped[:, 0], f32(0)) *
              np.maximum(clipped[:, 3] - clipped[:, 1], f32(0))) > 0
        props = clipped[ok]; p = p[ok]
        tf_props = change_order(props)
        sel = T.non_max_suppression(tf_props, p, int(pcfg['class_max_detections']),
                                    float(pcfg['class_nms_threshold']))
        sel_boxes.append(tf_props[sel].reshape(-1, 4))
        sel_probs.append(p[sel])
        sel_labels.append(np.full((sel.shape[0],), c, np.int32))
    proposals = change_order(np.concatenate(sel_boxes, axis=0))
    labels = np.concatenate(sel_labels, axis=0)
    probs = np.concatenate(sel_probs, axis=0)
    k = min(int(pcfg['total_max_detections']), probs.shape[0])
    top_probs, idx = T.top_k(probs, k)
    return {'objects': proposals[idx].reshape(-1, 4), 'labels': labels[idx], 'probs': top_probs}


def forward(image, wts, config, dtype=np.float32):
    """``SSD._build`` inference; image (fixed_height, fixed_width, 3) raw 0..255, uint8 or float (dtype=float64: see
    fasterrcnn.forward)."""
    m = config['model']
    ip = config['dataset']['image_preprocessing']
    image_shape = [ip['fixed_height'], ip['fixed_width'], 3]     # ssd.py:30-31,63
    image = np.asarray(image, dtype)
    assert list(image.shape) == image_shape, image.shape
    fmaps = ssd_feature_maps(image[None], wts)
    nc = m['network']['num_classes']
    a = m['anchors']
    loc, scores, probs = ssd_heads(fmaps, wts, nc, a['anchors_per_point'])
    shapes = [fm.shape[1:3] for fm in fmaps.values()]
    anchors = ssd_anchors(shapes, a['min_scale'], a['max_scale'], a['ratios'],
                          a['anchors_per_point'], image_shape)
    pred = ssd_proposal(probs, loc, anchors, (float(image.shape[0]), float(image.shape[1])),
                        nc, m['proposals'], m['variances'])
    return {'feature_maps': fmaps, 'loc_pred': loc, 'cls_pred': scores, 'cls_prob': probs,
            'all_anchors': anchors, 'classification_prediction': pred}
