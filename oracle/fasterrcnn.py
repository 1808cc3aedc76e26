"""Faster R-CNN inference forward (oracle only).

Each function cites the reference lines it follows (paths under
``luminoth/models/fasterrcnn/``).  Inference only: ``gt_boxes is None``,
``is_training=False``; batch is always one image like the reference
(``fasterrcnn.py:101-103``).
"""
import numpy as np

from . import tf_ops as T
from . import resnet
from .anchors import fasterrcnn_anchors
from .bbox import decode, clip_boxes, change_order


def cfg_get(cfg, path, default=None):
    cur = cfg
    for k in path.split('.'):
        if cur is None or k not in cur:
            return default
        cur = cur[k]
    return cur


def activation(name):
    """``utils/vars.py:80-88`` (get_activation_function): None or '' is the identity, else the tf.nn function of
    that name (relu and relu6 here)."""
    if not name:
        return lambda a: a
    return {'relu6': T.relu6, 'relu': T.relu}[name]


# ---------------------------------------------------------------- RPN
def rpn_head(fmap, wts, act='relu6', scope='fasterrcnn/rpn'):
    """``rpn.py:67-90,136-170``: 3x3 conv(+bias) -> activation -> 1x1 cls (2A)
    and 1x1 bbox (4A) -> reshape(-1,2) softmax / reshape(-1,4)."""
    x = T.conv2d(fmap, wts[scope + '/conv/w'], 1, 'SAME', bias=wts[scope + '/conv/b'])
    x = activation(act)(x)
    cls = T.conv2d(x, wts[scope + '/cls_conv/w'], 1, 'VALID', bias=wts[scope + '/cls_conv/b'])
    box = T.conv2d(x, wts[scope + '/bbox_conv/w'], 1, 'VALID', bias=wts[scope + '/bbox_conv/b'])
    cls_score = cls.reshape(-1, 2)
    cls_prob = T.softmax(cls_score)
    bbox_pred = box.reshape(-1, 4)
    return {'rpn_feature': x, 'rpn_cls_score': cls_score, 'rpn_cls_prob': cls_prob,
            'rpn_bbox_pred': bbox_pred}


def rpn_proposal(rpn_cls_prob, rpn_bbox_pred, all_anchors, im_shape, pcfg):
    """``rpn_proposal.py:41-197``."""
    f32 = np.float32
    all_scores = rpn_cls_prob[:, 1].reshape(-1).astype(f32)
    all_anchors = np.asarray(all_anchors)
    rpn_bbox_pred = rpn_bbox_pred.astype(f32)
    if pcfg.get('filter_outside_anchors', False):            # :71-90
        a = all_anchors
        keep = ((a[:, 0] >= 0) & (a[:, 1] >= 0) &
                (a[:, 2] < im_shape[1]) & (a[:, 3] < im_shape[0]))
        all_anchors = a[keep]; rpn_bbox_pred = rpn_bbox_pred[keep]
        all_scores = all_scores[keep]
    all_proposals = decode(all_anchors, rpn_bbox_pred)       # :93
    min_prob = all_scores >= f32(float(pcfg.get('min_prob_threshold', 0.0)))   # :96-98
    x0, y0, x1, y1 = (all_proposals[:, i] for i in range(4))
    area_ok = (np.maximum(x1 - x0, f32(0)) * np.maximum(y1 - y0, f32(0))) > 0  # :101-105
    pf = area_ok & min_prob
    unsorted_scores = all_scores[pf]
    unsorted_proposals = all_proposals[pf]
    proposals_unclipped = unsorted_proposals.copy()
    clip_after = bool(pcfg.get('clip_after_nms', False))
    if not clip_after:
        unsorted_proposals = clip_boxes(unsorted_proposals, im_shape)   # :121-123
    k = min(int(pcfg['pre_nms_top_n']), unsorted_scores.shape[0])       # :139
    top_scores, top_idx = T.top_k(unsorted_scores, k)
    sorted_top_proposals = unsorted_proposals[top_idx]
    if pcfg.get('apply_nms', True):
        tf_order = change_order(sorted_top_proposals)
        sel = T.non_max_suppression(tf_order, top_scores, int(pcfg['post_nms_top_n']),
                                    float(pcfg['nms_threshold']))
        proposals = change_order(tf_order[sel])
        scores = top_scores[sel]
    else:
        proposals, scores = sorted_top_proposals, top_scores
    if clip_after:
        proposals = clip_boxes(proposals, im_shape)
    return {'proposals': proposals.astype(f32).reshape(-1, 4), 'scores': scores,
            'sorted_top_scores': top_scores, 'sorted_top_proposals': sorted_top_proposals,
            'unsorted_proposals': unsorted_proposals, 'unsorted_scores': unsorted_scores,
            'all_proposals': all_proposals, 'all_scores': all_scores,
            'proposals_unclipped': proposals_unclipped}


# ---------------------------------------------------------------- ROI pooling
def roi_pool(proposals, fmap, im_shape, pooled_w=7, pooled_h=7, padding='VALID'):
    """``roi_pool.py:37-95``: boxes normalised by IMAGE h/w (quirk Q3),
    crop_and_resize to [pooled_w*2, pooled_h*2] (sic, :77), 2x2/2 max pool."""
    f32 = fmap.dtype.type
    p = proposals.astype(fmap.dtype)
    h, w = f32(im_shape[0]), f32(im_shape[1])
    bboxes = np.stack([p[:, 1] / h, p[:, 0] / w, p[:, 3] / h, p[:, 2] / w], axis=1)
    ind = np.zeros((p.shape[0],), np.int32)
    crops = T.crop_and_resize(fmap, bboxes, ind, pooled_w * 2, pooled_h * 2)
    if crops.shape[0] == 0:
        pooled = np.zeros((0, pooled_w, pooled_h, fmap.shape[-1]), fmap.dtype)
    else:
        pooled = T.max_pool(crops, 2, 2, padding)
    return {'roi_pool': pooled, 'crops': crops, 'bboxes': bboxes}


# ---------------------------------------------------------------- RCNN
def rcnn_head(pooled, wts, rcfg, arch, scope='fasterrcnn/rcnn', use_tail=True):
    """``rcnn.py:174-222``: tail -> mean(7x7) -> flatten -> [fc_i + act] ->
    fc_classifier softmax / fc_bbox."""
    feats = resnet.tail(pooled, wts, arch, use_tail=use_tail)
    if rcfg.get('use_mean', True):
        if feats.shape[0]:
            feats = feats.mean(axis=(1, 2), dtype=feats.dtype)
        else:
            feats = feats.reshape(0, feats.shape[-1])
    net = feats.reshape(feats.shape[0], int(np.prod(feats.shape[1:])))   # tf.contrib.layers.flatten: known inner size
    act = activation(rcfg.get('activation_function', 'relu6'))
    dt = net.dtype
    for i, _ in enumerate(rcfg.get('layer_sizes') or []):
        net = act(net @ wts['%s/fc_%d/w' % (scope, i)].astype(dt) + wts['%s/fc_%d/b' % (scope, i)].astype(dt))
    cls_score = net @ wts[scope + '/fc_classifier/w'].astype(dt) + wts[scope + '/fc_classifier/b'].astype(dt)
    cls_prob = T.softmax(cls_score)
    bbox_offsets = net @ wts[scope + '/fc_bbox/w'].astype(dt) + wts[scope + '/fc_bbox/b'].astype(dt)
    return {'features': net, 'cls_score': cls_score, 'cls_prob': cls_prob,
            'bbox_offsets': bbox_offsets}


def rcnn_proposal(proposals, bbox_pred, cls_prob, im_shape, num_classes, pcfg,
                  variances=None):
    """``rcnn_proposal.py:46-164``."""
    f32 = np.float32
    proposals = np.asarray(proposals, f32)
    bbox_pred = np.asarray(bbox_pred, f32)
    cls_prob = np.asarray(cls_prob, f32)
    min_prob = f32(pcfg.get('min_prob_threshold') or 0.0)
    sel_boxes, sel_probs, sel_labels = [], [], []
    for c in range(num_classes):
        class_prob = cls_prob[:, c + 1]
        raw = decode(proposals, bbox_pred[:, 4 * c:4 * c + 4], variances=variances)
        objs = clip_boxes(raw, im_shape)
        prob_ok = class_prob >= min_prob
        area_ok = (np.maximum(objs[:, 2] - objs[:, 0], f32(0)) *
                   np.maximum(objs[:, 3] - objs[:, 1], f32(0))) > 0
        ok = area_ok & prob_ok
        objs = objs[ok]; class_prob = class_prob[ok]
        tf_objs = change_order(objs)
        sel = T.non_max_suppression(tf_objs, class_prob, int(pcfg['class_max_detections']),
                                    float(pcfg['class_nms_threshold']))
        sel_boxes.append(change_order(tf_objs[sel]).reshape(-1, 4))
        sel_probs.append(class_prob[sel])
        sel_labels.append(np.full((sel.shape[0],), c, np.int32))
    objects = np.concatenate(sel_boxes, axis=0)
    labels = np.concatenate(sel_labels, axis=0)
    probs = np.concatenate(sel_probs, axis=0)
    k = min(int(pcfg['total_max_detections']), probs.shape[0])
    top_probs, top_idx = T.top_k(probs, k)
    return {'objects': objects[top_idx].reshape(-1, 4), 'proposal_label': labels[top_idx],
            'proposal_label_prob': top_probs, 'selected_boxes': sel_boxes,
            'selected_probs': sel_probs, 'selected_labels': sel_labels}


# ---------------------------------------------------------------- full model
def forward(image, wts, config, dtype=np.float32):
    """``FasterRCNN._build`` (``fasterrcnn.py:70-156``), inference.
    image: (H,W,3) (already resized); returns prediction dict.  dtype=float64
    runs the conv / FC arithmetic in double (tests use it as the exact-arithmetic
    yardstick for fp32 noise); box post-processing always runs in fp32 like TF."""
    m = config['model']
    arch = m['base_network']['architecture']
    image = np.asarray(image, dtype)
    fmap = resnet.trunk(image[None], wts, arch,
                        output_stride=m['base_network'].get('output_stride', 16))
    im_shape = image.shape[:2]
    a = m['anchors']
    anchors = fasterrcnn_anchors(fmap.shape[1], fmap.shape[2], a['base_size'],
                                 a['ratios'], a['scales'], a['stride'])
    r = rpn_head(fmap, wts, m['rpn'].get('activation_function', 'relu6'))
    rp = rpn_proposal(r['rpn_cls_prob'], r['rpn_bbox_pred'], anchors, im_shape,
                      m['rpn']['proposals'])
    out = {'conv_feature_map': fmap, 'all_anchors': anchors, 'rpn': r,
           'rpn_prediction': rp}
    if not m['network'].get('with_rcnn', False):
        return out
    roi = m['rcnn']['roi']
    rp_out = roi_pool(rp['proposals'], fmap, im_shape, roi['pooled_width'],
                      roi['pooled_height'], roi['padding'])
    head = rcnn_head(rp_out['roi_pool'], wts, m['rcnn'], arch,
                     use_tail=m['base_network'].get('use_tail', True))
    pred = rcnn_proposal(rp['proposals'], head['bbox_offsets'], head['cls_prob'], im_shape,
                         m['network']['num_classes'], m['rcnn']['proposals'],
                         variances=m['rcnn'].get('target_normalization_variances'))
    out.update({'roi': rp_out, 'rcnn': head, 'classification_prediction': {
        'objects': pred['objects'], 'labels': pred['proposal_label'],
        'probs': pred['proposal_label_prob']}})
    return out
