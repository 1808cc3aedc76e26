"""CPU oracle of the pre-activation slim ``resnet_v2_{50,101,152}`` trunk to ``block3`` and of Faster R-CNN on it
(test infrastructure, next to ``oracle/``, whose stages it reuses).

Reference wiring: ``luminoth/models/base/base_network.py:94-101`` calls slim's ``resnet_v2_NN`` with
``output_stride=16`` after the same RGB mean subtraction as v1 (:153-157); the endpoint is ``block3`` and
``_build_tail`` is the identity for every v2 arch (``truncated_base_network.py:56-95``).  The arithmetic is
``tf.contrib.slim.nets.resnet_v2`` (third-party), restated from its published definition:

* stem: ``conv2d_same(64, 7, stride 2)`` with a bias, no batch norm, no activation, then ``max_pool 3x3/2 SAME``;
* unit ``bottleneck_v2``: ``preact = relu(BN(x))`` (variables directly under ``preact/``); the shortcut is
  ``subsample(x, stride)`` when the depth is unchanged, else a biased 1x1 conv of ``preact``; conv1 / conv2 with
  batch norm and relu, conv3 with a bias only; the output is the raw sum, no activation;
* units (3, 4, 6, 3) / (3, 4, 23, 3) / (3, 8, 36, 3), stride on the last unit of each block, like v1.
"""
import numpy as np

from oracle import fasterrcnn as ofr
from oracle import resnet
from oracle import tf_ops as T
from oracle.anchors import fasterrcnn_anchors

UNITS = {'resnet_v2_50': (3, 4, 6, 3), 'resnet_v2_101': (3, 4, 23, 3), 'resnet_v2_152': (3, 8, 36, 3)}


def bottleneck_v2(x, wts, scope, depth, stride, rate=1):
    s = scope + '/bottleneck_v2'
    p = s + '/preact/'
    preact = T.relu(T.batch_norm_inference(x, wts[p + 'gamma'], wts[p + 'beta'], wts[p + 'moving_mean'],
                                           wts[p + 'moving_variance'], resnet.BN_EPS))
    if x.shape[-1] == depth:
        shortcut = x if stride == 1 else x[:, ::stride, ::stride, :]
    else:
        shortcut = T.conv2d(preact, wts[s + '/shortcut/weights'], stride, 'SAME', bias=wts[s + '/shortcut/biases'])
    r = T.conv2d(preact, wts[s + '/conv1/weights'], 1, 'SAME')
    r = T.relu(resnet._bn(r, wts, s + '/conv1'))
    r = T.conv2d_same(r, wts[s + '/conv2/weights'], stride, rate)
    r = T.relu(resnet._bn(r, wts, s + '/conv2'))
    r = T.conv2d(r, wts[s + '/conv3/weights'], 1, 'SAME', bias=wts[s + '/conv3/biases'])
    return shortcut + r


def trunk(images, wts, arch, scope='truncated_base_network', output_stride=16):
    """images (N,H,W,3) float RGB 0..255 -> block3 feature map (N,H/16,W/16,1024); v1 archs go to oracle.resnet."""
    if arch not in UNITS:
        return resnet.trunk(images, wts, arch, scope, output_stride)
    root = '%s/%s' % (scope, arch)
    x = resnet.subtract_means(images)
    x = T.conv2d_same(x, wts[root + '/conv1/weights'], 2) + wts[root + '/conv1/biases'].astype(images.dtype)
    x = T.max_pool(x, 3, 2, 'SAME')
    target = output_stride // 4
    current, rate = 1, 1
    for b in range(3):
        n_units = UNITS[arch][b]
        for u in range(n_units):
            unit_stride = resnet.BLOCK_STRIDE[b] if u == n_units - 1 else 1
            sc = '%s/block%d/unit_%d' % (root, b + 1, u + 1)
            if current == target:
                x = bottleneck_v2(x, wts, sc, resnet.BASE_DEPTH[b] * 4, 1, rate)
                rate *= unit_stride
            else:
                x = bottleneck_v2(x, wts, sc, resnet.BASE_DEPTH[b] * 4, unit_stride, 1)
                current *= unit_stride
    return x


def fasterrcnn_forward(image, wts, config, dtype=np.float32):
    """``oracle.fasterrcnn.forward`` for any ResNet arch: the same stages after the trunk (no v2 arch has a tail)."""
    m = config['model']
    arch = m['base_network']['architecture']
    if arch not in UNITS:
        return ofr.forward(image, wts, config, dtype)
    image = np.asarray(image, dtype)
    fmap = trunk(image[None], wts, arch, output_stride=m['base_network'].get('output_stride', 16))
    im_shape = image.shape[:2]
    a = m['anchors']
    anchors = fasterrcnn_anchors(fmap.shape[1], fmap.shape[2], a['base_size'], a['ratios'], a['scales'], a['stride'])
    r = ofr.rpn_head(fmap, wts, m['rpn'].get('activation_function', 'relu6'))
    rp = ofr.rpn_proposal(r['rpn_cls_prob'], r['rpn_bbox_pred'], anchors, im_shape, m['rpn']['proposals'])
    out = {'conv_feature_map': fmap, 'all_anchors': anchors, 'rpn': r, 'rpn_prediction': rp}
    if not m['network'].get('with_rcnn', False):
        return out
    roi = m['rcnn']['roi']
    rp_out = ofr.roi_pool(rp['proposals'], fmap, im_shape, roi['pooled_width'], roi['pooled_height'], roi['padding'])
    head = ofr.rcnn_head(rp_out['roi_pool'], wts, m['rcnn'], arch, use_tail=m['base_network'].get('use_tail', True))
    pred = ofr.rcnn_proposal(rp['proposals'], head['bbox_offsets'], head['cls_prob'], im_shape,
                             m['network']['num_classes'], m['rcnn']['proposals'],
                             variances=m['rcnn'].get('target_normalization_variances'))
    out.update({'roi': rp_out, 'rcnn': head, 'classification_prediction': {
        'objects': pred['objects'], 'labels': pred['proposal_label'], 'probs': pred['proposal_label_prob']}})
    return out
