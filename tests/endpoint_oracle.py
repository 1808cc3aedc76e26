"""CPU oracle of the ResNet trunk truncated at any endpoint slim collects, and of Faster R-CNN on it (test
infrastructure next to ``oracle/`` and ``resnet_v2_oracle``, whose stages it reuses; with the default endpoint it
computes what they compute).

Reference wiring: ``luminoth/models/base/truncated_base_network.py:18-37, 146-169``.  Slim builds the whole network,
all four blocks at ``output_stride``, and collects the outputs of its ``conv2d``, ``bottleneck`` and
``stack_blocks_dense`` calls under their scope names; the feature map is the output whose name ends with
``truncated_base_network/<arch>/<endpoint>``, and no match is a ValueError.  This walk runs the network in slim's order,
names each collected output the same way, and stops at the endpoint:

* ``conv1``: the stem conv (v1: BN + relu; v2: bias only), before ``pool1``;
* ``blockN/unit_K/bottleneck_vX``: the unit's output (v1: relu of the sum; v2: the raw sum);
* ``.../conv1``, ``.../conv2``: conv + BN + relu (v2's conv1 reads ``preact``);
* ``.../conv3``: v1 conv + BN, v2 conv + bias, both before the residual add;
* ``.../shortcut``: the projection (v1 conv + BN, v2 conv + bias on ``preact``); identity shortcuts are not convs;
* ``blockN``: the block's last unit.
"""
import numpy as np

import resnet_v2_oracle as V2
from oracle import fasterrcnn as ofr
from oracle import resnet
from oracle import tf_ops as T
from oracle.anchors import fasterrcnn_anchors

UNITS = dict(resnet.UNITS, **V2.UNITS)


def _unit(x, wts, s, depth, stride, rate, v2, want, record):
    """One bottleneck unit at scope ``s`` (``.../bottleneck_vX``): (output, True) when ``want`` is collected inside the
    unit (only what it reads is computed), else (the unit's output, whether ``want`` is the unit).  ``record(name,
    value)`` sees each collected output and says whether it is ``want``."""
    def bias(name):
        return wts[name].astype(x.dtype)

    if v2:
        p = s + '/preact/'
        pre = T.relu(T.batch_norm_inference(x, wts[p + 'gamma'], wts[p + 'beta'], wts[p + 'moving_mean'],
                                            wts[p + 'moving_variance'], resnet.BN_EPS))
    else:
        pre = x

    def projection():
        if v2:
            return T.conv2d(pre, wts[s + '/shortcut/weights'], stride, 'SAME', bias=bias(s + '/shortcut/biases'))
        return resnet._bn(T.conv2d(x, wts[s + '/shortcut/weights'], stride, 'SAME'), wts, s + '/shortcut')

    if want == s + '/shortcut' and x.shape[-1] != depth:
        return projection(), True
    r = T.relu(resnet._bn(T.conv2d(pre, wts[s + '/conv1/weights'], 1, 'SAME'), wts, s + '/conv1'))
    if record(s + '/conv1', r):
        return r, True
    r = T.relu(resnet._bn(T.conv2d_same(r, wts[s + '/conv2/weights'], stride, rate), wts, s + '/conv2'))
    if record(s + '/conv2', r):
        return r, True
    if v2:
        r = T.conv2d(r, wts[s + '/conv3/weights'], 1, 'SAME', bias=bias(s + '/conv3/biases'))
    else:
        r = resnet._bn(T.conv2d(r, wts[s + '/conv3/weights'], 1, 'SAME'), wts, s + '/conv3')
    if record(s + '/conv3', r):
        return r, True
    if x.shape[-1] == depth:
        shortcut = x if stride == 1 else x[:, ::stride, ::stride, :]
    else:
        shortcut = projection()
        record(s + '/shortcut', shortcut)
    out = shortcut + r if v2 else T.relu(shortcut + r)
    return out, record(s, out)


def trunk(images, wts, arch, endpoint='block3', output_stride=16, scope='truncated_base_network', collect=None):
    """images (N,H,W,3) float RGB 0..255 -> the endpoint's feature map.  ``output_stride`` None builds the network of
    32.  ``collect``, a dict, receives every output collected on the way, keyed by its name relative to ``<arch>/``."""
    root = '%s/%s' % (scope, arch)
    want = '%s/%s' % (root, endpoint or 'block3')
    v2 = arch in V2.UNITS

    def record(name, value):
        if collect is not None:
            collect[name[len(root) + 1:]] = value
        return name == want

    x = resnet.subtract_means(images)
    x = T.conv2d_same(x, wts[root + '/conv1/weights'], 2)
    x = x + wts[root + '/conv1/biases'].astype(x.dtype) if v2 else T.relu(resnet._bn(x, wts, root + '/conv1'))
    if record(root + '/conv1', x):
        return x
    x = T.max_pool(x, 3, 2, 'SAME')
    target = (output_stride or 32) // 4
    current, rate = 1, 1
    for b in range(4):
        n_units = UNITS[arch][b]
        for u in range(n_units):
            unit_stride = resnet.BLOCK_STRIDE[b] if u == n_units - 1 else 1
            s = '%s/block%d/unit_%d/bottleneck_v%d' % (root, b + 1, u + 1, 2 if v2 else 1)
            if current == target:
                x, hit = _unit(x, wts, s, resnet.BASE_DEPTH[b] * 4, 1, rate, v2, want, record)
                rate *= unit_stride
            else:
                x, hit = _unit(x, wts, s, resnet.BASE_DEPTH[b] * 4, unit_stride, 1, v2, want, record)
                current *= unit_stride
            if hit:
                return x
        if record('%s/block%d' % (root, b + 1), x):
            return x
    raise ValueError('"%s" is an invalid value of endpoint for this architecture.' % want)


def fasterrcnn_forward(image, wts, config, dtype=np.float32):
    """``oracle.fasterrcnn.forward`` from the configured endpoint, for any ResNet arch.  resnet_v1_101's tail reuses
    block4's variables, so it raises TF's ValueError on an endpoint that is not 1024 channels deep."""
    m = config['model']
    bn = m['base_network']
    arch = bn['architecture']
    use_tail = bn.get('use_tail', True)
    image = np.asarray(image, dtype)
    fmap = trunk(image[None], wts, arch, bn.get('endpoint'), bn.get('output_stride', 16))
    im_shape = image.shape[:2]
    a = m['anchors']
    anchors = fasterrcnn_anchors(fmap.shape[1], fmap.shape[2], a['base_size'], a['ratios'], a['scales'], a['stride'])
    r = ofr.rpn_head(fmap, wts, m['rpn'].get('activation_function', 'relu6'))
    rp = ofr.rpn_proposal(r['rpn_cls_prob'], r['rpn_bbox_pred'], anchors, im_shape, m['rpn']['proposals'])
    out = {'conv_feature_map': fmap, 'all_anchors': anchors, 'rpn': r, 'rpn_prediction': rp}
    if not m['network'].get('with_rcnn', False):
        return out
    if arch == 'resnet_v1_101' and use_tail and fmap.shape[-1] != 1024:
        raise ValueError('Trying to share variable block4/unit_1/bottleneck_v1/shortcut/weights, but specified shape '
                         '(1, 1, %d, 2048) and found shape (1, 1, 1024, 2048).' % fmap.shape[-1])
    roi = m['rcnn']['roi']
    rp_out = ofr.roi_pool(rp['proposals'], fmap, im_shape, roi['pooled_width'], roi['pooled_height'], roi['padding'])
    head = ofr.rcnn_head(rp_out['roi_pool'], wts, m['rcnn'], arch, use_tail=use_tail)
    pred = ofr.rcnn_proposal(rp['proposals'], head['bbox_offsets'], head['cls_prob'], im_shape,
                             m['network']['num_classes'], m['rcnn']['proposals'],
                             variances=m['rcnn'].get('target_normalization_variances'))
    out.update({'roi': rp_out, 'rcnn': head, 'classification_prediction': {
        'objects': pred['objects'], 'labels': pred['proposal_label'], 'probs': pred['proposal_label_prob']}})
    return out
