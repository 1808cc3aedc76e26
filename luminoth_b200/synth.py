"""Synthetic (random-init) weights and images for tests and benchmarks.

The reference initialises randomly when no checkpoint exists
(``luminoth/utils/predicting.py:64-72``) but TF's RNG stream cannot be
reproduced, so the harness owns the arrays and feeds the SAME dict -- keyed by
TF variable name, TF layouts (conv ``[kh,kw,Cin,Cout]``, linear ``[in,out]``)
-- to the CPU oracle and to the engine (SURVEY.md section 8d).

Variable names follow Sonnet/slim scoping (SURVEY.md section 8b):
``truncated_base_network/<arch>/...``, ``fasterrcnn/rpn/...``,
``fasterrcnn/rcnn/...``, ``ssd/ssd_feature_extractor/...``, ``ssd/MultiBox_i_*``.
Init distributions: ``models/fasterrcnn/base_config.yml:185-199,246-261``
('reference' profile); the 'peaky' profile scales the classifier / box
regressors so probabilities spread and NMS has real work.
"""
import re

import numpy as np

RESNET_UNITS = {'resnet_v1_50': (3, 4, 6, 3), 'resnet_v1_101': (3, 4, 23, 3), 'resnet_v1_152': (3, 8, 36, 3),
                'resnet_v2_50': (3, 4, 6, 3), 'resnet_v2_101': (3, 4, 23, 3), 'resnet_v2_152': (3, 8, 36, 3)}
BASE_DEPTH = (64, 128, 256, 512)
# resnet_v2 adds every unit's conv3 output to the raw residual stream, so its scale grows with depth: conv3 is drawn
# V2_CONV3_SCALE / sqrt(units in the block) times He init, which keeps block3 at O(1-10) up to resnet_v2_152
V2_CONV3_SCALE = 0.6


def _conv(rng, kh, kw, cin, cout, std=None):
    if std is None:
        std = np.sqrt(2.0 / (kh * kw * cin))
    return (rng.standard_normal((kh, kw, cin, cout)) * std).astype(np.float32)


def _bn(rng, wts, scope, c, gamma_scale=1.0):
    p = scope + '/BatchNorm/'
    wts[p + 'gamma'] = (rng.uniform(0.8, 1.2, c) * gamma_scale).astype(np.float32)
    wts[p + 'beta'] = (rng.standard_normal(c) * 0.05).astype(np.float32)
    wts[p + 'moving_mean'] = (rng.standard_normal(c) * 0.05).astype(np.float32)
    wts[p + 'moving_variance'] = rng.uniform(0.8, 1.2, c).astype(np.float32)


def _bias(rng, c):
    return (rng.standard_normal(c) * 0.05).astype(np.float32)


def _v2_block(rng, wts, root, arch, b):
    """One block of slim resnet_v2 (pre-activation) units."""
    bd = BASE_DEPTH[b]
    depth = bd * 4
    cin = BASE_DEPTH[b - 1] * 4 if b else 64
    for u in range(RESNET_UNITS[arch][b]):
        s = '%s/block%d/unit_%d/bottleneck_v2' % (root, b + 1, u + 1)
        p = s + '/preact/'
        wts[p + 'gamma'] = rng.uniform(0.8, 1.2, cin).astype(np.float32)
        wts[p + 'beta'] = (rng.standard_normal(cin) * 0.05).astype(np.float32)
        wts[p + 'moving_mean'] = (rng.standard_normal(cin) * 0.05).astype(np.float32)
        wts[p + 'moving_variance'] = rng.uniform(0.8, 1.2, cin).astype(np.float32)
        if cin != depth:
            wts[s + '/shortcut/weights'] = _conv(rng, 1, 1, cin, depth)
            wts[s + '/shortcut/biases'] = _bias(rng, depth)
        wts[s + '/conv1/weights'] = _conv(rng, 1, 1, cin, bd)
        _bn(rng, wts, s + '/conv1', bd)
        wts[s + '/conv2/weights'] = _conv(rng, 3, 3, bd, bd)
        _bn(rng, wts, s + '/conv2', bd)
        wts[s + '/conv3/weights'] = _conv(rng, 1, 1, bd, depth,
                                          std=V2_CONV3_SCALE * np.sqrt(2.0 / bd / RESNET_UNITS[arch][b]))
        wts[s + '/conv3/biases'] = _bias(rng, depth)
        cin = depth


def _v1_block(rng, wts, root, arch, b):
    """One block of slim resnet_v1 units."""
    bd = BASE_DEPTH[b]
    depth = bd * 4
    cin = BASE_DEPTH[b - 1] * 4 if b else 64
    for u in range(RESNET_UNITS[arch][b]):
        s = '%s/block%d/unit_%d/bottleneck_v1' % (root, b + 1, u + 1)
        if cin != depth:
            wts[s + '/shortcut/weights'] = _conv(rng, 1, 1, cin, depth)
            _bn(rng, wts, s + '/shortcut', depth)
        wts[s + '/conv1/weights'] = _conv(rng, 1, 1, cin, bd)
        _bn(rng, wts, s + '/conv1', bd)
        wts[s + '/conv2/weights'] = _conv(rng, 3, 3, bd, bd)
        _bn(rng, wts, s + '/conv2', bd)
        wts[s + '/conv3/weights'] = _conv(rng, 1, 1, bd, depth)
        _bn(rng, wts, s + '/conv3', depth, gamma_scale=0.25)
        cin = depth


def resnet_v2_weights(rng, arch, scope='truncated_base_network'):
    """slim resnet_v2 (pre-activation) variables through block3."""
    wts = {}
    root = '%s/%s' % (scope, arch)
    wts[root + '/conv1/weights'] = _conv(rng, 7, 7, 3, 64, std=np.sqrt(2.0 / 147) / 64.0)
    wts[root + '/conv1/biases'] = _bias(rng, 64)
    for b in range(3):
        _v2_block(rng, wts, root, arch, b)
    return wts


def resnet_weights(rng, arch, with_block4, scope='truncated_base_network'):
    if arch.startswith('resnet_v2'):
        return resnet_v2_weights(rng, arch, scope)
    wts = {}
    root = '%s/%s' % (scope, arch)
    # conv1 sees raw pixels minus mean (|x| ~ 60 rms): scale the stem down so
    # activations stay O(1) like a trained net.
    wts[root + '/conv1/weights'] = _conv(rng, 7, 7, 3, 64, std=np.sqrt(2.0 / 147) / 64.0)
    _bn(rng, wts, root + '/conv1', 64)
    for b in range(4 if with_block4 else 3):
        _v1_block(rng, wts, root, arch, b)
    return wts


ENDPOINT_PARTS = ('conv1', 'conv2', 'conv3', 'shortcut')


def parse_endpoint(arch, endpoint):
    """``(block, unit, part, depth)`` of a Faster R-CNN ``base_network.endpoint`` among the outputs slim's resnet
    collects: block -1 is the stem ``conv1``, ``part`` None a unit's output (``blockN`` is its last unit's).  Anything
    else raises the reference's ValueError (``truncated_base_network.py:146-169``)."""
    units = RESNET_UNITS[arch]
    kind = 'bottleneck_v2' if arch.startswith('resnet_v2') else 'bottleneck_v1'
    if endpoint == 'conv1':
        return -1, 0, None, 64
    for b in range(4):
        deep = BASE_DEPTH[b] * 4
        if endpoint == 'block%d' % (b + 1):
            return b, units[b] - 1, None, deep
        for u in range(units[b]):
            s = 'block%d/unit_%d/%s' % (b + 1, u + 1, kind)
            if endpoint == s:
                return b, u, None, deep
            for p in ENDPOINT_PARTS:
                if endpoint == s + '/' + p and (p != 'shortcut' or u == 0):    # only a block's first unit projects
                    return b, u, p, BASE_DEPTH[b] if p in ('conv1', 'conv2') else deep
    raise ValueError('"truncated_base_network/%s/%s" is an invalid value of endpoint for this architecture.'
                     % (arch, endpoint))


def _truncate(wts, arch, endpoint, tail, scope='truncated_base_network'):
    """Drop the trunk variables the forward to ``endpoint`` never reads (keeping block4 for the tail)."""
    eb, eu, epart, _ = parse_endpoint(arch, endpoint)
    unit_var = re.compile(r'%s/%s/block(\d)/unit_(\d+)/bottleneck_v\d/(\w+)/' % (scope, arch))

    def reads(key):
        m = unit_var.match(key)
        if not m:
            return True                         # the stem, and everything outside the trunk
        b, u, part = int(m.group(1)) - 1, int(m.group(2)) - 1, m.group(3)
        if b == 3 and tail:
            return True
        if (b, u) != (eb, eu):
            return (b, u) < (eb, eu)
        if epart is None or part == 'preact':
            return True
        if 'shortcut' in (part, epart):         # the shortcut only feeds the unit's sum
            return part == epart
        return ENDPOINT_PARTS.index(part) <= ENDPOINT_PARTS.index(epart)
    return {k: v for k, v in wts.items() if reads(k)}


def fasterrcnn_weights(config, seed=0, profile='peaky'):
    m = config['model']
    bn = m['base_network']
    arch = bn['architecture']
    if arch not in RESNET_UNITS:
        raise ValueError('synthetic weights: unsupported architecture %r' % arch)
    endpoint = bn.get('endpoint') or 'block3'
    block, _, _, depth = parse_endpoint(arch, endpoint)
    rng = np.random.default_rng(seed)
    wts = resnet_weights(rng, arch, with_block4=(arch == 'resnet_v1_101'))
    if endpoint != 'block3':
        if block == 3 and arch != 'resnet_v1_101':
            # a generator of its own: the draws of every block3 configuration stay as they are
            block4 = _v2_block if arch.startswith('resnet_v2') else _v1_block
            block4(np.random.default_rng([seed, 4]), wts, 'truncated_base_network/' + arch, arch, 3)
        tail = arch == 'resnet_v1_101' and bn.get('use_tail', True) and m['network'].get('with_rcnn', False)
        wts = _truncate(wts, arch, endpoint, tail)
    a = m['anchors']
    A = len(a['scales']) * len(a['ratios'])
    C = m['network']['num_classes']
    nch = m['rpn']['num_channels']
    kh, kw = m['rpn']['kernel_shape']
    peaky = profile == 'peaky'
    r = 'fasterrcnn/rpn'
    wts[r + '/conv/w'] = _conv(rng, kh, kw, depth, nch, std=0.01)
    wts[r + '/conv/b'] = (rng.standard_normal(nch) * 0.01).astype(np.float32)
    wts[r + '/cls_conv/w'] = _conv(rng, 1, 1, nch, 2 * A, std=0.02 if peaky else 0.01)
    wts[r + '/cls_conv/b'] = (rng.standard_normal(2 * A) * 0.01).astype(np.float32)
    wts[r + '/bbox_conv/w'] = _conv(rng, 1, 1, nch, 4 * A, std=0.005 if peaky else 0.001)
    wts[r + '/bbox_conv/b'] = (rng.standard_normal(4 * A) * 0.001).astype(np.float32)
    d = 2048 if arch == 'resnet_v1_101' and bn.get('use_tail', True) and depth == 1024 else depth   # the tail's output
    if not m['rcnn'].get('use_mean', True):
        d *= m['rcnn']['roi']['pooled_width'] * m['rcnn']['roi']['pooled_height']
    c = 'fasterrcnn/rcnn'
    for i, n in enumerate(m['rcnn'].get('layer_sizes') or []):
        wts['%s/fc_%d/w' % (c, i)] = (rng.standard_normal((d, n)) * np.sqrt(2.0 / (d + n))).astype(np.float32)
        wts['%s/fc_%d/b' % (c, i)] = np.zeros(n, np.float32)
        d = n
    wcls = rng.standard_normal((d, C + 1))
    if peaky:       # centre over features: pooled features are all-positive, so an
        wcls -= wcls.mean(axis=0, keepdims=True)   # uncentred draw makes one class win everywhere
    wts[c + '/fc_classifier/w'] = (wcls * (0.03 if peaky else 0.01)).astype(np.float32)
    wts[c + '/fc_classifier/b'] = (rng.standard_normal(C + 1) * 0.01).astype(np.float32)
    wts[c + '/fc_bbox/w'] = (rng.standard_normal((d, 4 * C)) * (0.01 if peaky else 0.001)).astype(np.float32)
    wts[c + '/fc_bbox/b'] = (rng.standard_normal(4 * C) * 0.001).astype(np.float32)
    return wts


SSD_VGG = [('conv1', 2, 64), ('conv2', 2, 128), ('conv3', 3, 256), ('conv4', 3, 512),
           ('conv5', 3, 512)]
SSD_EXTRA = [('conv6', 3, 512, 1024), ('conv7', 1, 1024, 1024), ('conv8_1', 1, 1024, 256),
             ('conv8_2', 3, 256, 512), ('conv9_1', 1, 512, 128), ('conv9_2', 3, 128, 256),
             ('conv10_1', 1, 256, 128), ('conv10_2', 3, 128, 256), ('conv11_1', 1, 256, 128),
             ('conv11_2', 3, 128, 256)]
SSD_FMAP_CH = [512, 1024, 512, 256, 256, 256]


def ssd_weights(config, seed=0, profile='peaky'):
    m = config['model']
    rng = np.random.default_rng(seed)
    wts = {}
    s = 'ssd/ssd_feature_extractor'
    cin = 3
    for name, reps, cout in SSD_VGG:
        for r in range(reps):
            p = '%s/vgg_16/%s/%s_%d' % (s, name, name, r + 1)
            std = np.sqrt(2.0 / (9 * cin)) / (64.0 if cin == 3 else 1.0)   # raw 0..255 input
            wts[p + '/weights'] = _conv(rng, 3, 3, cin, cout, std=std)
            wts[p + '/biases'] = (rng.standard_normal(cout) * 0.01).astype(np.float32)
            cin = cout
    wts[s + '/conv_4_3_norm/gamma'] = np.full((1, 1, 1, 512), 20.0, np.float32)
    for name, k, ci, co in SSD_EXTRA:
        wts['%s/extra_feature_layers/%s/w' % (s, name)] = _conv(rng, k, k, ci, co)
        wts['%s/extra_feature_layers/%s/b' % (s, name)] = (rng.standard_normal(co) * 0.01).astype(np.float32)
    C = m['network']['num_classes']
    peaky = profile == 'peaky'
    for i, (A, ch) in enumerate(zip(m['anchors']['anchors_per_point'], SSD_FMAP_CH)):
        n = 'ssd/MultiBox_%d' % i
        fan = 9 * ch
        wts[n + '_offsets_conv/w'] = _conv(rng, 3, 3, ch, 4 * A, std=0.1 / np.sqrt(fan))
        wts[n + '_offsets_conv/b'] = np.zeros(4 * A, np.float32)
        wts[n + '_classes_conv/w'] = _conv(rng, 3, 3, ch, (C + 1) * A,
                                           std=(0.7 if peaky else 0.25) / np.sqrt(fan))
        wts[n + '_classes_conv/b'] = np.zeros((C + 1) * A, np.float32)
    return wts


def make_weights(config, seed=0, profile='peaky'):
    t = config['model']['type']
    if t == 'fasterrcnn':
        return fasterrcnn_weights(config, seed, profile)
    if t == 'ssd':
        return ssd_weights(config, seed, profile)
    raise ValueError("Model type '{}' not supported".format(t))


def make_images(n, h, w, seed=0):
    """uint8 uniform [0,255] NHWC, like the reference's own tests
    (``fasterrcnn_test.py:141``)."""
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, size=(n, h, w, 3), dtype=np.uint8)
