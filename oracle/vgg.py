"""``truncated_vgg_16`` + SSD extra feature layers (oracle only).

``luminoth/models/base/truncated_vgg.py:60-121`` (3x3 SAME conv + bias + relu,
2x2/2 max pools with slim's default VALID padding -> 300,150,75,37,18) and
``luminoth/models/ssd/feature_extractor.py:27-132`` (conv4_3 L2-norm x gamma,
pool5 3x3/1 SAME, conv6 rate 6 ... conv11_2, relu after each).  No mean
subtraction: ``truncated_vgg_16`` does not start with ``vgg``
(``base_network.py:104-105,153-157``, quirk Q7).
"""
from collections import OrderedDict

from . import tf_ops as T

VGG_CFG = [('conv1', 2, 64), ('conv2', 2, 128), ('conv3', 3, 256),
           ('conv4', 3, 512), ('conv5', 3, 512)]


def ssd_feature_maps(images, wts, scope='ssd/ssd_feature_extractor'):
    """images (N,H,W,3) raw 0..255, any fixed size -> OrderedDict of the 6 feature maps."""
    v = scope + '/vgg_16'
    x = images
    conv4_3 = None
    for bi, (name, reps, _) in enumerate(VGG_CFG):
        for r in range(reps):
            p = '%s/%s/%s_%d' % (v, name, name, r + 1)
            x = T.relu(T.conv2d(x, wts[p + '/weights'], 1, 'SAME', bias=wts[p + '/biases']))
        if name == 'conv4':
            conv4_3 = x
        if bi < 4:
            x = T.max_pool(x, 2, 2, 'VALID')
    fmaps = OrderedDict()
    norm = T.l2_normalize(conv4_3, 3, 1e-12)
    fmaps['conv4_3_norm'] = (norm * wts[scope + '/conv_4_3_norm/gamma'].reshape(1, 1, 1, -1).astype(images.dtype)
                             ).astype(images.dtype)
    e = scope + '/extra_feature_layers'

    def sconv(x, name, stride=1, rate=1, padding='SAME'):
        return T.relu(T.conv2d(x, wts['%s/%s/w' % (e, name)], stride, padding, rate,
                               bias=wts['%s/%s/b' % (e, name)]))
    x = T.max_pool(x, 3, 1, 'SAME')
    x = sconv(x, 'conv6', rate=6)
    x = sconv(x, 'conv7'); fmaps['conv7'] = x
    x = sconv(x, 'conv8_1'); x = sconv(x, 'conv8_2', stride=2); fmaps['conv8_2'] = x
    x = sconv(x, 'conv9_1'); x = sconv(x, 'conv9_2', stride=2); fmaps['conv9_2'] = x
    x = sconv(x, 'conv10_1'); x = sconv(x, 'conv10_2', padding='VALID'); fmaps['conv10_2'] = x
    x = sconv(x, 'conv11_1'); x = sconv(x, 'conv11_2', padding='VALID'); fmaps['conv11_2'] = x
    return fmaps
