"""Base networks for Faster R-CNN beyond resnet_v1_{50,101}: resnet_v1_152 and the pre-activation
resnet_v2_{50,101,152} (host side, no GPU)."""
import numpy as np
import pytest

import resnet_v2_oracle as V2
from luminoth_b200 import config as C, engine, synth

ARCHS = ['resnet_v1_50', 'resnet_v1_101', 'resnet_v1_152', 'resnet_v2_50', 'resnet_v2_101', 'resnet_v2_152']


@pytest.mark.parametrize('arch', ARCHS)
def test_trunk_output_shape(arch):
    """truncated_base_network_test.py:22-34: a 320x320 image gives the (1, 20, 20, 1024) block3 map."""
    cfg = C.default_config('fasterrcnn', ['model.base_network.architecture=' + arch])
    wts = synth.make_weights(cfg, seed=0)
    img = synth.make_images(1, 320, 320, seed=0).astype(np.float32)
    fmap = V2.trunk(img, wts, arch)
    assert fmap.shape == (1, 20, 20, 1024)
    assert np.isfinite(fmap).all()


def test_resnet_v2_synthetic_weights_have_no_block4_or_postnorm():
    cfg = C.default_config('fasterrcnn', ['model.base_network.architecture=resnet_v2_50'])
    names = synth.make_weights(cfg, seed=0)
    root = 'truncated_base_network/resnet_v2_50/'
    assert not [n for n in names if n.startswith(root + 'block4') or n.startswith(root + 'postnorm')]
    assert root + 'block1/unit_1/bottleneck_v2/preact/gamma' in names
    assert root + 'block1/unit_1/bottleneck_v2/shortcut/biases' in names
    assert root + 'block1/unit_2/bottleneck_v2/shortcut/weights' not in names


def test_resnet_v2_unit_matches_its_definition():
    """bottleneck_v2: the identity shortcut is subsample(x), not of preact, and the output is the raw sum."""
    rng = np.random.default_rng(0)
    s = 'u/bottleneck_v2'
    wts = {s + '/preact/gamma': np.full(8, 2.0), s + '/preact/beta': np.full(8, -1.0),
           s + '/preact/moving_mean': np.zeros(8), s + '/preact/moving_variance': np.full(8, 1.0 - 1e-5)}
    for c, (k, ci, co) in {'conv1': (1, 8, 4), 'conv2': (3, 4, 4)}.items():
        wts['%s/%s/weights' % (s, c)] = np.zeros((k, k, ci, co))
        for v, val in (('gamma', 1.0), ('beta', 0.0), ('moving_mean', 0.0), ('moving_variance', 1.0)):
            wts['%s/%s/BatchNorm/%s' % (s, c, v)] = np.full(co, val)
    wts[s + '/conv3/weights'] = np.zeros((1, 1, 4, 8))
    wts[s + '/conv3/biases'] = np.arange(8.0)
    x = rng.standard_normal((1, 6, 6, 8))
    y = V2.bottleneck_v2(x, wts, 'u', 8, 2)
    np.testing.assert_allclose(y, x[:, ::2, ::2, :] + np.arange(8.0), rtol=0, atol=1e-12)


@pytest.mark.parametrize('model,arch,match', [('fasterrcnn', 'vgg_16', 'resnet_v2_152'),
                                              ('ssd', 'vgg_16', 'Invalid architecture')])
def test_engine_still_rejects_vgg_16(model, arch, match):
    cfg = C.default_config(model, ['model.base_network.architecture=' + arch])
    with pytest.raises(ValueError, match=match):
        engine.Engine(cfg)


def test_preact_abi_symbols_are_exported():
    lib = engine.load_library()
    for name in ('lumi_op_conv2d_preact', 'lumi_op_max_pool_preact'):
        assert hasattr(lib, name)
