"""Faster R-CNN's model.base_network.output_stride on the ResNet base networks (host side, no GPU): the oracle trunk's
block3 grid at every stride, and the engine's config check, which runs before any device is touched."""
import numpy as np
import pytest

import resnet_v2_oracle as V2
from luminoth_b200 import config as C, engine, synth


def _cfg(arch, output_stride):
    return C.default_config('fasterrcnn', ['model.base_network.architecture=' + arch,
                                           'model.base_network.output_stride=%s' % output_stride])


@pytest.mark.parametrize('arch,output_stride', [(a, s) for a in ('resnet_v1_50', 'resnet_v2_50') for s in (4, 8, 16, 32)]
                         + [('resnet_v1_101', 8)])
def test_trunk_grid_follows_output_stride(arch, output_stride):
    """A 128x128 image gives a (128 / output_stride)^2 block3 map of 1024 channels."""
    wts = synth.make_weights(_cfg(arch, output_stride), seed=0)
    img = synth.make_images(1, 128, 128, seed=0).astype(np.float32)
    fmap = V2.trunk(img, wts, arch, output_stride=output_stride)
    side = 128 // output_stride
    assert fmap.shape == (1, side, side, 1024)
    assert np.isfinite(fmap).all()


@pytest.mark.parametrize('output_stride', [4, 8, 32])
def test_trunk_grid_of_an_odd_size_is_the_ceiling(output_stride):
    wts = synth.make_weights(_cfg('resnet_v1_50', output_stride), seed=0)
    img = synth.make_images(1, 129, 159, seed=0).astype(np.float32)
    fmap = V2.trunk(img, wts, 'resnet_v1_50', output_stride=output_stride)
    assert fmap.shape == (1, -(-129 // output_stride), -(-159 // output_stride), 1024)


@pytest.mark.parametrize('output_stride,match', [(6, 'needs to be a multiple of 4'), (2, 'needs to be a multiple of 4'),
                                                 (12, 'cannot be reached'), (64, 'cannot be reached'),
                                                 (24, 'cannot be reached')])
def test_engine_rejects_unreachable_output_strides(output_stride, match):
    """slim's resnet_v1 / stack_blocks_dense messages, as ValueError, from the config check before any device."""
    with pytest.raises(ValueError, match=match):
        engine.Engine(_cfg('resnet_v1_50', output_stride))


@pytest.mark.parametrize('output_stride', [4, 8, 16, 32, 'None'])
def test_engine_accepts_the_reachable_output_strides(output_stride):
    """4, 8, 16, 32 and null pass the config check: without a GPU the engine then stops at the device, not at the
    config."""
    cfg = _cfg('resnet_v2_50', output_stride)
    if output_stride == 'None':
        assert cfg['model']['base_network']['output_stride'] is None
    try:
        eng = engine.Engine(cfg)
    except RuntimeError as e:
        assert 'output_stride' not in str(e)
    else:
        eng.close()
