"""Faster R-CNN's model.base_network.endpoint on the ResNet base networks (host side, no GPU): the oracle trunk's grid
and depth at every endpoint slim collects, the engine's config check, which runs before any device is touched, and the
synthetic weights drawn through the endpoint."""
import re

import numpy as np
import pytest

import endpoint_oracle as EO
import resnet_v2_oracle as V2
from luminoth_b200 import config as C, engine, synth


def _cfg(arch, endpoint, *extra):
    return C.default_config('fasterrcnn', ['model.base_network.architecture=' + arch,
                                           'model.base_network.endpoint=' + endpoint] + list(extra))


def _kind(arch):
    return 'bottleneck_v2' if arch.startswith('resnet_v2') else 'bottleneck_v1'


# endpoint (``{u}`` the arch's unit kind) -> (feature stride at output_stride 8, 16, 32; depth).  conv1 is at stride 2,
# pool1 at 4; each block's last unit doubles the stride in its conv2 and its shortcut until the output_stride is
# reached.  block2 has four units in both ResNet-50s, so unit_4 is the one that strides.
TABLE = {
    'conv1': ((2, 2, 2), 64),
    'block1': ((8, 8, 8), 256),
    'block2': ((8, 16, 16), 512),
    'block3': ((8, 16, 32), 1024),
    'block4': ((8, 16, 32), 2048),
    'block2/unit_1/{u}': ((8, 8, 8), 512),
    'block2/unit_1/{u}/conv1': ((8, 8, 8), 128),
    'block2/unit_1/{u}/conv2': ((8, 8, 8), 128),
    'block2/unit_1/{u}/conv3': ((8, 8, 8), 512),
    'block2/unit_1/{u}/shortcut': ((8, 8, 8), 512),
    'block2/unit_4/{u}/conv1': ((8, 8, 8), 128),
    'block2/unit_4/{u}/conv2': ((8, 16, 16), 128),
    'block2/unit_4/{u}': ((8, 16, 16), 512),
    'block3/unit_1/{u}/shortcut': ((8, 16, 16), 1024),
}
OUTPUT_STRIDES = (8, 16, 32)


@pytest.mark.parametrize('output_stride', OUTPUT_STRIDES)
@pytest.mark.parametrize('arch', ['resnet_v1_50', 'resnet_v2_50'])
def test_trunk_grid_and_depth_follow_the_endpoint(arch, output_stride):
    """A 320x320 image gives a ceil(320 / stride)^2 map of the endpoint's depth; the trunk stopped at an endpoint
    returns what the whole network collects under that name."""
    wts = synth.make_weights(_cfg(arch, 'block4'), seed=0)
    img = synth.make_images(1, 320, 320, seed=0).astype(np.float32)
    collected = {}
    EO.trunk(img, wts, arch, 'block4', output_stride, collect=collected)
    for name, (strides, depth) in TABLE.items():
        ep = name.format(u=_kind(arch))
        side = -(-320 // strides[OUTPUT_STRIDES.index(output_stride)])
        assert collected[ep].shape == (1, side, side, depth), ep
        assert np.isfinite(collected[ep]).all()
    for ep in ('conv1', 'block2', 'block2/unit_4/{u}/conv1', 'block2/unit_1/{u}/shortcut', 'block2/unit_1/{u}/conv3'):
        ep = ep.format(u=_kind(arch))
        np.testing.assert_array_equal(EO.trunk(img, wts, arch, ep, output_stride), collected[ep])


@pytest.mark.parametrize('arch', ['resnet_v1_50', 'resnet_v2_50'])
def test_trunk_default_endpoint_is_the_block3_oracle(arch):
    wts = synth.make_weights(_cfg(arch, 'block3'), seed=0)
    img = synth.make_images(1, 96, 128, seed=0).astype(np.float32)
    np.testing.assert_array_equal(EO.trunk(img, wts, arch), V2.trunk(img, wts, arch))


@pytest.mark.parametrize('output_stride', OUTPUT_STRIDES)
def test_trunk_grid_of_an_odd_size_is_the_ceiling(output_stride):
    arch = 'resnet_v1_50'
    wts = synth.make_weights(_cfg(arch, 'block4'), seed=0)
    img = synth.make_images(1, 129, 159, seed=0).astype(np.float32)
    collected = {}
    EO.trunk(img, wts, arch, 'block4', output_stride, collect=collected)
    for name, (strides, depth) in TABLE.items():
        ep = name.format(u=_kind(arch))
        s = strides[OUTPUT_STRIDES.index(output_stride)]
        assert collected[ep].shape == (1, -(-129 // s), -(-159 // s), depth), ep


def _invalid(arch, endpoint):
    return '^' + re.escape('"truncated_base_network/%s/%s" is an invalid value of endpoint for this architecture.'
                           % (arch, endpoint)) + '$'


# outputs slim does not collect (pool1, preact, postnorm, global_pool), units past a block's count, the other
# ResNet version's unit kind, a shortcut of an identity-shortcut unit, VGG names and malformed names
INVALID = [('resnet_v1_50', 'pool1'), ('resnet_v1_50', 'global_pool'), ('resnet_v1_50', 'block1/unit_4/bottleneck_v1'),
           ('resnet_v1_50', 'block3/unit_7/bottleneck_v1/conv1'), ('resnet_v1_50', 'block1/unit_1/bottleneck_v2'),
           ('resnet_v1_50', 'block1/unit_2/bottleneck_v1/shortcut'), ('resnet_v1_50', 'conv5/conv5_3'),
           ('resnet_v1_50', 'vgg_16/conv5/conv5_3'), ('resnet_v1_50', 'block5'), ('resnet_v1_50', 'block0'),
           ('resnet_v1_50', 'block3/unit_01/bottleneck_v1'), ('resnet_v1_50', 'block2/unit_1/bottleneck_v1/conv4'),
           ('resnet_v1_101', 'block3/unit_24/bottleneck_v1'), ('resnet_v2_50', 'block1/unit_1/bottleneck_v2/preact'),
           ('resnet_v2_50', 'postnorm'), ('resnet_v2_50', 'pool1'), ('resnet_v2_50', 'block2/unit_1/bottleneck_v1'),
           ('resnet_v2_50', 'block4/unit_3/bottleneck_v2/shortcut')]


@pytest.mark.parametrize('arch,endpoint', INVALID, ids=['%s-%s' % c for c in INVALID])
def test_engine_rejects_endpoints_slim_does_not_collect(arch, endpoint):
    """The reference's ValueError, from the engine's config check before any device, from the synthetic weights and
    from the oracle."""
    with pytest.raises(ValueError, match=_invalid(arch, endpoint)):
        engine.Engine(_cfg(arch, endpoint))
    with pytest.raises(ValueError, match=_invalid(arch, endpoint)):
        synth.parse_endpoint(arch, endpoint)
    if arch == 'resnet_v1_50':
        wts = synth.make_weights(_cfg(arch, 'block4'), seed=0)
        with pytest.raises(ValueError, match=_invalid(arch, endpoint)):
            EO.trunk(synth.make_images(1, 32, 32).astype(np.float32), wts, arch, endpoint)


@pytest.mark.parametrize('endpoint', ['block4', 'block2', 'conv1', 'block4/unit_1/bottleneck_v1/conv2'])
def test_engine_rejects_a_resnet_v1_101_tail_behind_other_depths(endpoint):
    """resnet_v1_101's tail reuses block4's variables, whose first unit reads 1024 channels."""
    with pytest.raises(ValueError, match='resnet_v1_101 tail needs a 1024-channel endpoint'):
        engine.Engine(_cfg('resnet_v1_101', endpoint))


def _passes_config_check(cfg):
    """Without a GPU the engine stops at the device once the config check passes."""
    try:
        eng = engine.Engine(cfg)
    except RuntimeError as e:
        assert 'endpoint' not in str(e)
    else:
        eng.close()


@pytest.mark.parametrize('extra', [['model.base_network.use_tail=false'], ['model.network.with_rcnn=false']])
@pytest.mark.parametrize('endpoint', ['block4', 'block2'])
def test_engine_accepts_resnet_v1_101_endpoints_without_the_tail(endpoint, extra):
    _passes_config_check(_cfg('resnet_v1_101', endpoint, *extra))


@pytest.mark.parametrize('arch,endpoint', [('resnet_v1_50', e.format(u='bottleneck_v1')) for e in TABLE]
                         + [('resnet_v2_50', e.format(u='bottleneck_v2')) for e in TABLE]
                         + [('resnet_v1_101', 'block3/unit_12/bottleneck_v1'), ('resnet_v1_101', 'block3'),
                            ('resnet_v2_152', 'block2/unit_8/bottleneck_v2/conv2'), ('resnet_v1_50', '')])
def test_engine_accepts_collected_endpoints(arch, endpoint):
    _passes_config_check(_cfg(arch, endpoint))


class _Reads(dict):
    """A weight dict that records the names read from it."""
    def __init__(self, *a):
        super().__init__(*a)
        self.read = set()

    def __getitem__(self, k):
        self.read.add(k)
        return super().__getitem__(k)


# (arch, endpoint, extra overrides): the GPU suite's endpoint configurations
SYNTH = [('resnet_v1_50', 'block4', ()), ('resnet_v1_50', 'block2', ()), ('resnet_v1_50', 'block1', ()),
         ('resnet_v1_50', 'conv1', ()), ('resnet_v1_50', 'block3/unit_4/bottleneck_v1/conv3', ()),
         ('resnet_v1_50', 'block2/unit_4/bottleneck_v1/conv1', ()),
         ('resnet_v1_50', 'block2/unit_1/bottleneck_v1/shortcut', ()),
         ('resnet_v1_50', 'block2', ('model.network.with_rcnn=false',)),
         ('resnet_v1_50', 'block4', ('model.rcnn.use_mean=false',)),
         ('resnet_v1_101', 'block3/unit_12/bottleneck_v1', ()),
         ('resnet_v1_101', 'block4', ('model.base_network.use_tail=false',)),
         ('resnet_v2_50', 'block4', ()), ('resnet_v2_50', 'block2/unit_2/bottleneck_v2/conv3', ()),
         ('resnet_v2_50', 'conv1', ()), ('resnet_v2_50', 'block3/unit_1/bottleneck_v2/shortcut', ())]


@pytest.mark.parametrize('arch,endpoint,extra', SYNTH, ids=['-'.join((a, e) + x) for a, e, x in SYNTH])
def test_synthetic_weights_are_what_the_forward_reads(arch, endpoint, extra):
    """No trunk variable past the endpoint except the tail's block4, and every one the oracle forward reads."""
    cfg = _cfg(arch, endpoint, 'model.network.num_classes=3', 'model.rpn.proposals.post_nms_top_n=20', *extra)
    wts = _Reads(synth.make_weights(cfg, seed=1))
    out = EO.fasterrcnn_forward(synth.make_images(1, 64, 96, seed=2)[0], wts, cfg.to_dict())
    depth = synth.parse_endpoint(arch, endpoint)[3]
    assert out['conv_feature_map'].shape[-1] == depth
    if cfg['model']['network']['with_rcnn']:
        assert wts.read == set(wts)
    else:
        assert wts.read == {k for k in wts if not k.startswith('fasterrcnn/rcnn/')}
    tail = arch == 'resnet_v1_101' and cfg['model']['base_network']['use_tail']
    assert any('/block4/' in k for k in wts) == (tail or endpoint.startswith('block4'))


@pytest.mark.parametrize('arch', ['resnet_v1_50', 'resnet_v2_50', 'resnet_v1_101'])
def test_block4_draws_leave_the_block3_stream_alone(arch):
    """The trunk of a block4 configuration is the block3 configuration's plus block4: the extra variables come from
    a generator of their own."""
    base = synth.make_weights(_cfg(arch, 'block3'), seed=3)
    deep = synth.make_weights(_cfg(arch, 'block4', 'model.base_network.use_tail=false'), seed=3)
    for k, v in base.items():
        if k.startswith('truncated_base_network/'):
            np.testing.assert_array_equal(deep[k], v)
    np.testing.assert_array_equal(synth.make_weights(_cfg(arch, 'None'), seed=3)['fasterrcnn/rpn/conv/w'],
                                  base['fasterrcnn/rpn/conv/w'])
