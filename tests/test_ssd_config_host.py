"""SSD at sizes and anchor settings other than the default 300x300 (host side, no GPU): the engine's config check, which
runs before any device is touched, and the oracle's feature-map grids and anchor counts for every configuration that
tests/test_gpu_ssd_configs.py runs on the GPU."""
import numpy as np
import pytest

from luminoth_b200 import config as C, engine, synth
from oracle import anchors as oanchors
from oracle import vgg


def ssd_cfg(h, w, num_classes=20, anchors_per_point=None, **anchor_keys):
    cfg = C.default_config('ssd', ['dataset.image_preprocessing.fixed_height=%d' % h,
                                   'dataset.image_preprocessing.fixed_width=%d' % w,
                                   'model.network.num_classes=%d' % num_classes])
    # list-valued keys cannot be given as override strings (config.py rejects a str for a list key)
    if anchors_per_point is not None:
        cfg['model']['anchors']['anchors_per_point'] = list(anchors_per_point)
    for k, v in anchor_keys.items():
        cfg['model']['anchors'][k] = v
    return cfg


# (h, w, num_classes, anchors_per_point or None for the default, other anchor keys) -> the six feature-map grids and
# the total anchor count.  VALID 2x2 pools drop an odd row (301 -> 150 -> 75 -> 37), SAME stride-2 convs round up
# (37 -> 18 -> 9 -> 5), the two VALID 3x3 convs take 2 each.  272 is the smallest side whose last map is 1x1.
SSD_CASES = [
    ((512, 512, 20, None, {}), [(64, 64), (32, 32), (16, 16), (8, 8), (6, 6), (4, 4)], 24656),
    ((272, 272, 20, None, {}), [(34, 34), (17, 17), (9, 9), (5, 5), (3, 3), (1, 1)], 7034),
    ((301, 333, 20, None, {}), [(37, 41), (18, 20), (9, 10), (5, 5), (3, 3), (1, 1)], 8958),
    ((300, 500, 80, None, {}), [(37, 62), (18, 31), (9, 16), (5, 8), (3, 6), (1, 4)], 13716),
    ((300, 300, 20, [3, 5, 5, 5, 3, 3], {}), [(37, 37), (18, 18), (9, 9), (5, 5), (3, 3), (1, 1)], 6287),
    ((300, 300, 80, [6, 6, 6, 6, 6, 6], {'min_scale': 0.2, 'max_scale': 0.95}),
     [(37, 37), (18, 18), (9, 9), (5, 5), (3, 3), (1, 1)], 10854),
]


def _case_id(case):
    (h, w, nc, app, other), _, _ = case
    return '%dx%d-c%d%s%s' % (h, w, nc, '-a' + ''.join(map(str, app)) if app else '', '-scales' if other else '')


@pytest.mark.parametrize('case', SSD_CASES, ids=_case_id)
def test_oracle_feature_maps_and_anchor_count(case):
    (h, w, nc, app, other), shapes, total = case
    cfg = ssd_cfg(h, w, nc, app, **other)
    wts = synth.make_weights(cfg, seed=0)
    img = synth.make_images(1, h, w, seed=0).astype(np.float32)
    fmaps = vgg.ssd_feature_maps(img, wts)
    got = [tuple(fm.shape[1:3]) for fm in fmaps.values()]
    assert got == shapes
    a = cfg['model']['anchors']
    anchors = oanchors.ssd_anchors(got, a['min_scale'], a['max_scale'], a['ratios'], a['anchors_per_point'], [h, w, 3])
    assert anchors.shape == (total, 4)
    assert total == sum(fh * fw * k for (fh, fw), k in zip(shapes, a['anchors_per_point']))


@pytest.mark.parametrize('h,w', [(271, 271), (272, 271), (271, 272), (200, 300)])
def test_engine_refuses_an_ssd_input_too_small_for_its_last_map(h, w):
    """A side below 272 leaves the last feature map empty: ValueError from the config check, before any device."""
    with pytest.raises(ValueError, match='SSD input too small'):
        engine.Engine(ssd_cfg(h, w))


@pytest.mark.parametrize('h,w', [(272, 272), (301, 333), (512, 512)])
def test_engine_accepts_ssd_sizes_with_a_last_map(h, w):
    """The config check passes: without a GPU the engine then stops at the device, not at the config."""
    try:
        eng = engine.Engine(ssd_cfg(h, w))
    except RuntimeError as e:
        assert 'too small' not in str(e)
    else:
        eng.close()


def test_engine_refuses_ratios_shorter_than_anchors_per_point():
    """anchors_per_point A needs A - 1 ratios (ssd/utils.py takes ratios[:A - 1])."""
    with pytest.raises(ValueError, match='ratios too short'):
        engine.Engine(ssd_cfg(300, 300, ratios=[1, 0.5, 2, 0.333]))           # default A = 6 needs 5
    with pytest.raises(ValueError, match='ratios too short'):
        engine.Engine(ssd_cfg(300, 300, anchors_per_point=[4, 4, 4, 4, 4, 7]))


@pytest.mark.parametrize('app', [[4, 6, 6, 6, 4], [4, 6, 6, 6, 4, 4, 4], []])
def test_engine_refuses_anchors_per_point_without_six_entries(app):
    with pytest.raises(ValueError, match='must have 6 entries'):
        engine.Engine(ssd_cfg(300, 300, anchors_per_point=app))
