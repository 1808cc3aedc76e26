"""CPU-only checks: the C-ABI library loads and exports every symbol the header
declares, fails loudly without a GPU, and the YAML config surface behaves like
luminoth/utils/config.py."""
import os
import re

import numpy as np
import pytest

from luminoth_b200 import config as C

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _built_lib():
    import __graft_entry__ as g
    g.build()
    from luminoth_b200 import engine
    return engine.load_library(), engine


def test_library_exports_every_declared_symbol():
    lib, engine = _built_lib()
    hdr = open(os.path.join(ROOT, 'include', 'luminoth_b200.h')).read()
    declared = set(re.findall(r'\b(lumi_[a-z0-9_]+)\s*\(', hdr))
    assert declared, 'no declarations parsed'
    assert declared == set(engine.SIGNATURES), declared ^ set(engine.SIGNATURES)
    for name in declared:
        assert hasattr(lib, name)
    assert lib.lumi_version().startswith(b'luminoth_b200')


def test_library_is_hopper_native_sass():
    """The built library carries the sm_90a instructions the design claims (DESIGN 4.1) and no legacy tensor path:
    wgmma (HGMMA, both tile widths of the conv kernel), TMA tensor loads, mbarrier transaction counts."""
    import shutil
    import subprocess
    from luminoth_b200 import build as B
    exe = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(exe) or not os.path.exists(B.LIB):
        pytest.skip('cuobjdump or the built library is not available')
    sass = subprocess.run([exe, '-sass', B.LIB], capture_output=True, text=True).stdout
    assert 'sm_90a' in sass and 'sm_100' not in sass
    for mnemonic in ('HGMMA.64x128x16.F32', 'HGMMA.64x64x16.F32', 'UTMALDG.4D', 'UTMALDG.2D', 'SYNCS.ARRIVE.TRANS'):
        assert mnemonic in sass, mnemonic
    assert not re.search(r'\bHMMA\b', sass), 'legacy (mma.sync) tensor-core instructions in the library'


def test_engine_has_no_cpu_fallback():
    lib, engine = _built_lib()
    if lib.lumi_device_count() > 0:
        pytest.skip('GPU present')
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        engine.Engine(C.default_config('fasterrcnn'))


def test_engine_rejects_bad_configs_like_the_reference():
    _, engine = _built_lib()
    cfg = C.default_config('fasterrcnn')
    cfg.model.type = 'yolo'                                   # models/models.py:13-17 ValueError
    with pytest.raises(ValueError, match='not a valid model_type'):
        engine.Engine(cfg)
    cfg = C.default_config('fasterrcnn', ['model.rcnn.roi.pooling_mode=roi_pooling'])   # roi_pool.py:97-102
    with pytest.raises(ValueError, match='not implemented'):
        engine.Engine(cfg)
    cfg = C.default_config('fasterrcnn', ['model.anchors.base_size=1'])                 # utils/anchors.py:45-50
    cfg.model.anchors.scales = [0.5]; cfg.model.anchors.ratios = [0.5]
    with pytest.raises(ValueError, match='too small'):
        engine.Engine(cfg)
    cfg = C.default_config('ssd', ['model.base_network.architecture=vgg_16'])           # feature_extractor.py:19-23
    with pytest.raises(ValueError, match='Invalid architecture'):
        engine.Engine(cfg)


# ---------------------------------------------------------------- config surface (utils/config.py)
def test_parse_override_and_values():
    """utils/config.py:151-196"""
    d = C.parse_override(['a.b.c=1', 'a.b.d=2.5', 'x=true', 'y=None', 'z=hello', 'w=False'])
    assert d == {'a': {'b': {'c': 1, 'd': 2.5}}, 'x': True, 'y': None, 'z': 'hello', 'w': False}
    with pytest.raises(ValueError):
        C.parse_override(['a=b=c'])
    assert C.parse_override(None) == {}


def test_merge_into_type_check_and_replace():
    """utils/config.py:73-148"""
    base = C.Config({'a': 1, 'b': {'c': 2, 'd': 3}, 'e': None, 'opt': {'_replace': True, 'type': 'momentum', 'momentum': 0.9}})
    new = C.Config({'b': {'c': 5}, 'e': 'now-set', 'opt': {'type': 'adam'}})
    out = C.merge_into(new, base, overwrite=True)
    assert out.b.c == 5 and out.b.d == 3 and out.e == 'now-set'
    assert dict(out.opt) == {'type': 'adam'}                  # replaced wholesale (base had _replace)
    with pytest.raises(ValueError, match='Incorrect type'):
        C.merge_into(C.Config({'a': 'string'}), C.Config({'a': 1}), overwrite=True)
    out = C.merge_into(C.Config({'a': 7}), C.Config({'a': 1}), overwrite=False)
    assert out.a == 1                                         # no overwrite -> base wins


def test_get_config_from_yaml(tmp_path):
    p = tmp_path / 'c.yml'
    p.write_text('model:\n  type: fasterrcnn\n  network:\n    num_classes: 80\n  base_network:\n    architecture: resnet_v1_50\n')
    cfg = C.get_config([str(p)], ['model.rcnn.proposals.total_max_detections=100'])
    assert cfg.model.network.num_classes == 80
    assert cfg.model.base_network.architecture == 'resnet_v1_50'
    assert cfg.model.rcnn.proposals.total_max_detections == 100
    assert cfg.model.rpn.proposals.pre_nms_top_n == 12000      # base default survives
    assert cfg.dataset.image_preprocessing.min_size == 600
    p.write_text('model:\n  type: nope\n')
    with pytest.raises(ValueError):
        C.get_config([str(p)])


def test_default_configs_match_reference_defaults():
    f = C.default_config('fasterrcnn')
    assert f.model.anchors.scales == [0.25, 0.5, 1, 2] and f.model.anchors.ratios == [0.5, 1, 2]
    assert f.model.rpn.proposals.nms_threshold == 0.7 and f.model.rpn.proposals.post_nms_top_n == 2000
    assert f.model.rcnn.proposals.class_nms_threshold == 0.5 and f.model.rcnn.proposals.min_prob_threshold == 0.5
    assert f.model.rcnn.target_normalization_variances == [0.1, 0.2]
    s = C.default_config('ssd')
    assert s.model.anchors.anchors_per_point == [4, 6, 6, 6, 4, 4]
    assert s.model.proposals.class_nms_threshold == 0.45 and s.model.variances == [0.1, 0.2]


def test_format_predictions_matches_oracle_finalize():
    """utils/predicting.py:114-148 restated twice (wrapper + oracle) must agree, incl. banker's rounding."""
    from luminoth_b200.predicting import format_predictions, preprocess_image
    from oracle.predict import finalize_predictions, preprocess
    rng = np.random.default_rng(0)
    obj = rng.uniform(0, 1000, (50, 4)).astype(np.float32)
    obj[0] = [0.5, 1.5, 2.5, 3.5]
    lab = rng.integers(0, 20, 50).astype(np.int32)
    pr = rng.uniform(0, 1, 50).astype(np.float32)
    for sf in (np.float32(1.0), np.float32(0.625), (np.float32(0.3), np.float32(0.46875))):
        assert format_predictions(obj, lab, pr, sf) == finalize_predictions(obj, lab, pr, sf)
    names = ['c%d' % i for i in range(20)]
    assert format_predictions(obj, lab, pr, np.float32(1.0), names)[0]['label'].startswith('c')
    img = rng.integers(0, 256, (120, 200, 3)).astype(np.uint8)
    for cfg in (C.default_config('fasterrcnn'), C.default_config('ssd')):
        a, sa = preprocess_image(img, cfg); b, sb = preprocess(img, cfg)
        np.testing.assert_array_equal(a, b)
        assert np.all(np.asarray(sa) == np.asarray(sb))


def test_target_size_matches_oracle_preprocess_shapes():
    """utils/image.py:38-114 / :117-147: the product wrapper's float32 size arithmetic (used to drive the GPU
    resize) agrees with the oracle's preprocess on the resulting shape and scale factor."""
    from luminoth_b200 import default_config
    from luminoth_b200.predicting import target_size, preprocess_image
    from oracle import predict as opredict
    rng = np.random.default_rng(0)
    for cfg in (default_config('fasterrcnn'), default_config('ssd')):
        for _ in range(40):
            h, w = int(rng.integers(40, 2200)), int(rng.integers(40, 2200))
            img = np.zeros((h, w, 3), np.uint8)
            ref_img, ref_scale = opredict.preprocess(img, cfg)
            nh, nw, scale = target_size(img.shape, cfg)
            assert (nh, nw) == ref_img.shape[:2]
            assert np.all(np.asarray(scale, np.float32) == np.asarray(ref_scale, np.float32))
    img = rng.integers(0, 256, (333, 517, 3)).astype(np.uint8)
    got, _ = preprocess_image(img, default_config('fasterrcnn'))
    ref, _ = opredict.preprocess(img, default_config('fasterrcnn'))
    np.testing.assert_array_equal(got, ref)


def test_prediction_filters_follow_the_reference_callers():
    """predict.py:246-259 / tasks.py:64-67 / web.py:97-100 (quirk Q10): where min_prob and max_detections land."""
    from luminoth_b200 import default_config, set_prediction_filters
    c = set_prediction_filters(default_config('fasterrcnn'), min_prob=0.5, max_detections=100)
    assert c.model.rcnn.proposals.total_max_detections == 100 and c.model.rcnn.proposals.min_prob_threshold == 0.5
    assert c.model.rpn.proposals.post_nms_top_n == 2000
    c = set_prediction_filters(default_config('fasterrcnn', ['model.network.with_rcnn=False']), 0.5, 100)
    assert c.model.rpn.proposals.post_nms_top_n == 100 and c.model.rcnn.proposals.total_max_detections == 300
    c = set_prediction_filters(default_config('ssd'), min_prob=0.01)
    assert c.model.proposals.min_prob_threshold == 0.01 and c.model.proposals.total_max_detections == 100
    c = default_config('ssd')
    c.model.type = 'yolo'
    with pytest.raises(ValueError, match='not supported'):
        set_prediction_filters(c, 0.5, 10)
