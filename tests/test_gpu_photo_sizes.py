"""Faster R-CNN at the sizes photos are predicted at (`-m gpu`, except the host checks).

With the default preprocessing (min_size 600, max_size 1024) common photo shapes map to targets such as 600x800,
899x600, 600x899 and 576x1024, where the conv layers run on other tiles than at 600x1024: partial last tile rows and
columns, many waves of them, the auto stream-K split and the pipelined half-batch's reserved SMs all meet there.

* Launches: every R50 trunk and RPN conv at four photo targets and at the canvas of a packed photo mix, batch 4 as
  the engine runs it, plus resnet_v2_50 and output stride 8 at 600x899, against float64 at sampled pixels with the
  rule of test_gpu_conv_engine_layers (rows already in its table are left out).
* End to end: predict_resize on batches of 4 photo-sized sources, production config and path (R50, 80 classes,
  2000 proposals, bench's weights; pipeline, default stream-K, graph replay), images of both pipeline halves against
  the fp32 and float64 oracle fed the source resized on the host, with the rule of test_gpu_baseline_configs.  One
  R101 case with config 4's overrides.
* Packed: a mix of four photo targets on an 800x899 canvas equals the single-image calls byte for byte with stream-K
  off, and meets the oracle with the default stream-K.

The parity numbers are written next to the baseline configs' (parity_report_baseline.json in the output directory);
run with -s for each launch's largest err / bound.
"""
import zlib

import numpy as np
import pytest

from luminoth_b200 import default_config, synth
from luminoth_b200.predicting import target_size
from test_gpu_baseline_configs import _assert_parity, _det_compare, _report
from test_gpu_conv_engine_layers import (ENGINE, ENGINE_F32, ENGINE_F32_RESERVE, ENGINE_RESERVE, LAYERS, Launch,
                                         _dedupe, _gather, _inputs, check, frcnn_heads, out_geometry, reference,
                                         resnet_rows, sample_pixels)
from test_gpu_conv_numerics import preact_reference
from test_gpu_e2e import rel_err
from test_gpu_packed_sizes import assert_crops, singles
from test_gpu_resize_input import assert_same, sources

PREPROCESSING = default_config('fasterrcnn', [])          # min_size 600, max_size 1024
PHOTOS = [(480, 640), (640, 480), (427, 640), (640, 427), (1080, 1920), (1920, 1080), (500, 500), (333, 500)]


def target(src):
    return target_size(tuple(src) + (3,), PREPROCESSING)[:2]


# the launch table's targets: landscape and portrait 3:4, 2:3 (640 x 600 / 427 truncates to 899 wide), 9:16 portrait
LAUNCH_SOURCES = [(480, 640), (640, 480), (427, 640), (1920, 1080)]
# the packed mix: 600x800, 800x600, 600x899 and 600x600 on an 800x899 canvas
PACK_SOURCES = [(480, 640), (640, 480), (427, 640), (500, 500)]
PACK_TARGETS = [target(s) for s in PACK_SOURCES]
CANVAS = (max(h for h, _ in PACK_TARGETS), max(w for _, w in PACK_TARGETS))
STRIDE = 16


def _tag(prefix, hw):
    return '%s_%dx%d' % (prefix, hw[0], hw[1])


def _photo_layers():
    rows = []
    for hw in [target(s) for s in LAUNCH_SOURCES] + [CANVAS]:
        trunk, fhw = resnet_rows(_tag('r50', hw), 4, *hw)
        rows += trunk + frcnn_heads(_tag('r50', hw), 4, fhw, 1024)
    hw = target((427, 640))
    rows += resnet_rows(_tag('r50_v2', hw), 4, *hw, v2=True)[0]
    _, hw8 = resnet_rows(_tag('r50_os8', hw), 4, *hw, output_stride=8, blocks=(0, 1))
    rows += resnet_rows(_tag('r50_os8', hw), 4, *hw, output_stride=8, blocks=(2,), hw=hw8)[0]
    known = {r[1:] for r in LAYERS}
    return [r for r in _dedupe(rows) if r[1:] not in known]


PHOTO_LAYERS = _photo_layers()


# ---------------------------------------------------------------------------------------------- host checks
def test_photo_targets():
    """The targets the default preprocessing derives for the photo shapes, and the packed mix's canvas."""
    assert [target(s) for s in PHOTOS] == [(600, 800), (800, 600), (600, 899), (899, 600), (576, 1024), (1024, 576),
                                          (600, 600), (600, 900)]
    assert PACK_TARGETS == [(600, 800), (800, 600), (600, 899), (600, 600)] and CANVAS == (800, 899)


def test_photo_layer_table_geometry():
    """Every target has rows of block1, block2, block3 and the RPN conv, one of them with an output width that is not
    a multiple of 8; spot checks of the derived maps; no row repeats a launch of the 600x1024 table."""
    names = [r.name for r in PHOTO_LAYERS]
    for hw in [target(s) for s in LAUNCH_SOURCES] + [CANVAS]:
        tag = _tag('r50', hw)
        for part in ('/block1/', '/block2/', '/block3/', '/rpn/conv'):
            assert any(n.startswith(tag + part) for n in names), (tag, part)
        widths = [out_geometry(r.h, r.w, r.k, r.stride, r.rate, r.padding)[1] for r in PHOTO_LAYERS
                  if r.name.startswith(tag + '/')]
        assert any(wo % 8 for wo in widths), (tag, sorted(set(widths)))
    by = {r.name: r for r in PHOTO_LAYERS}
    hw_of = lambda name: (by[name].h, by[name].w)
    assert hw_of('r50_600x800/block3/unit_1/conv1') == (38, 50)
    assert hw_of('r50_800x600/block3/unit_1/conv1') == (50, 38)
    assert hw_of('r50_600x899/block2/unit_1/conv1') == (75, 113)
    assert hw_of('r50_600x899/rpn/conv') == (38, 57)
    assert hw_of('r50_1024x576/rpn/conv') == (64, 36)
    assert hw_of('r50_800x899/rpn/conv') == (50, 57)
    assert hw_of('r50_os8_600x899/block3/unit_1/conv2')[1] == 113 and by['r50_os8_600x899/block3/unit_1/conv2'].rate == 2
    assert any(n.startswith('r50_v2_600x899/block3/') for n in names)
    assert all(r.n == 4 for r in PHOTO_LAYERS)
    assert not any('/rcnn/' in n for n in names)              # the RCNN heads do not depend on the image size
    assert not {r[1:] for r in PHOTO_LAYERS} & {r[1:] for r in LAYERS}


# ---------------------------------------------------------------------------------------------- GPU: conv launches
@pytest.mark.gpu
@pytest.mark.parametrize('row', PHOTO_LAYERS, ids=[r.name for r in PHOTO_LAYERS])
def test_photo_launch_matches_float64(row):
    """Codes 16 / 17 (18 / 19 for fp32 outputs) against float64 at the sampled pixels (every border pixel of each
    image and one pixel in 16), held to the per-element bound of test_gpu_conv_numerics."""
    launch_against_float64(row, 'photo_sizes/conv/')


def launch_against_float64(row, report_prefix):
    inputs = _inputs(row)
    x, w, scale, bias, res, pre = inputs
    launch = Launch(row, inputs)
    codes = (ENGINE_F32, ENGINE_F32_RESERVE) if row.f32 else (ENGINE, ENGINE_RESERVE)
    ho, wo, _, _ = out_geometry(row.h, row.w, row.k, row.stride, row.rate, row.padding)
    at = sample_pixels(row.n, ho, wo, zlib.crc32(row.name.encode()) + 1)
    rs = row.res[2] if row.res else 1
    ref, bound = reference(x, w, row.stride, row.padding, scale, bias, res, rs, row.act, codes[0], rate=row.rate, at=at)
    if pre:
        pref, pbound = preact_reference(ref, bound, *pre)
    worst = 0.0
    for impl in codes:
        y, p = launch.run(impl)
        tag = '%s/impl%d (%d px)' % (row.name, impl, len(at[0]))
        if y is not None:
            assert y.shape == (row.n, ho, wo, row.cout)
            worst = max(worst, check(tag, _gather(y, at), ref, bound))
        if p is not None:
            worst = max(worst, check(tag + '/p', _gather(p, at), pref, pbound))
    _report(report_prefix + row.name, err_over_bound=worst)


# ---------------------------------------------------------------------------------------------- GPU: end to end
R101_OVERRIDES = ['model.rpn.proposals.post_nms_top_n=300', 'model.rcnn.proposals.min_prob_threshold=0.0']


def _production(arch, overrides=()):
    """bench.py's Faster R-CNN config and weights (80 classes, post_nms_top_n 2000 unless overridden)."""
    cfg = default_config('fasterrcnn', ['model.base_network.architecture=' + arch, 'model.network.num_classes=80']
                         + list(overrides))
    return cfg, synth.make_weights(cfg, seed=0, profile='peaky')


def _engine(cfg, wts, n, h, w):
    from luminoth_b200.engine import Engine
    eng = Engine(cfg, max_batch=n, max_h=h, max_w=w)
    eng.load_weights(wts).finalize()
    return eng


def oracle_pair(cfg, wts, src, hw):
    """The fp32 and float64 oracle forward of `src` resized to hw on the host."""
    from oracle import fasterrcnn as ofr
    from oracle import tf_ops as T
    img = T.resize_bilinear(src.astype(np.float32), *hw)          # bit-identical to the engine's staging
    return ofr.forward(img, wts, cfg), ofr.forward(img, wts, cfg, dtype=np.float64)


def _against_oracle(key, cfg, wts, src, hw, i, out, fmap, pcnt, oracle=None):
    """Image i of a production call (out) against the fp32 and float64 oracle fed `src` resized to hw on the host
    (or `oracle`, the oracle_pair of that image already evaluated); fmap / pcnt: the feature map and proposal counts
    of a debug-taps run of the same call."""
    ref, tru = oracle or oracle_pair(cfg, wts, src, hw)
    fm = fmap[i, :-(-hw[0] // STRIDE), :-(-hw[1] // STRIDE)]
    assert fm.shape == tru['conv_feature_map'][0].shape, (fm.shape, tru['conv_feature_map'].shape)
    extra = dict(image_index=i, target_h=hw[0], target_w=hw[1],
                 fmap_rel_engine_vs_oracle64=rel_err(fm, tru['conv_feature_map'][0]),
                 fmap_rel_oracle32_vs_oracle64=rel_err(ref['conv_feature_map'][0], tru['conv_feature_map'][0]),
                 proposals_engine=int(pcnt[i]), proposals_oracle32=len(ref['rpn_prediction']['proposals']),
                 proposals_oracle64=len(tru['rpn_prediction']['proposals']))
    boxes, scores, labels, counts = out
    return _det_compare(key, boxes[i], scores[i], labels[i], int(counts[i]), ref['classification_prediction'],
                        tru['classification_prediction'], extra)


def _assert_all(results):
    for what, r in results:
        _assert_parity(r, what)
        assert r['detections_engine'] > 0, '%s: the comparison must not be vacuous' % what


# (name, arch, overrides, source shape, images compared): 600x800 once from each pipeline half
E2E = [('r50_600x800', 'resnet_v1_50', (), (480, 640), (0, 3)),
       ('r50_899x600', 'resnet_v1_50', (), (640, 427), (1,)),
       ('r50_576x1024', 'resnet_v1_50', (), (1080, 1920), (2,)),
       ('r101_600x899', 'resnet_v1_101', R101_OVERRIDES, (427, 640), (3,))]


@pytest.mark.gpu
@pytest.mark.parametrize('name,arch,overrides,shape,picks', E2E, ids=[c[0] for c in E2E])
def test_predict_resize_photos_meet_the_oracle(name, arch, overrides, shape, picks):
    """Four sources of one photo shape through predict_resize on the production path, the second call a graph
    replay of the first; the compared images' detections against the fp32 and float64 oracle."""
    cfg, wts = _production(arch, overrides)
    hw = target(shape)
    srcs = sources([shape] * 4, False, seed=zlib.crc32(name.encode()))
    eng = _engine(cfg, wts, 4, *hw)
    out = eng.predict_resize(srcs, *hw)
    assert_same(out, eng.predict_resize(srcs, *hw), name + ' graph replay')
    assert eng.last_graph_replays > 0
    eng.set_debug_taps(True)
    eng.predict_resize(srcs, *hw)
    fmap, pcnt = eng.get_tensor('conv_feature_map'), eng.get_tensor('proposal_counts').astype(int)
    eng.close()
    _assert_all([('%s image %d' % (name, i),
                  _against_oracle('photo_sizes/%s/img%d' % (name, i), cfg, wts, srcs[i], hw, i, out, fmap, pcnt))
                 for i in picks])


# ---------------------------------------------------------------------------------------------- GPU: packed photos
@pytest.mark.gpu
def test_packed_photos_equal_single_images():
    """Stream-K off: each image of the photo mix through predict_sizes (eager, then a graph replay) equals its own
    predict_resize call byte for byte, and its feature map cropped to its grid equals that call's map."""
    cfg, wts = _production('resnet_v1_50')
    srcs = sources(PACK_SOURCES, False, seed=7)
    eng = _engine(cfg, wts, len(srcs), *CANVAS)
    eng.set_conv_streamk('off')
    want, _ = singles(eng, srcs, PACK_TARGETS)
    assert int(want[3].sum()) > 0, 'the comparison must not be vacuous'
    for call in range(2):
        assert_same(want, eng.predict_sizes(srcs, PACK_TARGETS), 'photo mix call %d' % call)
    assert eng.last_graph_replays > 0
    eng.set_debug_taps(True)
    want, maps = singles(eng, srcs, PACK_TARGETS, 'conv_feature_map')
    assert_same(want, eng.predict_sizes(srcs, PACK_TARGETS), 'photo mix taps run')
    fmap = eng.get_tensor('conv_feature_map')
    assert fmap.shape[1:3] == (-(-CANVAS[0] // STRIDE), -(-CANVAS[1] // STRIDE))
    assert_crops(fmap, maps, PACK_TARGETS, STRIDE, 'photo mix')
    eng.close()


@pytest.mark.gpu
def test_packed_photos_meet_the_oracle():
    """Default stream-K: the 800x600 and 600x899 images of the packed photo mix against the fp32 and float64 oracle."""
    cfg, wts = _production('resnet_v1_50')
    srcs = sources(PACK_SOURCES, False, seed=8)
    eng = _engine(cfg, wts, len(srcs), *CANVAS)
    out = eng.predict_sizes(srcs, PACK_TARGETS)
    eng.set_debug_taps(True)
    eng.predict_sizes(srcs, PACK_TARGETS)
    fmap, pcnt = eng.get_tensor('conv_feature_map'), eng.get_tensor('proposal_counts').astype(int)
    eng.close()
    _assert_all([('packed photo mix image %d' % i,
                  _against_oracle('photo_sizes/packed/img%d' % i, cfg, wts, srcs[i], PACK_TARGETS[i], i, out, fmap,
                                  pcnt))
                 for i in (1, 2)])
