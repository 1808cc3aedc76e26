"""Faster R-CNN on banner, tower and tiny images, and on empty proposal lists (`-m gpu`, except the host checks).

The default preprocessing multiplies its up- and down-scale factors (utils/image.py:66-86), so strongly elongated
inputs land far beyond max_size: a 100x6000 banner becomes 102x6143, a 6000x100 tower 6143x102.  There the conv layers
run on one-pixel tiles: 128 rows by 1 column on every tower map from block1's stride-2 conv2 on (the stem's too), one
row by 128 columns on the banner's.  Tiny maps go the other way and pack several images into one tile.  Images under
55 px high have no anchor inside them, so with filter_outside_anchors their proposal list is empty.

* Launches: every R50 trunk and RPN conv at the four elongated targets and at 16x16 (batch 4) and 33x17 (batch 3:
  the last multi-image tile is ragged), plus resnet_v2_50 at the tower target, against float64 at sampled pixels
  (rows already in the 600x1024 or photo tables are left out); the stem through its tap at the tower, banner and
  16x16 sizes.
* End to end: predict_resize on four banner and on four tower sources, production config and path (R50, 80
  classes, 2000 proposals, bench's weights; pipeline, default stream-K, graph replay) on an engine created for
  600x1024, which these targets outgrow: the 600x1024 batch it served before must give the same bytes after.  One
  image of each pipeline half against the fp32 and float64 oracle; the tower also on the SIMT conv.
* Empty lists: batches without proposals (R50, R101 and the RPN-only mode), the 54 / 55 px anchor boundary packed
  with a full image, the record output of an empty image, PredictorNetwork on a 40x15000 strip, and the 1x1 and
  16x16 images without the filter.
"""
import zlib

import numpy as np
import pytest

from luminoth_b200 import synth
from oracle.anchors import fasterrcnn_anchors
from test_gpu_baseline_configs import _assert_parity, _det_compare, _report
from test_gpu_conv_engine_layers import LAYERS, _dedupe, frcnn_heads, out_geometry, resnet_rows, stem_against_float64
from test_gpu_conv_numerics import pick_tile
from test_gpu_e2e import box_dev, float_bound, frcnn_cfg
from test_gpu_packed_sizes import singles
from test_gpu_photo_sizes import (PHOTO_LAYERS, PREPROCESSING, _against_oracle, _assert_all, _engine, _production,
                                  _tag, launch_against_float64, oracle_pair, target)
from test_gpu_resize_input import assert_same, sources

# banner, tower, a 3:40 panorama and a 40x15000 strip (no anchor fits inside it: it has no proposals)
ELONGATED = [(100, 6000), (6000, 100), (300, 4000), (40, 15000)]
BANNER, TOWER = target((100, 6000)), target((6000, 100))
TINY = [((16, 16), 4), ((33, 17), 3)]                    # (map, batch)
STRIDE = 16


def _extreme_layers():
    rows = []
    for hw in [target(s) for s in ELONGATED]:
        trunk, fhw = resnet_rows(_tag('r50', hw), 4, *hw)
        rows += trunk + frcnn_heads(_tag('r50', hw), 4, fhw, 1024)[:2]
    for hw, n in TINY:
        trunk, fhw = resnet_rows(_tag('r50', hw), n, *hw)
        rows += trunk + frcnn_heads(_tag('r50', hw), n, fhw, 1024)[:2]
    rows += resnet_rows(_tag('r50_v2', TOWER), 4, *TOWER, v2=True)[0]
    known = {r[1:] for r in LAYERS} | {r[1:] for r in PHOTO_LAYERS}
    return [r for r in _dedupe(rows) if r[1:] not in known]


EXTREME_LAYERS = _extreme_layers()


def _tile(row):
    ho, wo, _, _ = out_geometry(row.h, row.w, row.k, row.stride, row.rate, row.padding)
    return pick_tile(row.n, ho, wo)


def _stem_map(h, w):
    return out_geometry(h, w, 7, 2, 1, 'SLIM')[:2]


def anchors_inside(h, w):
    """Anchors of an h x w image that lie inside it (rpn_proposal.py:71-90, filter_outside_anchors)."""
    from luminoth_b200 import default_config
    a = default_config('fasterrcnn', [])['model']['anchors']
    an = fasterrcnn_anchors(-(-h // STRIDE), -(-w // STRIDE), a['base_size'], a['ratios'], a['scales'], a['stride'])
    return int(((an[:, 0] >= 0) & (an[:, 1] >= 0) & (an[:, 2] < w) & (an[:, 3] < h)).sum())


# ---------------------------------------------------------------------------------------------- host checks
def test_extreme_targets():
    """The targets the default preprocessing derives for elongated inputs: far beyond max_size on the long side."""
    assert [target(s) for s in ELONGATED] == [(102, 6143), (6143, 102), (153, 2048), (40, 15360)]
    assert PREPROCESSING['dataset']['image_preprocessing']['max_size'] == 1024


def test_extreme_layer_table_geometry():
    """Feature maps of the derived targets, and the conv kernel's M tiles on them.  The tiles restate conv.cu's
    pick_tile (test_gpu_conv_numerics.pick_tile): the table must hold one-column tiles (tw = 1) on maps wider than
    one pixel, one-row tiles (th = 1) and multi-image tiles (nb > 1), one of them ragged."""
    by = {r.name: r for r in EXTREME_LAYERS}
    hw_of = lambda name: (by[name].h, by[name].w)
    assert hw_of('r50_102x6143/rpn/conv') == (7, 384)
    assert hw_of('r50_6143x102/rpn/conv') == (384, 7)
    assert hw_of('r50_153x2048/rpn/conv') == (10, 128)
    assert hw_of('r50_40x15360/rpn/conv') == (3, 960)
    assert hw_of('r50_6143x102/block1/unit_1/conv1') == (1536, 26)
    assert hw_of('r50_16x16/rpn/conv') == (1, 1) and hw_of('r50_33x17/rpn/conv') == (3, 2)
    # the stem (tested through its tap) and the trunk of the tower: 128 x 1 tiles, block1 64 x 2; the banner 1 x 128
    assert pick_tile(4, *_stem_map(*TOWER)) == (1, 128, 1) and pick_tile(4, *_stem_map(*BANNER)) == (1, 1, 128)
    assert _tile(by['r50_6143x102/block1/unit_1/conv2']) == (1, 64, 2)
    for name in ('block1/unit_3/conv2', 'block2/unit_1/conv2', 'block3/unit_1/conv1', 'rpn/conv'):
        assert _tile(by['r50_6143x102/' + name]) == (1, 128, 1), name
        assert _tile(by['r50_102x6143/' + name]) == (1, 1, 128), name
    assert _tile(by['r50_40x15360/rpn/conv']) == (1, 3, 42)
    assert _tile(by['r50_16x16/block2/unit_4/conv2']) == (4, 1, 1)         # 2x2 -> 1x1, four images per tile
    assert _tile(by['r50_33x17/block1/unit_1/conv1']) == (2, 9, 5)          # three images: the last tile holds one
    tiles = [(r, _tile(r)) for r in EXTREME_LAYERS]
    out_w = lambda r: out_geometry(r.h, r.w, r.k, r.stride, r.rate, r.padding)[1]
    assert any(t[2] == 1 and out_w(r) > 1 for r, t in tiles)
    assert any(t[1] == 1 and t[2] > 1 for r, t in tiles)
    assert any(t[0] > 1 for r, t in tiles) and any(t[0] > 1 and r.n % t[0] for r, t in tiles)
    assert any(n.startswith('r50_v2_6143x102/block3/') for n in by)
    assert not any('/rcnn/' in n for n in by)
    assert not {r[1:] for r in EXTREME_LAYERS} & ({r[1:] for r in LAYERS} | {r[1:] for r in PHOTO_LAYERS})


def test_anchors_inside_boundary():
    """The flattest anchors (scale 0.25, ratio 0.5) span y = 16 r - 22 ... 16 r + 22 on feature row r, so the first
    inside an image is row 2's, 10 ... 54, which needs 55 px: no anchor lies inside an image under 55 px high."""
    assert anchors_inside(54, 640) == 0 and anchors_inside(55, 640) == 35
    assert anchors_inside(*target((40, 15000))) == 0 and anchors_inside(40, 640) == 0


# ---------------------------------------------------------------------------------------------- GPU: conv launches
@pytest.mark.gpu
@pytest.mark.parametrize('row', EXTREME_LAYERS, ids=[r.name for r in EXTREME_LAYERS])
def test_extreme_launch_matches_float64(row):
    """Codes 16 / 17 (18 / 19 for fp32 outputs) against float64 at the sampled pixels, held to the per-element
    bound of test_gpu_conv_numerics."""
    launch_against_float64(row, 'extreme_sizes/conv/')


@pytest.mark.gpu
@pytest.mark.parametrize('n,h,w', [(2,) + TOWER, (2,) + BANNER, (4, 16, 16)], ids=['tower', 'banner', '16x16'])
def test_extreme_stem_matches_float64(n, h, w):
    """The stem over its space-to-depth view: 128 x 1 tiles on the tower, 1 x 128 on the banner, two images per
    tile at 16x16."""
    _report('extreme_sizes/stem/%dx%dx%d' % (n, h, w), err_over_bound=stem_against_float64(n, h, w))


# ---------------------------------------------------------------------------------------------- GPU: end to end
HINT = (600, 1024)          # the engine's sizing hint: an RPN workspace for 38 x 64 x 12 = 29 184 anchors


@pytest.mark.gpu
@pytest.mark.parametrize('name,shape', [('banner', (100, 6000)), ('tower', (6000, 100))], ids=['banner', 'tower'])
def test_predict_resize_elongated_meets_the_oracle(name, shape):
    """Four sources through predict_resize on the production path, on an engine that served (and graph-captured) a
    600x1024 batch first.  The target's 7 x 384 x 12 = 32 256 anchors outgrow the workspace, so the call grows it and
    drops the graphs; the 600x1024 batch then gives the same bytes, eager and on replay.  Images 0 and 3 (one per
    pipeline half) against the fp32 and float64 oracle; the tower's image 0 also on the SIMT conv."""
    cfg, wts = _production('resnet_v1_50')
    hw = target(shape)
    assert (-(-hw[0] // STRIDE)) * (-(-hw[1] // STRIDE)) * 12 > (-(-HINT[0] // STRIDE)) * (-(-HINT[1] // STRIDE)) * 12
    srcs = sources([shape] * 4, False, seed=zlib.crc32(name.encode()))
    photos = sources([(480, 640)] * 4, False, seed=zlib.crc32(name.encode()) + 1)
    eng = _engine(cfg, wts, 4, *HINT)
    before = eng.predict_resize(photos, *HINT)
    assert_same(before, eng.predict_resize(photos, *HINT), '600x1024 graph replay')
    assert eng.last_graph_replays > 0 and int(before[3].sum()) > 0
    out = eng.predict_resize(srcs, *hw)
    assert_same(out, eng.predict_resize(srcs, *hw), name + ' graph replay')
    assert eng.last_graph_replays > 0
    for call in ('eager', 'graph replay'):
        assert_same(before, eng.predict_resize(photos, *HINT), '600x1024 %s after the growth' % call)
        assert (eng.last_graph_replays > 0) == (call == 'graph replay'), 'the growth must drop the graphs'
    eng.set_debug_taps(True)
    eng.predict_resize(srcs, *hw)
    taps = {'tc': (out, eng.get_tensor('conv_feature_map'), eng.get_tensor('proposal_counts').astype(int))}
    if name == 'tower':
        eng.set_debug_taps(False)
        eng.set_conv_impl('simt')
        simt = eng.predict_resize(srcs, *hw)
        eng.set_debug_taps(True)
        assert_same(simt, eng.predict_resize(srcs, *hw), 'simt taps run')
        taps['simt'] = (simt, eng.get_tensor('conv_feature_map'), eng.get_tensor('proposal_counts').astype(int))
    eng.close()
    results = []
    for i in (0, 3):
        oracle = oracle_pair(cfg, wts, srcs[i], hw)
        for impl, (o, fmap, pcnt) in sorted(taps.items()):
            if impl == 'tc' or i == 0:
                results.append(('%s %s image %d' % (name, impl, i),
                                _against_oracle('extreme_sizes/%s_%s/img%d' % (name, impl, i), cfg, wts, srcs[i], hw,
                                                i, o, fmap, pcnt, oracle)))
    _assert_all(results)


# ---------------------------------------------------------------------------------------------- GPU: empty lists
FILTER = ('model.rpn.proposals.filter_outside_anchors=true',)
EMPTY = [('r50', 'resnet_v1_50', ()), ('r101', 'resnet_v1_101', ()),
         ('r50_rpn_only', 'resnet_v1_50', ('model.network.with_rcnn=false',))]


def _small(arch, extra=(), filt=True):
    cfg = frcnn_cfg(arch, (FILTER if filt else ()) + tuple(extra))
    return cfg, synth.make_weights(cfg, seed=1)


def _small_engine(cfg, wts, n, h, w):
    from luminoth_b200.engine import Engine
    eng = Engine(cfg, max_batch=n, max_h=h, max_w=w)
    eng.load_weights(wts).finalize()
    return eng


@pytest.mark.gpu
@pytest.mark.parametrize('name,arch,extra', EMPTY, ids=[c[0] for c in EMPTY])
def test_batch_without_proposals(name, arch, extra):
    """Three 40x640 images (pipeline halves of 2 and 1): no anchor inside any of them, so the RPN keeps nothing, the
    ROI and RCNN stages (R101: the block4 tail) run on padding rows only, and every count is exactly 0 -- eager, on
    graph replay and in the debug-taps run; no LUMI_EOVERFLOW (predict_raw raises it)."""
    from oracle import fasterrcnn as ofr
    cfg, wts = _small(arch, extra)
    imgs = synth.make_images(3, 40, 640, seed=51)
    eng = _small_engine(cfg, wts, 3, 40, 640)
    out = eng.predict_raw(imgs)
    np.testing.assert_array_equal(out[3], [0, 0, 0])
    assert_same(out, eng.predict_raw(imgs), name + ' graph replay')
    assert eng.last_graph_replays > 0
    eng.set_debug_taps(True)
    assert_same(out, eng.predict_raw(imgs), name + ' taps run')
    np.testing.assert_array_equal(eng.get_tensor('proposal_counts').astype(int), [0, 0, 0])
    eng.close()
    ref = ofr.forward(imgs[0], wts, cfg)
    assert len(ref['rpn_prediction']['proposals']) == 0
    assert 'classification_prediction' not in ref or len(ref['classification_prediction']['probs']) == 0


BOUNDARY_TARGETS = [(54, 640), (55, 640), (600, 640)]
BOUNDARY_SOURCES = [(54, 640), (50, 580), (480, 512)]


@pytest.mark.gpu
@pytest.mark.parametrize('arch', ['resnet_v1_50', 'resnet_v1_101'], ids=['r50', 'r101'])
def test_anchor_boundary_packed(arch):
    """54, 55 and 600 px high images in one predict_sizes call.  Stream-K off: each equals its single-image call
    byte for byte, eager and on graph replay.  Default stream-K: the 54 px image has no proposals and no detections,
    the others meet the oracle (its proposal count, and the detections under the baseline parity rule)."""
    cfg, wts = _small(arch)
    srcs = sources(BOUNDARY_SOURCES, False, seed=61)
    eng = _small_engine(cfg, wts, 3, 600, 640)
    eng.set_conv_streamk('off')
    want, _ = singles(eng, srcs, BOUNDARY_TARGETS)
    assert want[3][0] == 0 and (want[3][1:] > 0).all(), want[3]
    for call in range(2):
        assert_same(want, eng.predict_sizes(srcs, BOUNDARY_TARGETS), 'boundary mix call %d' % call)
    assert eng.last_graph_replays > 0
    eng.set_conv_streamk('auto')
    out = eng.predict_sizes(srcs, BOUNDARY_TARGETS)
    eng.set_debug_taps(True)
    eng.predict_sizes(srcs, BOUNDARY_TARGETS)
    fmap, pcnt = eng.get_tensor('conv_feature_map'), eng.get_tensor('proposal_counts').astype(int)
    eng.close()
    assert out[3][0] == 0 and pcnt[0] == 0
    for i, hw in enumerate(BOUNDARY_TARGETS):
        r = _against_oracle('extreme_sizes/boundary_%s/img%d' % (arch, i), cfg, wts, srcs[i], hw, i, out, fmap, pcnt)
        what = '%s %dx%d' % (arch, hw[0], hw[1])
        assert r['proposals_engine'] in (r['proposals_oracle32'], r['proposals_oracle64']), (what, r)
        assert (r['proposals_engine'] == 0) == (i == 0), (what, r)
        _assert_parity(r, what)
        assert (r['detections_engine'] > 0) == (i > 0), (what, r)


@pytest.mark.gpu
def test_record_output_of_an_image_without_proposals():
    """set_record_output: the record of the 54 px image says 0, the other's its count; both rows repeat the returned
    arrays, eager and on graph replay."""
    import torch
    cfg, wts = _small('resnet_v1_50')
    srcs = sources([(54, 640), (600, 640)], False, seed=71)
    targets = [(54, 640), (600, 640)]
    eng = _small_engine(cfg, wts, 2, 600, 640)
    k = eng.max_detections
    rec = torch.full((2, 1 + 6 * k), 7.0, dtype=torch.float32, device='cuda')
    eng.set_record_output(rec)
    for call in ('eager', 'graph replay'):
        rec.fill_(7.0)
        boxes, scores, labels, counts = eng.predict_sizes(srcs, targets)
        r = rec.cpu().numpy()
        assert counts[0] == 0 and counts[1] > 0, counts
        for i in range(2):
            np.testing.assert_array_equal(r[i, 0], counts[i], err_msg=call)
            np.testing.assert_array_equal(r[i, 1:1 + 4 * k], boxes[i].reshape(-1), err_msg=call)
            np.testing.assert_array_equal(r[i, 1 + 4 * k:1 + 5 * k], scores[i], err_msg=call)
            np.testing.assert_array_equal(r[i, 1 + 5 * k:], labels[i].astype(np.float32), err_msg=call)
    assert eng.last_graph_replays > 0
    eng.set_record_output(None)
    eng.close()


@pytest.mark.gpu
def test_predictor_on_a_strip_returns_no_detections():
    """PredictorNetwork.predict_image on a 40x15000 strip (target 40x15360, no anchor inside) returns [], as the
    oracle's predict_image does."""
    from luminoth_b200.predicting import PredictorNetwork
    from oracle import predict as opredict
    cfg, wts = _small('resnet_v1_50')
    img = synth.make_images(1, 40, 15000, seed=81)[0]
    net = PredictorNetwork(cfg, weights=wts)
    assert net.predict_image(img) == []
    net.engine.close()
    assert opredict.predict_image(img, wts, cfg) == []


@pytest.mark.gpu
@pytest.mark.parametrize('h,w,proposals', [(1, 1, 12), (16, 16, 1)], ids=['1x1', '16x16'])
def test_tiny_image_without_the_filter(h, w, proposals):
    """Without the filter a 1x1 image keeps its 12 anchors' proposals, all clipped to the zero-area box (NMS keeps
    every one: the IoU is 0 when an area is <= 0), and has no detections; a 16x16 image (a one-cell feature map)
    keeps one proposal.  Proposals and detections against the oracle."""
    from oracle import fasterrcnn as ofr
    cfg, wts = _small('resnet_v1_50', filt=False)
    img = synth.make_images(1, h, w, seed=2)
    eng = _small_engine(cfg, wts, 1, 16, 16)
    eng.set_debug_taps(True)
    boxes, scores, labels, counts = eng.predict_raw(img)
    props, pcnt = eng.get_tensor('proposals'), int(eng.get_tensor('proposal_counts').astype(int)[0])
    eng.close()
    ref, tru = ofr.forward(img[0], wts, cfg), ofr.forward(img[0], wts, cfg, dtype=np.float64)
    assert pcnt == proposals == len(tru['rpn_prediction']['proposals']) == len(ref['rpn_prediction']['proposals'])
    got = props.reshape(1, -1, 4)[0, :pcnt]
    if (h, w) == (1, 1):
        np.testing.assert_array_equal(got, np.zeros((12, 4), np.float32))
        np.testing.assert_array_equal(tru['rpn_prediction']['proposals'], np.zeros((12, 4)))
    z = np.zeros(pcnt, int)
    e, o = box_dev(got, z, tru['rpn_prediction']['proposals'], z), box_dev(ref['rpn_prediction']['proposals'], z,
                                                                           tru['rpn_prediction']['proposals'], z)
    assert e <= float_bound(o, 1e-3), 'proposals: engine %.2e px vs oracle32 %.2e px' % (e, o)
    k = int(counts[0])
    r = _det_compare('extreme_sizes/tiny_%dx%d' % (h, w), boxes[0], scores[0], labels[0], k,
                     ref['classification_prediction'], tru['classification_prediction'])
    _assert_parity(r, '%dx%d image' % (h, w))
    assert (k > 0) == ((h, w) == (16, 16)), k
