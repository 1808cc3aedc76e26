"""Images of different sizes in one forward: ``lumi_predict_sizes`` (`-m gpu`).

Each image sits at the top left of a canvas of the largest target height and width.  The staging zeros the canvas
outside it, a band clear ahead of every windowed conv restores the zero padding its valid outputs read when it runs
alone, and pool1, the RPN, the ROI pool and the detections use its own size.  With stream-K off a conv's whole-tile
result does not depend on the tiling, so every image's results must equal the single-image ``predict_resize`` call
byte for byte, and so must its feature map cropped to its own grid.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import resnet_v2_oracle as V2
from luminoth_b200 import synth
from luminoth_b200.engine import Engine
from oracle import tf_ops as T
from test_gpu_e2e import box_dev, float_bound, frcnn_cfg, _report
from test_gpu_resize_input import assert_same, on_device, sources
from test_ssd_config_host import ssd_cfg

# Targets on a 320 x 320 canvas: one image shorter and one narrower than it, odd stem heights (201 -> 101, 250 -> 125:
# pool1 pads those images 1 in front, the even canvas 0) next to even ones, and one image a pixel smaller than the
# canvas.  Five images: the pipeline halves differ in size.
MIX = [(224, 320), (320, 224), (201, 299), (319, 319), (250, 283)]
# A second mix on the same canvas (the graph replay test).
MIX2 = [(320, 300), (300, 320), (222, 222), (320, 320), (257, 199)]
CANVAS = (320, 320)


def source_sizes(targets, seed):
    """A source size per target: down- and upscales, and one source already at its target size."""
    rng = np.random.default_rng(seed)
    out = [(max(1, int(h * rng.uniform(0.6, 1.4))), max(1, int(w * rng.uniform(0.6, 1.4)))) for h, w in targets]
    out[0] = tuple(targets[0])
    return out


def make_engine(cfg, wts, n, impl, taps=False, pipeline=True):
    eng = Engine(cfg, max_batch=n, max_h=CANVAS[0], max_w=CANVAS[1])
    eng.load_weights(wts).finalize()
    eng.set_conv_impl(impl)
    eng.set_conv_streamk('off')
    eng.set_pipeline(pipeline)
    eng.set_debug_taps(taps)
    return eng


def singles(eng, srcs, targets, tap=None, stride=None):
    """Results of one predict_resize call per image, stacked like a batched call; with `tap`, also that tap's map of
    every image."""
    outs, maps = [], []
    for im, (h, w) in zip(srcs, targets):
        outs.append(eng.predict_resize([im], h, w))
        if tap:
            maps.append(eng.get_tensor(tap)[0])
    return [np.concatenate([o[k] for o in outs]) for k in range(4)], maps


def assert_crops(packed_map, maps, targets, stride, what):
    for i, ((h, w), ref) in enumerate(zip(targets, maps)):
        fh, fw = -(-h // stride), -(-w // stride)
        assert ref.shape[:2] == (fh, fw), (ref.shape, fh, fw)
        np.testing.assert_array_equal(packed_map[i, :fh, :fw], ref, err_msg='%s: image %d map' % (what, i))


# (name, arch, config overrides, conv impl, pipeline, endpoint stride)
CASES = [
    ('r50_tc', 'resnet_v1_50', (), 'tc', True, 16),
    ('r50_tc_nopipe', 'resnet_v1_50', (), 'tc', False, 16),
    ('r50_simt', 'resnet_v1_50', (), 'simt', True, 16),
    ('r50v2_tc', 'resnet_v2_50', (), 'tc', True, 16),
    ('r101_tail_tc', 'resnet_v1_101', (), 'tc', True, 16),
    ('r50_os8', 'resnet_v1_50', ('model.base_network.output_stride=8',), 'tc', True, 8),
    ('r50_conv1', 'resnet_v1_50', ('model.base_network.endpoint=conv1', 'model.network.with_rcnn=false'), 'tc', True,
     2),
    ('r50_block1', 'resnet_v1_50', ('model.base_network.endpoint=block1',), 'tc', True, 8),
    ('r50_block4', 'resnet_v1_50', ('model.base_network.endpoint=block4', 'model.base_network.output_stride=32'),
     'tc', True, 32),
    ('r50_rpn_only_filter', 'resnet_v1_50', ('model.network.with_rcnn=false',
                                            'model.rpn.proposals.filter_outside_anchors=true'), 'tc', True, 16),
]


@pytest.mark.parametrize('name,arch,extra,impl,pipeline,stride', CASES, ids=[c[0] for c in CASES])
def test_packed_equals_single_images(name, arch, extra, impl, pipeline, stride):
    """uint8 host sources through predict_sizes equal one predict_resize call per image, and with debug taps the
    feature map cropped to each image's grid equals that image's own map.  The first case also runs float32 and
    device sources."""
    cfg = frcnn_cfg(arch, list(extra))
    wts = synth.make_weights(cfg, seed=1)
    n = len(MIX)
    eng = make_engine(cfg, wts, n, impl, pipeline=pipeline)
    kinds = [(False, 'host'), (True, 'host'), (False, 'device'), (True, 'device')] if name == 'r50_tc' else \
        [(False, 'host')]
    for f32, where in kinds:
        srcs = sources(source_sizes(MIX, seed=3), f32, seed=4 + f32)
        want, _ = singles(eng, srcs, MIX)
        assert int(want[3].sum()) > 0, 'the comparison must not be vacuous'
        feed = on_device(srcs) if where == 'device' else srcs
        for call in range(2):
            assert_same(want, eng.predict_sizes(feed, MIX), '%s %s %s call %d' % (name, f32, where, call))
    eng.close()
    dbg = make_engine(cfg, wts, n, impl, taps=True)
    srcs = sources(source_sizes(MIX, seed=3), False, seed=4)
    want, maps = singles(dbg, srcs, MIX, 'conv_feature_map')
    assert_same(want, dbg.predict_sizes(srcs, MIX), name + ' taps run')
    fmap = dbg.get_tensor('conv_feature_map')
    assert fmap.shape[1:3] == (-(-CANVAS[0] // stride), -(-CANVAS[1] // stride))
    assert_crops(fmap, maps, MIX, stride, name)
    dbg.close()


def test_packed_graph_replays_read_the_new_mix():
    """Two mixes on one canvas with graphs on: the later calls replay the captured forwards, read the second mix's
    sizes from the table and still equal the single-image calls."""
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=1)
    eng = make_engine(cfg, wts, len(MIX), 'tc')
    ref = make_engine(cfg, wts, len(MIX), 'tc')
    ref.set_graphs(False)
    a = sources(source_sizes(MIX, seed=5), False, seed=6)
    b = sources(source_sizes(MIX, seed=5), False, seed=8)      # sources of A's sizes: the source buffer does not grow
    want_a, _ = singles(ref, a, MIX)
    want_b, _ = singles(ref, b, MIX2)
    for call in range(3):                                   # eager, capture, replay
        assert_same(want_a, eng.predict_sizes(a, MIX), 'mix A call %d' % call)
    assert eng.last_graph_replays > 0
    for call in range(2):
        assert_same(want_b, eng.predict_sizes(b, MIX2), 'mix B call %d' % call)
        assert eng.last_graph_replays > 0, 'mix B call %d was not a replay' % call
    eng.close()
    ref.close()


def test_packed_meets_the_float64_oracle():
    """Default stream-K: each image of a packed call against the float64 oracle fed that image resized to its own
    target -- the rule of test_fasterrcnn_float_pixels_stages_and_detections, with identical counts and classes."""
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=1)
    targets = [(224, 320), (201, 299)]
    srcs = sources([(160, 224), (150, 210)], True, seed=9)
    eng = Engine(cfg, max_batch=2, max_h=224, max_w=320)
    eng.load_weights(wts).finalize()
    boxes, scores, labels, counts = eng.predict_sizes(srcs, targets)
    for i, (im, (h, w)) in enumerate(zip(srcs, targets)):
        img = T.resize_bilinear(im, h, w)
        ref = V2.fasterrcnn_forward(img, wts, cfg)
        tru = V2.fasterrcnn_forward(img, wts, cfg, dtype=np.float64)
        k = int(counts[i])
        tc_, rc_ = tru['classification_prediction'], ref['classification_prediction']
        assert k == tc_['labels'].shape[0], 'image %d: %d detections vs %d' % (i, k, tc_['labels'].shape[0])
        assert sorted(labels[i, :k].tolist()) == sorted(np.asarray(tc_['labels']).tolist())
        e_det = box_dev(boxes[i, :k], labels[i, :k], tc_['objects'], tc_['labels'])
        o_det = box_dev(rc_['objects'], rc_['labels'], tc_['objects'], tc_['labels'])
        e_p = float(np.abs(np.sort(scores[i, :k]) - np.sort(tc_['probs'])).max()) if k else 0.0
        _report('packed_sizes/frcnn/img%d' % i, detections_px_engine=e_det, detections_px_oracle32=o_det,
                probs_abs_engine=e_p, detections=k)
        assert k > 0
        assert e_det <= float_bound(o_det, 1e-3), 'detections: engine %.2e px vs oracle32 %.2e px' % (e_det, o_det)
        assert e_p <= 2e-5
    eng.close()


def test_packed_bad_input_and_ssd():
    """Targets below 1, more images than max_batch and SSD at other sizes than its fixed one are ValueErrors, after
    which the engine serves the next call; SSD with every target at its fixed size is predict_resize."""
    cfg = frcnn_cfg('resnet_v1_50')
    eng = make_engine(cfg, synth.make_weights(cfg, seed=1), 2, 'tc')
    srcs = sources([(100, 120), (90, 80)], False, seed=10)
    good = eng.predict_sizes(srcs, [(224, 320), (201, 299)])
    for targets in ([(0, 320), (201, 299)], [(224, 320), (201, -1)]):
        with pytest.raises(ValueError, match='targets must be >= 1'):
            eng.predict_sizes(srcs, targets)
    with pytest.raises(ValueError, match='max_batch'):
        eng.predict_sizes(srcs + srcs[:1], [(224, 320), (201, 299), (100, 100)])
    assert_same(good, eng.predict_sizes(srcs, [(224, 320), (201, 299)]), 'after the refused calls')
    eng.close()

    cfg = ssd_cfg(300, 300)
    cfg['model']['proposals']['min_prob_threshold'] = 0.2
    ssd = Engine(cfg, max_batch=2, max_h=300, max_w=300)
    ssd.load_weights(synth.make_weights(cfg, seed=5)).finalize()
    srcs = sources([(375, 500), (120, 90)], False, seed=11)
    with pytest.raises(ValueError, match='fixed size'):
        ssd.predict_sizes(srcs, [(300, 300), (200, 300)])
    want = ssd.predict_resize(srcs, 300, 300)
    assert int(want[3].sum()) > 0
    assert_same(want, ssd.predict_sizes(srcs, [(300, 300), (300, 300)]), 'ssd at its fixed size')
    ssd.close()
