"""Sliced prediction of large images (`-m gpu`): ``lumi_predict_windows``.

* Window staging: every chunk's per-window detections equal ``predict_resize`` on the host-cropped windows of that
  chunk, byte for byte (uint8 / float32 sources on the host and on the device, Faster R-CNN R50 and SSD 300, windows at
  the four borders, 1 x 1 and 1 x W windows, the whole image, more windows than max_batch, a graph replay).
* Merge: the call's outputs equal the numpy restatement (tests/tile_merge_ref.py) of the merge of those per-window
  detections, byte for byte: 80 classes at min_prob 0, the RPN-only mode, windows without detections.
* End to end: two images through ``predict_tiled`` against the fp32 and float64 oracle run per window and merged by
  the same restatement, with the rule of test_gpu_photo_sizes.
* Memory: a 4000 x 6000 photo at 600 px tiles, 80 classes and min_prob 0 completes with the merge workspace inside
  the bound of DESIGN section 4.2, and its merged detections equal the restatement byte for byte.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from luminoth_b200 import default_config, synth
from luminoth_b200.engine import Engine
from luminoth_b200.predicting import PredictorNetwork, target_size, tile_grid
from test_gpu_baseline_configs import _assert_parity, _det_compare
from test_gpu_e2e import frcnn_cfg
from test_gpu_resize_input import assert_same, on_device, sources
from test_ssd_config_host import ssd_cfg
from tile_merge_ref import merge_windows


def _engine(cfg, wts, max_batch, h, w):
    eng = Engine(cfg, max_batch=max_batch, max_h=h, max_w=w)
    eng.load_weights(wts).finalize()
    return eng


def _chunks(windows, max_batch):
    """[start, end) of each chunk the engine runs: runs of equal targets, cut at max_batch."""
    out, a = [], 0
    while a < len(windows):
        b = a + 1
        while b < len(windows) and b - a < max_batch and tuple(windows[b][5:]) == tuple(windows[a][5:]):
            b += 1
        out.append((a, b))
        a = b
    return out


def _crop(src, wdw):
    _, y0, x0, h, w = wdw[:5]
    return src[y0:y0 + h, x0:x0 + w]


def _check_staging(eng, srcs, feed, windows, tag):
    scales = [(1.0, 1.0)] * len(windows)
    eng.predict_windows(feed, windows, scales, 0.5)
    replays = eng.last_graph_replays
    wb, ws, wl, wc, _ = eng.last_window_detections()
    assert int(wc.sum()) > 0, tag + ': the comparison must not be vacuous'
    for a, b in _chunks(windows, eng.max_batch):
        crops = [_crop(srcs[w[0]], w) for w in windows[a:b]]
        want = eng.predict_resize(crops, *windows[a][5:])
        assert_same(want, (wb[a:b], ws[a:b], wl[a:b], wc[a:b]), '%s chunk [%d, %d)' % (tag, a, b))
    return replays


def _staging_case(kind):
    if kind == 'frcnn':
        cfg = frcnn_cfg('resnet_v1_50')
        return cfg, synth.make_weights(cfg, seed=1), (224, 320), (160, 224)
    cfg = ssd_cfg(300, 300)
    cfg['model']['proposals']['min_prob_threshold'] = 0.2
    return cfg, synth.make_weights(cfg, seed=5), (300, 300), (300, 300)


@pytest.mark.parametrize('kind', ['frcnn', 'ssd'])
def test_window_staging_equals_predict_resize_on_crops(kind):
    cfg, wts, t1, t2 = _staging_case(kind)
    eng = _engine(cfg, wts, 3, *t1)
    H, W = 300, 420
    windows = [(0, 0, 0, 200, 280), (0, 0, 140, 200, 280), (0, 100, 0, 200, 280), (0, 100, 140, 200, 280),
               (0, 150, 200, 1, 1), (0, 299, 0, 1, 420), (0, 0, 0, H, W), (1, 0, 0, 1, 350),
               (1, 0, 349, 1, 1), (0, 0, 419, 300, 1)]
    windows = [w + t1 for w in windows[:8]] + [w + t2 for w in windows[8:]]
    # the same shapes at other offsets: every chunk a graph replay of the first call's
    moved = [(w[0], max(0, w[1] - 1), max(0, w[2] - 3)) + w[3:] for w in windows]
    for f32 in (False, True):
        srcs = sources([(H, W), (1, 350)], f32, seed=21 + f32)
        for where, feed in (('host', srcs), ('device', on_device(srcs))):
            tag = '%s %s %s' % (kind, 'f32' if f32 else 'u8', where)
            _check_staging(eng, srcs, feed, windows, tag)
            replays = _check_staging(eng, srcs, feed, moved, tag + ' moved')
            assert replays > 0, tag + ': the second call should replay graphs'
    eng.close()


def _merge_ref(eng, windows, scales, nsrc, nc, class_max, total_max, thr):
    wb, ws, wl, wc, stats = eng.last_window_detections()
    wmap = [(w[1], w[2], s[0], s[1]) for w, s in zip(windows, scales)]
    return merge_windows(wb, ws, wl, wc, [w[0] for w in windows], wmap, nsrc, nc, class_max, total_max, thr), stats


def _assert_merge(out, ref, tag):
    boxes, scores, labels, counts = out
    for i, (rb, rs, rl) in enumerate(ref):
        k = int(counts[i])
        assert k == len(rs), '%s source %d: %d detections, numpy merge %d' % (tag, i, k, len(rs))
        np.testing.assert_array_equal(boxes[i, :k], rb, err_msg='%s source %d boxes' % (tag, i))
        np.testing.assert_array_equal(scores[i, :k], rs, err_msg='%s source %d scores' % (tag, i))
        np.testing.assert_array_equal(labels[i, :k], rl, err_msg='%s source %d labels' % (tag, i))


def _tiled_windows(cfg, shapes, tile, overlap=0.2):
    windows, scales = [], []
    for i, (h, w) in enumerate(shapes):
        grid = tile_grid(h, w, tile, tile, overlap) + [(0, 0, h, w)]
        for y0, x0, wh, ww in grid:
            nh, nw, s = target_size((wh, ww), cfg)
            windows.append((i, y0, x0, wh, ww, nh, nw))
            scales.append(tuple(s) if isinstance(s, tuple) else (s, s))
    return windows, scales


@pytest.mark.parametrize('mode', ['80_classes', 'rpn_only', 'no_detections'])
def test_merge_equals_numpy(mode):
    over = {'80_classes': ['model.network.num_classes=80', 'model.rcnn.proposals.min_prob_threshold=0.0'],
            'rpn_only': ['model.network.with_rcnn=false', 'model.rpn.proposals.post_nms_top_n=60'],
            'no_detections': ['model.rcnn.proposals.min_prob_threshold=1.5']}[mode]
    cfg = default_config('fasterrcnn', ['model.base_network.architecture=resnet_v1_50',
                                        'model.network.num_classes=20', 'model.rpn.proposals.post_nms_top_n=200',
                                        'dataset.image_preprocessing.min_size=200',
                                        'dataset.image_preprocessing.max_size=320'] + over)
    wts = synth.make_weights(cfg, seed=3, profile='peaky')
    shapes = [(500, 700), (230, 260)]
    windows, scales = _tiled_windows(cfg, shapes, 240)
    eng = _engine(cfg, wts, 4, 320, 320)
    srcs = sources(shapes, False, seed=7)
    rpn_only = mode == 'rpn_only'
    nc = 1 if rpn_only else cfg.model.network.num_classes
    k = eng.max_detections
    class_max = k if rpn_only else cfg.model.rcnn.proposals.class_max_detections
    thr = 0.6 if rpn_only else 0.5
    out = eng.predict_windows(srcs, windows, scales, thr)
    ref, stats = _merge_ref(eng, windows, scales, len(shapes), nc, class_max, k, thr)
    _assert_merge(out, ref, mode)
    if mode == 'no_detections':
        assert int(out[3].sum()) == 0 and stats['candidates'] == 0
    else:
        assert stats['candidates'] > 0 and all(int(c) > 0 for c in out[3])
    # the same call again (graph replays) gives the same bytes; host -> device sources too
    assert_same(out, eng.predict_windows(on_device(srcs), windows, scales, thr), mode + ' device sources')
    eng.close()


def test_tiled_meets_the_oracle():
    """predict_tiled on a 700 x 1100 and a 1300 x 500 image at 400 px tiles; every window through the fp32 and float64
    oracle, merged by the numpy restatement, against the engine with the rule of test_gpu_photo_sizes."""
    from test_gpu_photo_sizes import oracle_pair
    cfg = default_config('fasterrcnn', ['model.base_network.architecture=resnet_v1_50', 'model.network.num_classes=20',
                                        'model.rpn.proposals.post_nms_top_n=100',
                                        'model.rcnn.proposals.min_prob_threshold=0.05',
                                        'dataset.image_preprocessing.min_size=160',
                                        'dataset.image_preprocessing.max_size=224'])
    wts = synth.make_weights(cfg, seed=0)
    shapes = [(700, 1100), (1300, 500)]
    srcs = sources(shapes, False, seed=31)
    net = PredictorNetwork(cfg, weights=wts, max_batch=4)
    net.predict_tiled(srcs, 400)                                       # runs the windows; results read below
    windows, scales = [], []
    for i, im in enumerate(srcs):
        wins, scl = net.tile_windows(im.shape, 400)
        windows += [(i,) + w for w in wins]
        scales += scl
    out = net.engine.predict_windows(srcs, windows, scales, net.merge_iou_threshold())
    net.engine.close()
    k = out[0].shape[1]
    per = {32: [], 64: []}
    for w in windows:
        ref, tru = oracle_pair(cfg, wts, _crop(srcs[w[0]], w), w[5:])
        for bits, pred in ((32, ref['classification_prediction']), (64, tru['classification_prediction'])):
            per[bits].append(pred)
    thr = net.merge_iou_threshold()
    merged = {}
    for bits, preds in per.items():
        b = np.zeros((len(windows), k, 4), np.float32)
        s = np.zeros((len(windows), k), np.float32)
        lab = np.full((len(windows), k), -1, np.int32)
        c = np.zeros((len(windows),), np.int32)
        for j, p in enumerate(preds):
            n = len(p['probs'])
            b[j, :n] = p['objects']; s[j, :n] = p['probs']; lab[j, :n] = p['labels']; c[j] = n
        wmap = [(w[1], w[2], sc[0], sc[1]) for w, sc in zip(windows, scales)]
        merged[bits] = merge_windows(b, s, lab, c, [w[0] for w in windows], wmap, len(srcs), 20,
                                     cfg.model.rcnn.proposals.class_max_detections, k, thr)
    boxes, scores, labels, counts = out
    for i in range(len(srcs)):
        r32 = dict(zip(('objects', 'probs', 'labels'), merged[32][i]))
        r64 = dict(zip(('objects', 'probs', 'labels'), merged[64][i]))
        r = _det_compare('tiles/img%d' % i, boxes[i], scores[i], labels[i], int(counts[i]), r32, r64,
                         dict(windows=sum(1 for w in windows if w[0] == i)))
        _assert_parity(r, 'tiled image %d' % i)
        assert r['detections_engine'] > 0, 'the comparison must not be vacuous'


def merge_bound(stats, nsrc, nc, class_max):
    """DESIGN section 4.2: a call with T window detections, a longest per-(source, label) list of L and G list groups
    holds at most T x (84 + 4 G + 8 words(L)) + nsrc x nc x (52 class_max + 20) + 64 KiB bytes of merge workspace;
    words(L) = ceil(L / 64) + 1 rounded up to even."""
    t, lng, g = stats['candidates'], stats['longest_list'], stats['groups']
    words = ((lng + 63) // 64 + 1) & ~1
    return t * (84 + 4 * g + 8 * words) + nsrc * nc * (52 * class_max + 20) + 65536


def test_large_photo_merge_workspace_is_bounded():
    cfg = default_config('fasterrcnn', ['model.base_network.architecture=resnet_v1_50', 'model.network.num_classes=80',
                                        'model.rcnn.proposals.min_prob_threshold=0.0'])
    wts = synth.make_weights(cfg, seed=0, profile='peaky')
    photo = sources([(4000, 6000)], False, seed=41)
    net = PredictorNetwork(cfg, weights=wts, max_batch=8)
    res = net.predict_tiled(photo, 600)
    _, _, _, counts, stats = net.engine.last_window_detections()
    # the merged detections themselves, against the restatement of the same call's window detections
    wins, scales = net.tile_windows(photo[0].shape, 600)
    windows = [(0,) + w for w in wins]
    thr = net.merge_iou_threshold()
    out = net.engine.predict_windows(photo, windows, scales, thr)
    ref, _ = _merge_ref(net.engine, windows, scales, 1, 80, 100, net.engine.max_detections, thr)
    net.engine.close()
    _assert_merge(out, ref, 'photo')
    assert int(out[3][0]) == len(res[0])
    assert len(counts) == 9 * 13 + 1 and len(res) == 1 and len(res[0]) > 0
    assert stats['candidates'] == int(counts.sum()) > 0
    bound = merge_bound(stats, 1, 80, 100)
    print('merge workspace %d bytes for %d candidates (longest list %d, %d groups); bound %d'
          % (stats['workspace_bytes'], stats['candidates'], stats['longest_list'], stats['groups'], bound))
    assert stats['workspace_bytes'] <= bound
    # a [sources x classes][windows x class_max] layout would need 1.4 GB for its bit mask alone
    uniform = 80 * (118 * 100) * (((118 * 100 + 63) // 64 + 1) & ~1) * 8
    assert stats['workspace_bytes'] * 10 < uniform
    for o in res[0]:
        x1, y1, x2, y2 = o['bbox']
        assert -1 <= x1 <= x2 <= 6000 and -1 <= y1 <= y2 <= 4000
