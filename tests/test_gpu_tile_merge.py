"""The cross-window merge of sliced prediction (`-m gpu`) at the sizes and settings large photos take it, byte for byte
against the numpy restatement (tests/tile_merge_ref.py).

* Stand-alone merge (``lumi_op_window_merge``, the code ``lumi_predict_windows`` runs after its window forwards) on
  built candidate lists: single lists at the edges of the NMS paths (4 095 / 4 096 staged, 12 672 staged, 12 673 and
  20 000 unstaged), three lists of 4 096 and of 6 000 in one group (two-phase, kept boxes on both sides of its first
  2 048 candidates), long lists grouped with shorter ones (padded slots), and the content edges: one object seen by
  several windows, IoU at the threshold and within 2^-20 of it, zero-area boxes, unequal non-power-of-two scales with
  offsets up to 6 000, class_max and total_max cuts on score ties, an empty source.  Every case checks the list
  grouping against the restatement of plan_window_merge and prints the NMS path of each group.  IoU thresholds 0,
  0.5, 1 and +inf at SM budgets 1, 2, 16, 114 and the whole device.
* Engine (``predict_windows``): RPN-only lists long enough for the unstaged and the two-phase path, SSD tiles with a
  non-square whole-image window (s_y != s_x) against the restatement and the fp32 / float64 oracle, the threshold and
  SM-budget settings, and one engine reused across a photo call, a smaller call and the photo call again.
"""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import gpu_ops as G
from luminoth_b200 import default_config, synth
from luminoth_b200.predicting import PredictorNetwork
from test_gpu_resize_input import sources
from test_gpu_tiles import _assert_merge, _crop, _engine, _merge_ref
from tile_merge_ref import list_lengths, merge_windows, nms_path, plan_groups

STAGED, TWO_PHASE, UNSTAGED = 0, 1, 2
PATH_NAMES = {STAGED: 'staged', TWO_PHASE: 'two-phase', UNSTAGED: 'unstaged'}
THRESHOLDS = [0.0, 0.5, 1.0, float('inf')]
SM_BUDGETS = [1, 2, 16, 114, 0]                  # 0: the whole device
SCALES = [(0.37, 1.713), (1.713, 0.37), (0.6, 2.5), (3.1, 0.77), (1.0, 1.0), (0.5, 0.25)]


class Dets:
    """Window detections built on the host: rows per window (kmax slots), window -> source, window -> map."""

    def __init__(self, kmax):
        self.kmax = kmax
        self.b, self.s, self.l, self.c, self.src, self.map = [], [], [], [], [], []

    def add(self, src, wmap, boxes, scores, labels):
        """One window per kmax rows of (boxes, scores, labels), all of source src mapped by wmap = (y0, x0, s_y, s_x)."""
        n = len(scores)
        for a in range(0, max(n, 1), self.kmax):
            m = min(self.kmax, n - a)
            b = np.zeros((self.kmax, 4), np.float32)
            s = np.zeros((self.kmax,), np.float32)
            lab = np.full((self.kmax,), -1, np.int32)
            b[:m] = boxes[a:a + m]; s[:m] = scores[a:a + m]; lab[:m] = labels[a:a + m]
            self.b.append(b); self.s.append(s); self.l.append(lab); self.c.append(m)
            self.src.append(src); self.map.append(tuple(np.float32(v) for v in wmap))
        return self

    def arrays(self):
        return (np.stack(self.b), np.stack(self.s), np.stack(self.l), np.asarray(self.c, np.int32),
                np.asarray(self.src, np.int32), np.asarray(self.map, np.float32))


def _boxes(rng, n, extent=3000.0, size=120.0):
    x, y = rng.uniform(0, extent, n), rng.uniform(0, extent, n)
    w, h = rng.uniform(1, size, n), rng.uniform(1, size, n)
    return np.stack([x, y, x + w, y + h], 1).astype(np.float32)


def _scores(rng, n, levels=None):
    """Scores in (0, 1]; with `levels` only that many distinct values, so that ties are everywhere."""
    if levels:
        return (rng.randint(1, levels + 1, n) / np.float32(levels)).astype(np.float32)
    return rng.uniform(0.01, 1.0, n).astype(np.float32)


def _wmap(rng):
    sy, sx = SCALES[rng.randint(len(SCALES))]
    return (float(rng.randint(0, 6001)), float(rng.randint(0, 6001)), sy, sx)


def _list(d, rng, src, label, n, **kw):
    """n candidates of one (source, label) list, spread over windows with random maps."""
    for a in range(0, n, d.kmax):
        m = min(d.kmax, n - a)
        d.add(src, _wmap(rng), _boxes(rng, m, **kw), _scores(rng, m, 64), np.full(m, label, np.int32))
    return d


def _check(d, nsrc, nc, class_max, total_max, thr, sm=0, tag='', expect_paths=None, ref=None):
    """The op against the restatement (or `ref`, its result), byte for byte; the grouping against plan_groups.
    Returns the groups, their NMS paths and the output counts."""
    b, s, lab, c, src, wmap = d.arrays()
    ob, os_, ol, oc, stats = G.window_merge(b, s, lab, c, src, wmap, nsrc, nc, class_max, total_max, thr, sm)
    if ref is None:
        ref = merge_windows(b, s, lab, c, src, wmap, nsrc, nc, class_max, total_max, thr)
    _assert_merge((ob, os_, ol, oc), ref, tag)
    for i in range(nsrc):                                   # rows past the count: the empty detection
        k = int(oc[i])
        assert (ol[i, k:] == -1).all() and (os_[i, k:] == 0).all() and (ob[i, k:] == 0).all(), tag
    lengths = list_lengths(lab, c, src, nsrc, nc)
    groups = plan_groups(lengths)
    assert stats['candidates'] == int(c.sum()) == int(lengths.sum()), tag
    assert stats['longest_list'] == int(lengths.max(initial=0)), tag
    assert stats['groups'] == len(groups), '%s: %d groups, restatement %s' % (tag, stats['groups'], groups)
    paths = []
    for p, cap in groups:
        path = G.nms_path(p, cap, thr)
        assert path == nms_path(p, cap, thr), (tag, p, cap, thr)
        paths.append(path)
    if expect_paths is not None:
        assert paths == expect_paths, '%s: groups %s took %s' % (tag, groups, [PATH_NAMES[q] for q in paths])
    return groups, paths, oc


def _report(tag, groups, paths):
    print('%s: %s' % (tag, ', '.join('%d x %d %s' % (p, cap, PATH_NAMES[q]) for (p, cap), q in zip(groups, paths))))


# ---- path boundaries on built lists
def _path_case(name):
    rng = np.random.RandomState(sum(map(ord, name)))
    d = Dets(1000)
    if name.startswith('single_'):
        _list(d, rng, 0, 1, int(name[7:]))
        return d, 1, 3
    if name == 'three_4096':
        for src in range(3):
            _list(d, rng, src, 0, 4096)
        return d, 3, 1
    if name == 'three_6000':
        for lab in range(3):
            _list(d, rng, 0, lab, 6000)
        return d, 1, 3
    if name == 'long_with_short':        # one 6 000 list, then 40 lists of 10 to 60 padded to 60 in one group
        _list(d, rng, 0, 0, 6000)
        lens = [60] + list(rng.randint(10, 61, 39))
        for lab, n in enumerate(lens):
            _list(d, rng, 1 + lab % 2, lab // 2, int(n))
        return d, 3, 20
    if name == 'padded_two_phase':       # 5 000, 4 500 and 4 200 in one two-phase group, then 30 short lists
        for lab, n in enumerate([5000, 4500, 4200]):
            _list(d, rng, 0, lab, n)
        for k in range(30):
            _list(d, rng, 1 + k // 10, 3 + k % 10, 50)
        return d, 4, 13
    raise ValueError(name)


PATH_CASES = [('single_4095', [STAGED]), ('single_4096', [STAGED]), ('single_12672', [STAGED]),
              ('single_12673', [UNSTAGED]), ('single_20000', [UNSTAGED]), ('three_4096', [TWO_PHASE]),
              ('three_6000', [TWO_PHASE]), ('long_with_short', [STAGED, STAGED]),
              ('padded_two_phase', [TWO_PHASE, STAGED])]


@pytest.mark.parametrize('name,paths', PATH_CASES, ids=[c[0] for c in PATH_CASES])
def test_merge_path_boundaries(name, paths):
    d, nsrc, nc = _path_case(name)
    groups, got, oc = _check(d, nsrc, nc, 20000, 20000, 0.5, tag=name, expect_paths=paths)
    _report(name, groups, got)
    assert int(oc.sum()) > 0
    if TWO_PHASE in got:
        # the two-phase path resolves the first 2 048 candidates (R1) of a list, then the rest: the longest list
        # must keep boxes on both sides of R1 in score order, or the second phase went unchecked
        b, s, lab, c, src, wmap = d.arrays()
        ref = merge_windows(b, s, lab, c, src, wmap, nsrc, nc, 20000, 20000, 0.5)
        kept = {}
        for i, (rb, rs, rl) in enumerate(ref):
            for lb in np.unique(rl):
                kept[(i, int(lb))] = rs[rl == lb]
        lengths = list_lengths(lab, c, src, nsrc, nc)
        p = int(np.argmax(lengths))
        cand = np.sort(np.concatenate([s[k, :c[k]][lab[k, :c[k]] == p % nc] for k in range(len(c))
                                       if src[k] == p // nc]))[::-1]
        ks = kept[(p // nc, p % nc)]
        assert (ks > cand[2048]).any() and (ks < cand[2048]).any(), 'kept boxes on one side of R1 only'


# ---- content edges
def _content_case():
    rng = np.random.RandomState(11)
    d = Dets(64)
    # source 0: one object seen by three windows -- identical source boxes (IoU 1), equal scores -- among random
    # boxes of six labels at unequal non-power-of-two scales, scores on 16 levels (ties within and across labels)
    obj = np.array([[100, 40, 180, 90]], np.float32)                         # source pixels
    for y0, x0 in [(0, 0), (16, 8), (32, 40)]:
        sy, sx = 0.5, 0.25
        wb = np.array([[(obj[0, 0] - x0) * sx, (obj[0, 1] - y0) * sy, (obj[0, 2] - x0) * sx, (obj[0, 3] - y0) * sy]],
                      np.float32)
        n = 40
        b = np.concatenate([wb, _boxes(rng, n - 1, 400.0, 80.0)])
        s = np.concatenate([[np.float32(0.875)], _scores(rng, n - 1, 16)]).astype(np.float32)
        lab = np.concatenate([[2], rng.randint(0, 6, n - 1)]).astype(np.int32)
        d.add(0, (y0, x0, sy, sx), b, s, lab)
    for _ in range(12):
        n = int(rng.randint(20, 65))
        d.add(0, _wmap(rng), _boxes(rng, n, 600.0, 150.0), _scores(rng, n, 16), rng.randint(0, 6, n).astype(np.int32))
    # source 1: no candidates (one window without detections)
    d.add(1, (5, 7, 0.37, 1.713), np.zeros((0, 4), np.float32), np.zeros(0, np.float32), np.zeros(0, np.int32))
    # source 2, window at the origin with scale 1 (coordinates exact): IoU exactly 0.5 -- (0,0,2,1) against (0,0,1,1)
    # -- and 1 / a for a within 2^-20 of 2 on both sides, each pair on its own rows; zero-area boxes; label 7 with
    # 300 separated boxes, more than class_max survive
    rows = []
    eps = 2.0 ** -22
    for i, a in enumerate([2.0, 2.0 - eps, 2.0 + eps, 2.0 - 4 * eps, 2.0 + 4 * eps, 2.0 - 2 * eps, 2.0 + 2 * eps]):
        y = 10.0 * i
        rows.append(((0.0, y, np.float32(a), y + 1), 0.9 - 0.01 * i, 4))
        rows.append(((0.0, y, 1.0, y + 1), 0.85 - 0.01 * i, 4))
    for i in range(6):                                                       # zero width, zero height, a point
        x = 500.0 + 10 * (i // 3)
        rows.append([((x, 0.0, x, 5.0), 0.7, 5), ((x, 0.0, x + 5, 0.0), 0.7, 5), ((x, 3.0, x, 3.0), 0.6, 5)][i % 3])
    rows.append(((500.0, 0.0, 500.0, 5.0), 0.7, 5))                         # the same zero-area box again
    d.add(2, (0, 0, 1.0, 1.0), np.array([r[0] for r in rows], np.float32), np.array([r[1] for r in rows], np.float32),
          np.array([r[2] for r in rows], np.int32))
    n = 300
    x = (np.arange(n) % 30) * 40.0
    y = (np.arange(n) // 30) * 40.0 + 1000
    b = np.stack([x, y, x + 30, y + 30], 1).astype(np.float32)
    d.add(2, (1000.0, 6000.0, 1.713, 0.37), b, _scores(rng, n, 8), np.full(n, 7, np.int32))
    return d, 3, 8


def test_merge_content_edges():
    d, nsrc, nc = _content_case()
    # class_max 50 cuts label 7 (300 survivors) and the busy labels of source 0; total_max 130 cuts source 0 inside
    # its run of 0.75 scores, which spans all six labels
    groups, paths, oc = _check(d, nsrc, nc, 50, 130, 0.5, tag='content')
    _report('content', groups, paths)
    assert int(oc[1]) == 0 and int(oc[0]) == 130 and int(oc[2]) > 50
    b, s, lab, c, src, wmap = d.arrays()
    ref = merge_windows(b, s, lab, c, src, wmap, nsrc, nc, 50, 130, 0.5)
    # the object seen by three windows is kept once; IoU exactly 0.5 keeps both boxes of that pair
    rb, rs, rl = ref[0]
    assert ((rb == np.float32([100, 40, 180, 90])).all(1)).sum() == 1
    rb, rs, rl = ref[2]
    assert (rl == 7).sum() == 50
    pairs = rb[rl == 4]
    assert len(pairs) == 7 + 4           # a = 2 and a > 2 (IoU <= 0.5) keep both boxes, a < 2 suppresses one
    assert (rl == 5).sum() == 7          # zero-area boxes never suppress and are never suppressed


@pytest.mark.parametrize('case', ['content', 'three_4096'])
def test_merge_thresholds_and_sm_budgets(case):
    d, nsrc, nc = _content_case() if case == 'content' else _path_case('three_4096')
    cm, tm = (50, 130) if case == 'content' else (5000, 5000)
    b, s, lab, c, src, wmap = d.arrays()
    for thr in THRESHOLDS:
        ref = merge_windows(b, s, lab, c, src, wmap, nsrc, nc, cm, tm, thr)
        seen = None
        for sm in SM_BUDGETS:
            tag = '%s thr %g sm %d' % (case, thr, sm)
            groups, paths, oc = _check(d, nsrc, nc, cm, tm, thr, sm, tag=tag, ref=ref)
            seen = seen or (groups, paths)
        _report('%s thr %g' % (case, thr), *seen)


@pytest.mark.parametrize('what,change', [
    ('count above kmax', lambda a: a['c'].__setitem__(0, 5)),
    ('negative count', lambda a: a['c'].__setitem__(1, -1)),
    ('label above nc', lambda a: a['l'].__setitem__((0, 1), 3)),
    ('negative label', lambda a: a['l'].__setitem__((1, 0), -1)),
    ('source out of range', lambda a: a['src'].__setitem__(1, 2)),
    ('negative threshold', lambda a: a.__setitem__('thr', -0.5)),
    ('NaN threshold', lambda a: a.__setitem__('thr', float('nan'))),
])
def test_merge_rejects_bad_inputs(what, change):
    a = dict(b=np.zeros((2, 4, 4), np.float32), s=np.full((2, 4), 0.5, np.float32),
             l=np.array([[0, 1, 2, -1], [1, 2, -1, -1]], np.int32), c=np.array([3, 2], np.int32),
             src=np.array([0, 1], np.int32), thr=0.5)
    a['b'][..., 2:] = 10
    G.window_merge(a['b'], a['s'], a['l'], a['c'], a['src'], [(0, 0, 1, 1)] * 2, 2, 3, 4, 4, a['thr'])   # valid
    change(a)
    with pytest.raises(ValueError, match='window merge'):
        G.window_merge(a['b'], a['s'], a['l'], a['c'], a['src'], [(0, 0, 1, 1)] * 2, 2, 3, 4, 4, a['thr'])


# ---- through the engine
def _frcnn(over, seed=0):
    cfg = default_config('fasterrcnn', ['model.base_network.architecture=resnet_v1_50'] + over)
    return cfg, synth.make_weights(cfg, seed=seed)


def test_rpn_only_long_lists_take_the_unstaged_and_two_phase_paths():
    """RPN-only windows (kmax = post_nms_top_n, one label) with stream-K off, so that identical windows give
    identical detections: repeats of one window make one list past 12 672 (unstaged) and, over three sources, three
    equal lists of >= 4 096 in one group (two-phase)."""
    cfg, wts = _frcnn(['model.network.with_rcnn=false', 'model.rpn.proposals.post_nms_top_n=2000'], seed=2)
    eng = _engine(cfg, wts, 1, 600, 800)          # one window per forward: every window runs the same kernels
    eng.set_conv_streamk('off')
    thr = 0.7
    srcs = sources([(600, 800)], False, seed=17) * 3           # three sources holding the same image
    win = (0, 0, 600, 800, 600, 800)
    eng.predict_windows(srcs[:1], [(0,) + win], [(1.0, 1.0)], thr)
    per = int(eng.last_window_detections()[3][0])
    assert per >= 500, 'a window gives %d proposals; the lists would need too many windows' % per
    for name, nsrc, need, path in (('unstaged', 1, 12673, UNSTAGED), ('two-phase', 3, 4096, TWO_PHASE)):
        reps = math.ceil(need / per)
        windows = [(i,) + win for i in range(nsrc) for _ in range(reps)]
        scales = [(1.0, 1.0)] * len(windows)
        out = eng.predict_windows(srcs[:nsrc], windows, scales, thr)
        ref, stats = _merge_ref(eng, windows, scales, nsrc, 1, eng.max_detections, eng.max_detections, thr)
        wb, ws, wl, wc, _ = eng.last_window_detections()
        assert (wc == per).all() and (wb == wb[:1]).all() and (ws == ws[:1]).all(), 'windows differ'
        _assert_merge(out, ref, name)
        groups = plan_groups(list_lengths(wl, wc, [w[0] for w in windows], nsrc, 1))
        assert groups == [(nsrc, reps * per)] and stats['groups'] == 1 and stats['longest_list'] == reps * per
        got = G.nms_path(nsrc, reps * per, thr)
        print('rpn-only %s: %d x %d candidates, path %s' % (name, nsrc, reps * per, PATH_NAMES[got]))
        assert got == path
    eng.close()


def test_ssd_tiles_non_square_whole_image():
    """SSD predict_tiled on a 300 x 600 image at 300 px tiles: three tiles at scale 1 and the whole image at
    (s_y, s_x) = (1, 0.5).  The merge equals the restatement byte for byte and meets the fp32 and float64 oracle run
    per window and merged by the restatement, with the rule of test_tiled_meets_the_oracle."""
    from oracle import ssd as ossd
    from oracle import tf_ops as T
    from test_gpu_baseline_configs import _assert_parity, _det_compare
    from test_ssd_config_host import ssd_cfg
    cfg = ssd_cfg(300, 300)
    cfg['model']['proposals']['min_prob_threshold'] = 0.2
    wts = synth.make_weights(cfg, seed=5)
    srcs = sources([(300, 600)], False, seed=23)
    net = PredictorNetwork(cfg, weights=wts, max_batch=4)
    wins, scales = net.tile_windows(srcs[0].shape, 300)
    assert scales[-1][0] != scales[-1][1], 'the whole-image window must scale y and x differently'
    windows = [(0,) + w for w in wins]
    thr = net.merge_iou_threshold()
    res = net.predict_tiled(srcs, 300)
    out = net.engine.predict_windows(srcs, windows, scales, thr)
    k = net.engine.max_detections
    nc = cfg['model']['network']['num_classes']
    cm = cfg['model']['proposals']['class_max_detections']
    ref, stats = _merge_ref(net.engine, windows, scales, 1, nc, cm, k, thr)
    net.engine.close()
    _assert_merge(out, ref, 'ssd tiles')
    assert len(res[0]) == int(out[3][0]) > 0, 'the comparison must not be vacuous'
    merged = {}
    for bits, dt in ((32, np.float32), (64, np.float64)):
        b = np.zeros((len(windows), k, 4), np.float32)
        s = np.zeros((len(windows), k), np.float32)
        lab = np.full((len(windows), k), -1, np.int32)
        c = np.zeros((len(windows),), np.int32)
        for j, w in enumerate(windows):
            img = T.resize_bilinear(_crop(srcs[0], w).astype(np.float32), 300, 300)
            p = ossd.forward(img, wts, cfg, dtype=dt)['classification_prediction']
            n = len(p['probs'])
            b[j, :n] = p['objects']; s[j, :n] = p['probs']; lab[j, :n] = p['labels']; c[j] = n
        wmap = [(w[1], w[2], sc[0], sc[1]) for w, sc in zip(windows, scales)]
        merged[bits] = merge_windows(b, s, lab, c, [0] * len(windows), wmap, 1, nc, cm, k, thr)[0]
    boxes, scores, labels, counts = out
    r = _det_compare('ssd_tiles', boxes[0], scores[0], labels[0], int(counts[0]),
                     dict(zip(('objects', 'probs', 'labels'), merged[32])),
                     dict(zip(('objects', 'probs', 'labels'), merged[64])), dict(windows=len(windows)))
    _assert_parity(r, 'ssd tiles')


def _settings_call():
    cfg, wts = _frcnn(['model.network.num_classes=20', 'model.rpn.proposals.post_nms_top_n=200',
                       'model.rcnn.proposals.min_prob_threshold=0.0', 'dataset.image_preprocessing.min_size=200',
                       'dataset.image_preprocessing.max_size=320'], seed=3)
    from test_gpu_tiles import _tiled_windows
    shapes = [(500, 700), (230, 260)]
    windows, scales = _tiled_windows(cfg, shapes, 240)
    return cfg, wts, shapes, windows, scales


def test_engine_merge_thresholds_and_sm_budgets():
    cfg, wts, shapes, windows, scales = _settings_call()
    eng = _engine(cfg, wts, 4, 320, 320)
    srcs = sources(shapes, False, seed=7)
    nc, cm, k = 20, cfg.model.rcnn.proposals.class_max_detections, eng.max_detections
    for sm in SM_BUDGETS:
        eng.set_sm_limit(sm)
        for thr in THRESHOLDS:
            out = eng.predict_windows(srcs, windows, scales, thr)
            ref, stats = _merge_ref(eng, windows, scales, len(shapes), nc, cm, k, thr)
            _assert_merge(out, ref, 'engine thr %g sm %d' % (thr, sm))
            assert stats['candidates'] > 0 and int(out[3].min()) > 0
    eng.close()


def test_merge_scratch_reused_across_calls():
    """One engine: a 4000 x 6000 photo at 600 px tiles, then one 600 x 600 window of it (its labels a strict subset
    of the photo's), then the photo again.  Each call equals the restatement of its own window detections and the
    same call on a fresh engine; the second call is where kept counts or rows left by the first would show."""
    cfg, wts = _frcnn(['model.network.num_classes=20', 'model.rcnn.proposals.min_prob_threshold=0.1'])
    photo = sources([(4000, 6000)], False, seed=41)
    net = PredictorNetwork(cfg, weights=wts, max_batch=8)
    wins, scales = net.tile_windows(photo[0].shape, 600)
    big = ([(0,) + w for w in wins], scales)
    small = ([(0,) + wins[14]], [scales[14]])
    thr = net.merge_iou_threshold()
    nc, cm = 20, cfg.model.rcnn.proposals.class_max_detections

    def run(eng, call, tag):
        out = eng.predict_windows(photo, call[0], call[1], thr)
        ref, stats = _merge_ref(eng, call[0], call[1], 1, nc, cm, eng.max_detections, thr)
        _assert_merge(out, ref, tag)
        _, _, wl, wc, _ = eng.last_window_detections()
        return out, set(int(v) for k in range(len(wc)) for v in wl[k, :wc[k]]), stats

    eng = net.engine
    eng.set_conv_streamk('off')                # a window's detections do not depend on the chunk it runs in
    first, big_labels, stats = run(eng, big, 'photo')
    second, small_labels, _ = run(eng, small, 'window after the photo')
    assert small_labels and small_labels < big_labels, (small_labels, big_labels)
    third, _, _ = run(eng, big, 'photo again')
    eng.close()
    print('photo: %d candidates, longest list %d, %d groups, %d labels; window: %d labels'
          % (stats['candidates'], stats['longest_list'], stats['groups'], len(big_labels), len(small_labels)))
    for call, got in ((big, [first, third]), (small, [second])):
        fresh = PredictorNetwork(cfg, weights=wts, max_batch=8).engine
        fresh.set_conv_streamk('off')
        want = fresh.predict_windows(photo, call[0], call[1], thr)
        fresh.close()
        for g in got:
            for a, b in zip(g, want):
                np.testing.assert_array_equal(a, b)
