"""The three NMS paths of run_nms and the batched proposal / detection chains at the engine's layouts, bit for bit
against the oracle (`-m gpu`, needs an H100).

run_nms takes the staged one-phase scan, the two-phase NMS (>= 3 lists of >= 4096 candidates: phase 1 resolves the
first 2048 candidates, a pre-filter tests every later one against the phase-1 keepers, the survivors are compacted and
resolved by a second mask + scan that appends through an index map) or the unstaged scan (lists too long for the
staged scan's shared memory).  Every case first asserts which path it runs; the two-phase cases also measure, from the
oracle, k1 (keepers among the first 2048 candidates) and the number of later candidates that survive them, and assert
the conditions the case was built for, so that a case cannot quietly stop reaching phase 2.

Keep sets, order, labels and probabilities must be identical; boxes too, because every case decodes with dw = dh = 0
(exp(0) == 1 on both sides).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import tf_ops as T
from oracle import fasterrcnn as ofr
from oracle import ssd as ossd
from oracle.anchors import fasterrcnn_anchors, ssd_anchors
from oracle.bbox import decode, clip_boxes

R1 = 2048                                # candidates of phase 1 (NMS_LAZY_R1 in postproc.cu)
STAGED, TWO_PHASE, UNSTAGED = 0, 1, 2
F32 = np.float32


def ops():
    import gpu_ops
    return gpu_ops


def _tf(b):
    return b[:, [1, 0, 3, 2]]


def oracle_keep(boxes, thr, max_out):
    """T.non_max_suppression on boxes already in score order (x1, y1, x2, y2)."""
    n = boxes.shape[0]
    return T.non_max_suppression(_tf(boxes), np.arange(n, 0, -1).astype(F32), max_out, float(thr))


def two_phase_stats(boxes, thr, max_out):
    """(k1, survivors): the phase-1 keepers among the first R1 candidates and the later candidates none of them
    suppresses (the lists phase 2 resolves; nothing reaches phase 2 once k1 == max_out)."""
    head = oracle_keep(boxes[:R1], thr, max_out)
    k1 = len(head)
    tail = boxes[R1:]
    if k1 >= max_out or tail.shape[0] == 0:
        return k1, np.zeros((0,), np.int64)
    dead = np.zeros(tail.shape[0], bool)
    tt = _tf(tail)
    for i in head:
        dead |= T.iou_tf(_tf(boxes[i:i + 1])[0], tt) > F32(thr)
    return k1, R1 + np.flatnonzero(~dead)


# ---------------------------------------------------------------- two-phase NMS
CAP = 12672                              # the longest list the staged scan (and so the two-phase NMS) takes
NVALID = [1, 2047, 2048, 2049, 4095, 4096, 12000, 12672]
THR = F32(0.7)
SZ = 80                                  # cluster box side (a multiple of 8: exact IoU ratios below)


def _clustered_list(seed, n, clusters):
    """A clustered head: the first 2048 candidates are jittered copies of `clusters` boxes (IoU > 0.8 with the exact
    box, which comes first), so k1 is about `clusters`.  Then a tail of: copies killed by a phase-1 keeper, boxes at
    IoU exactly 0.7 = 4480 / 6400 against a keeper (80 x 56 inside an 80 x 80 keeper), fresh boxes in greedy chains
    (A suppresses B, B would suppress C, C is kept), duplicates, zero-area boxes, and exact-0.7 pairs among the fresh
    boxes, which the phase-2 mask decides.  Exact-0.7 pairs also sit inside the head (phase-1 mask), and the last head
    candidate is an isolated box, so phase 1 has to resolve all 2048."""
    rng = np.random.default_rng(seed)
    per_row = 48
    centres = np.array([[(c % per_row) * 2 * SZ, (c // per_row) * 2 * SZ] for c in range(clusters)], F32)
    box = lambda c, w=SZ, h=SZ: [centres[c, 0], centres[c, 1], centres[c, 0] + w, centres[c, 1] + h]
    head, seen = [], set()
    thr_in_head = set(range(0, clusters, 3))
    while len(head) < R1:
        u = rng.random()
        if u < 0.01:                                                   # zero-area: never suppresses, always kept
            x = float(rng.integers(0, 4000)); head.append([x, -500.0, x, -400.0]); continue
        c = int(rng.integers(0, clusters))
        if c not in seen:
            seen.add(c); head.append(box(c))
            if c in thr_in_head:
                head.append(box(c, SZ, 56))                             # IoU == RN(0.7) with its keeper
            continue
        if u < 0.03:
            head.append(box(c)); continue                              # duplicate of the keeper
        j = rng.uniform(-2, 2, 4).astype(F32)
        head.append([v + d for v, d in zip(box(c), j)])
    head = head[:R1]
    head[R1 - 1] = [-3000.0 - 200 * seed, -3000.0, -2900.0 - 200 * seed, -2900.0]   # the last phase-1 candidate: kept
    keepers = sorted(seen)
    items = []                                                         # tail blocks, shuffled below
    for c in keepers:
        if c not in thr_in_head:
            items.append([box(c, SZ, 56)])                             # at thr: survives f32(0.7), killed one ulp lower
            items.append([box(c, 56, SZ)])
    for _ in range(n):
        c = keepers[int(rng.integers(0, len(keepers)))]
        j = rng.uniform(-2, 2, 4).astype(F32)
        items.append([[v + d for v, d in zip(box(c), j)]])             # killed by a phase-1 keeper
    fresh = 0
    for row in range(n):                                               # one block per row, far from the clusters
        if fresh >= n:
            break
        y, x = 160.0 * row, 20000.0 + 1000.0 * float(rng.integers(0, 60))
        kind = rng.random()
        if kind < 0.6:                                                 # greedy chain: shift 12 on width 100
            L = int(rng.integers(2, 9))
            items.append([[x + 12.0 * k, y, x + 12.0 * k + 100.0, y + 100.0] for k in range(L)])
        elif kind < 0.8:                                               # duplicate pair
            items.append([[x, y, x + 90.0, y + 70.0]] * 2)
        elif kind < 0.9:                                               # exact-0.7 pair decided in phase 2
            items.append([[x, y, x + SZ, y + SZ], [x, y, x + SZ, y + 56.0]])
        else:
            items.append([[x, y, x, y + 50.0]])                        # zero area
        fresh += len(items[-1])
    order = rng.permutation(len(items))
    tail = [b for i in order for b in items[i]]
    out = np.array(head + tail, F32)[:n] if n > R1 else np.array(head, F32)[:n]
    return out


def _two_phase_lists():
    lists = []
    for p, n in enumerate(NVALID):
        clusters = 300 if n == 12000 else 20 + 7 * p                  # one list with k1 > 256
        lists.append(_clustered_list(100 + p, max(n, 1), clusters)[:n])
    return lists


def _pack(lists, cap, rng):
    """[P, cap, 4] with rows past nvalid filled with copies of real boxes: they must never be read."""
    P = len(lists)
    out = np.empty((P, cap, 4), F32)
    for p, b in enumerate(lists):
        out[p, :len(b)] = b
        pad = cap - len(b)
        if pad:
            out[p, len(b):] = lists[-1][rng.integers(0, len(lists[-1]), pad)]
    return out


@pytest.fixture(scope='module')
def two_phase_case():
    lists = _two_phase_lists()
    ref = {}
    for thr in (THR, np.nextafter(THR, F32(0)), np.nextafter(THR, F32(1))):
        ref[float(thr)] = [oracle_keep(b, thr, len(b)) for b in lists]
    return lists, ref


def test_two_phase_lists_reach_phase_2(two_phase_case):
    """The design conditions of the two-phase lists, measured on the oracle."""
    lists, ref = two_phase_case
    stats = {}
    for b in lists:
        k1, surv = two_phase_stats(b, THR, len(b))
        stats[len(b)] = (k1, len(surv))
        print('two-phase list nvalid %5d: k1 %4d, survivors %5d, kept %5d' % (len(b), k1, len(surv),
                                                                           len(ref[float(THR)][NVALID.index(len(b))])))
    for n in (4095, 4096, 12000, 12672):
        assert stats[n][1] > 0, n
    assert stats[12000][0] > 256                        # the pre-filter's keeper loop runs more than one 256-chunk
    assert max(s for _, s in stats.values()) > 1024     # the compaction loop iterates; phase 2 spans many 64-chunks
    assert min(stats[n][0] for n in (4095, 4096, 12672)) < 100     # a small k1 behind a heavily overlapping head
    # every suppression kind happens in the tail: exact-threshold boxes flip with one ulp of the threshold
    lo = float(np.nextafter(THR, F32(0)))
    assert any(len(ref[lo][i]) < len(ref[float(THR)][i]) for i in range(len(lists)))


def _max_out_cases(lists):
    """max_out values of the batched calls: no limit; k1 of the 12 672 list (phase 2 appends nothing); and k1 + 100
    of the 4096 list, which ends inside a phase-2 64-chunk."""
    k1_full, _ = two_phase_stats(lists[-1], THR, CAP)
    k1_mid, surv = two_phase_stats(lists[5], THR, CAP)
    return [CAP, k1_full, k1_mid + 100], k1_full, (k1_mid, surv)


def test_two_phase_nms_matches_oracle_and_one_phase(two_phase_case):
    lists, ref = two_phase_case
    P = len(lists)
    assert ops().nms_path(P, CAP, THR) == TWO_PHASE
    assert ops().nms_path(1, CAP, THR) == STAGED
    rng = np.random.default_rng(5)
    boxes = _pack(lists, CAP, rng)
    nvalid = [len(b) for b in lists]
    max_outs, k1_full, (k1_mid, surv_mid) = _max_out_cases(lists)
    full = ref[float(THR)][-1]
    assert len(full) > k1_full                          # the 12 672 list has phase-2 keepers that max_out = k1 cuts
    mid = ref[float(THR)][5]
    assert len(mid) > k1_mid + 100
    last = mid[k1_mid + 99]                             # the max_out-th keeper is a phase-2 candidate ...
    pos = int(np.searchsorted(surv_mid, last))
    assert surv_mid[pos] == last and pos % 64 != 63 and pos + 1 < len(surv_mid)   # ... in the middle of a chunk
    for thr, keeps in ref.items():
        for max_out in max_outs:
            got = ops().nms_batched(boxes, nvalid, thr, max_out)
            for p in range(P):
                np.testing.assert_array_equal(got[p], keeps[p][:max_out],
                                              err_msg='two-phase, nvalid %d thr %r max_out %d' % (nvalid[p], thr, max_out))
        for p in range(P):                              # the same list alone: one-phase staged scan
            one = ops().nms_batched(boxes[p:p + 1], nvalid[p:p + 1], thr, CAP)[0]
            np.testing.assert_array_equal(one, keeps[p], err_msg='one-phase, nvalid %d thr %r' % (nvalid[p], thr))


# ---------------------------------------------------------------- unstaged scan
def _dense_boxes(seed, n):
    rng = np.random.default_rng(seed)
    c = rng.uniform(0, 900, (n, 2)); s = rng.uniform(20, 200, (n, 2))
    b = np.concatenate([c, c + s], 1).astype(F32)
    b[7] = b[6]; b[11] = [10, 10, 10, 50]              # duplicate + zero-area box
    return b


@pytest.fixture(scope='module')
def unstaged_refs():
    refs = {}
    for n in (12672, 12673, 13000, 20000):
        b = _dense_boxes(n, n)
        for thr in (0.5, 0.7):
            refs[(n, thr)] = (b, oracle_keep(b, thr, n))
    return refs


@pytest.mark.parametrize('n', [12672, 12673, 13000, 20000])
@pytest.mark.parametrize('thr', [0.5, 0.7])
def test_unstaged_scan_matches_oracle(unstaged_refs, n, thr):
    b, ref = unstaged_refs[(n, thr)]
    assert ops().nms_path(1, n, thr) == (STAGED if n == 12672 else UNSTAGED)
    assert len(ref) > 2000                              # max_out 2000 cuts the list
    for max_out in (2000, n):
        np.testing.assert_array_equal(ops().nms_sorted(b, thr, max_out), ref[:max_out], err_msg='max_out %d' % max_out)


def test_unstaged_scan_batched_above_the_staged_bound(unstaged_refs):
    """Three lists above the staged bound: no two-phase path, still exact."""
    n = 13000
    assert ops().nms_path(3, n, 0.7) == UNSTAGED
    b13, ref13 = unstaged_refs[(13000, 0.7)]
    b12, ref12 = unstaged_refs[(12673, 0.7)]
    b20 = unstaged_refs[(20000, 0.7)][0][:12800]
    ref20 = oracle_keep(b20, 0.7, n)
    lists, refs = [b13, b12, b20], [ref13, ref12, ref20]
    got = ops().nms_batched(_pack(lists, n, np.random.default_rng(3)), [len(x) for x in lists], 0.7, n)
    for g, r in zip(got, refs):
        np.testing.assert_array_equal(g, r)


# ---------------------------------------------------------------- batched RPN at the engine's layout
SCORE_ULPS = 4          # fused softmax (expf) vs T.softmax (numpy exp): measured bound, in ulps of the score
M_LATTICE = 1 << 18     # target probabilities (k + 1/2) / M: neighbours >= 1/M apart, far more than SCORE_ULPS


def _rpn_inputs(seed, nimg, fh, fw, A=12, ties=True):
    """The engine's fused head [nimg][cells][6A]: logits of anchor a at 2a (background) and 2a + 1, deltas at 2A + 4a
    with dw = dh = 0.  Foreground probabilities sit on a lattice whose spacing dwarfs the softmax's rounding, so the
    selection and order cannot depend on expf vs numpy exp; tie groups use exactly representable scores: equal logits
    (0.5) and logit gaps of +-120 (1.0 and 0: exp underflows to 0 on both sides)."""
    rng = np.random.default_rng(seed)
    cells = fh * fw
    na = cells * A
    heads = np.zeros((nimg, cells, 6 * A), F32)
    for i in range(nimg):
        k = rng.choice(M_LATTICE, na, replace=False)
        p = (k + 0.5) / M_LATTICE
        d = np.log(p / (1 - p))
        base = rng.normal(0, 2, na)
        bg, fg = base, base + d
        if ties:
            t = rng.permutation(na)
            half, one, zero = t[:600], t[600:900], t[900:1100]
            fg[half] = bg[half]
            fg[one] = bg[one] + 120.0
            fg[zero] = bg[zero] - 120.0
        lg = np.stack([bg, fg], 1).astype(F32).reshape(cells, 2 * A)
        dl = (rng.standard_normal((na, 4)) * 0.2).astype(F32)
        dl[:, 2:] = 0
        heads[i, :, :2 * A] = lg
        heads[i, :, 2 * A:] = dl.reshape(cells, 4 * A)
    return heads


def _rpn_oracle(heads, A, anchors, im, cfg):
    out = []
    for h in heads:
        cells = h.shape[0]
        logits = h[:, :2 * A].reshape(cells * A, 2)
        pred = h[:, 2 * A:].reshape(cells * A, 4)
        out.append(ofr.rpn_proposal(T.softmax(logits), pred, anchors, im, cfg))
    return out


def _ulps(a, b):
    a = np.asarray(a, F32).view(np.int32).astype(np.int64)
    b = np.asarray(b, F32).view(np.int32).astype(np.int64)
    return np.abs(a - b)


def _check_rpn(heads, A, anchors, cap, im, cfg, nimg=None):
    nimg = heads.shape[0] if nimg is None else nimg
    na = anchors.shape[0]
    props, scores, counts = ops().rpn_proposals_batched(heads[:nimg], A, anchors, na, cap, im, cfg)
    refs = _rpn_oracle(heads[:nimg], A, anchors, im, cfg)
    for i, ref in enumerate(refs):
        k = len(ref['scores'])
        assert counts[i] == k, (i, counts[i], k)
        np.testing.assert_array_equal(props[i, :k], ref['proposals'], err_msg='image %d' % i)
        assert _ulps(scores[i, :k], ref['scores']).max(initial=0) <= SCORE_ULPS, i
        assert (props[i, k:] == 0).all() and (scores[i, k:] == 0).all()
    return refs


R50_CFG = {'pre_nms_top_n': 12000, 'post_nms_top_n': 2000, 'nms_threshold': 0.7, 'min_prob_threshold': 0.0,
           'clip_after_nms': False, 'filter_outside_anchors': False, 'apply_nms': True}


@pytest.fixture(scope='module')
def r50_half_batch():
    A = 12
    anchors = fasterrcnn_anchors(38, 64, 256, [0.5, 1, 2], [0.25, 0.5, 1, 2], 16).astype(F32)
    assert anchors.shape[0] == 29184
    return A, anchors, _rpn_inputs(31, 4, 38, 64, A)


def test_rpn_fused_softmax_within_the_stated_ulp_bound(r50_half_batch):
    """The fused softmax's scores for every anchor against T.softmax (the selected ones are checked in every test)."""
    A, anchors, heads = r50_half_batch
    cfg = dict(R50_CFG, pre_nms_top_n=29184, post_nms_top_n=29184, apply_nms=False)
    props, scores, counts = ops().rpn_proposals_batched(heads[:1], A, anchors, 29184, 29184, (600, 1024), cfg)
    ref = _rpn_oracle(heads[:1], A, anchors, (600, 1024), cfg)[0]
    assert counts[0] == len(ref['scores']) == 29184
    np.testing.assert_array_equal(props[0], ref['proposals'])
    assert _ulps(scores[0], ref['scores']).max() <= SCORE_ULPS
    for v in (0.5, 1.0, 0.0):                              # the tie groups are exact and tie-ordered by anchor index
        assert (scores[0] == v).sum() >= 200, v


@pytest.mark.parametrize('nimg,path', [(4, TWO_PHASE), (2, STAGED)])
def test_rpn_r50_half_batch(r50_half_batch, nimg, path):
    """4 images of 38 x 64 x 12 anchors in a workspace sized for 40 x 66 (NaN-filled tail, image stride != na)."""
    A, anchors, heads = r50_half_batch
    cap = 40 * 66 * A
    assert ops().nms_path(nimg, min(cap, 12000), 0.7) == path
    refs = _check_rpn(heads, A, anchors, cap, (600, 1024), R50_CFG, nimg)
    for r in refs:
        sorted_boxes = r['sorted_top_proposals']
        k1, surv = two_phase_stats(sorted_boxes, 0.7, 2000)
        print('R50 RPN image: nvalid %d, k1 %d, survivors %d, kept %d' % (len(sorted_boxes), k1, len(surv),
                                                                          len(r['scores'])))
        assert len(sorted_boxes) == 12000 and k1 < 2000 and len(surv) > 0


def test_rpn_output_stride_8_cut_and_two_phase():
    """115 200 anchors per image: the top-k cut ahead of the sort and the two-phase NMS in one chain."""
    A = 12
    anchors = fasterrcnn_anchors(75, 128, 256, [0.5, 1, 2], [0.25, 0.5, 1, 2], 8).astype(F32)
    assert anchors.shape[0] == 115200
    heads = _rpn_inputs(41, 4, 75, 128, A)
    assert ops().nms_path(4, 12000, 0.7) == TWO_PHASE
    _check_rpn(heads, A, anchors, 115200, (600, 1024), R50_CFG)


def test_rpn_batched_filters_and_clip_after_nms(r50_half_batch):
    A, anchors, heads = r50_half_batch
    cfg = dict(R50_CFG, min_prob_threshold=0.3, filter_outside_anchors=True, clip_after_nms=True)
    refs = _check_rpn(heads, A, anchors, 29184 + 100, (600, 1024), cfg, 3)
    assert all(len(r['unsorted_scores']) < 12000 for r in refs)     # min_prob and the anchor filter both cut


def test_rpn_batched_without_nms(r50_half_batch):
    """apply_nms off: every sorted top-n candidate survives (the engine sets post_nms_top_n = pre_nms_top_n)."""
    A, anchors, heads = r50_half_batch
    assert ops().nms_path(4, 12000, float('inf')) == STAGED
    _check_rpn(heads, A, anchors, 29184, (600, 1024), dict(R50_CFG, apply_nms=False, post_nms_top_n=12000))


# ---------------------------------------------------------------- batched detections at the engine's layouts
def _frcnn_inputs(seed, nimg, r, C, clustered):
    """Proposals [nimg][r][4], the fc row [nimg * r][5C + 1] (deltas at C + 1), cls_prob [nimg * r][C + 1].
    clustered: the rows with the highest class probabilities are jittered copies of 24 boxes, the rest spread out."""
    rng = np.random.default_rng(seed)
    fcw = 5 * C + 1
    props = np.empty((nimg, r, 4), F32)
    logits = rng.standard_normal((nimg, r, C + 1)).astype(F32) * 2
    for i in range(nimg):
        c = rng.uniform(0, 900, (r, 2)); s = rng.uniform(16, 200, (r, 2))
        props[i] = np.concatenate([c, c + s], 1)
        if clustered:
            hot = rng.permutation(r)[:2600]
            centres = rng.uniform(0, 1, (24, 2)) * [880, 460]
            k = rng.integers(0, 24, hot.size)
            xy = centres[k] + rng.uniform(-2, 2, (hot.size, 2))
            props[i, hot] = np.concatenate([xy, xy + 120 + rng.uniform(-2, 2, (hot.size, 2))], 1)
            cold = np.ones(r, bool); cold[hot] = False
            logits[i, cold, 0] += 30                        # the spread rows: background by a wide margin
    fc = (rng.standard_normal((nimg * r, fcw)) * 0.5).astype(F32)
    fc[:, C + 3::4] = 0                                  # dw, dh of every class
    fc[:, C + 4::4] = 0
    prob = T.softmax(logits.reshape(nimg * r, C + 1))
    return props, fc, prob


def _frcnn_oracle(props, fc, prob, counts, C, im, cfg, var):
    nimg, r = props.shape[:2]
    out = []
    for i in range(nimg):
        n = counts[i]
        rows = slice(i * r, i * r + n)
        out.append(ofr.rcnn_proposal(props[i, :n], fc[rows, C + 1:], prob[rows], im, C, cfg, variances=var))
    return out


def _class_lists(props, deltas, prob, C, im, cfg, var):
    """The per-class candidate lists in score order, as rcnn_proposal builds them."""
    lists = []
    for c in range(C):
        p = prob[:, c + 1]
        b = clip_boxes(decode(props, deltas[:, 4 * c:4 * c + 4], variances=var), im)
        ok = ((np.maximum(b[:, 2] - b[:, 0], F32(0)) * np.maximum(b[:, 3] - b[:, 1], F32(0))) > 0) & \
             (p >= F32(cfg['min_prob_threshold']))
        b, p = b[ok], p[ok]
        lists.append(b[np.argsort(-p, kind='stable')])
    return lists


def _check_det(got, refs, tm, records=None):
    obj, lab, prob, cnt, rec = got
    for i, ref in enumerate(refs):
        k = len(ref['proposal_label'])
        assert cnt[i] == k, (i, cnt[i], k)
        np.testing.assert_array_equal(lab[i, :k], ref['proposal_label'])
        np.testing.assert_array_equal(prob[i, :k], ref['proposal_label_prob'])
        np.testing.assert_array_equal(obj[i, :k], ref['objects'])
        assert (lab[i, k:] == -1).all() and (prob[i, k:] == 0).all() and (obj[i, k:] == 0).all()
        if rec is not None:                             # the packed record row, field by field
            assert rec[i, 0] == k
            np.testing.assert_array_equal(rec[i, 1:1 + 4 * tm].reshape(tm, 4), obj[i])
            np.testing.assert_array_equal(rec[i, 1 + 4 * tm:1 + 5 * tm], prob[i])
            np.testing.assert_array_equal(rec[i, 1 + 5 * tm:], lab[i].astype(F32))


@pytest.mark.parametrize('min_prob', [0.0, 0.05])
def test_frcnn_detections_fc_row_layout_and_row_counts(min_prob):
    """3 images x 2000 proposals x 80 classes, deltas read inside the fc row, rows past row_counts [2000, 1234, 0]
    hold NaN deltas (even classes), garbage boxes and high probabilities that must not leak."""
    nimg, r, C = 3, 2000, 80
    im, var = (600, 1024), [0.1, 0.2]
    cfg = {'class_max_detections': 100, 'class_nms_threshold': 0.5, 'total_max_detections': 300,
           'min_prob_threshold': min_prob}
    props, fc, prob = _frcnn_inputs(7, nimg, r, C, clustered=False)
    counts = [2000, 1234, 0]
    for i in range(nimg):
        rows = slice(i * r + counts[i], (i + 1) * r)
        fc[rows, C + 1::8] = np.nan                      # NaN dx for the even classes; the odd ones decode fine
        props[i, counts[i]:] = [5, 5, 300, 300]
        prob[rows] = 0; prob[rows, 1:] = 0.9
    assert ops().nms_path(nimg * C, r, 0.5) == STAGED
    refs = _frcnn_oracle(props, fc, prob, counts, C, im, cfg, var)
    got = ops().class_detections_batched(props, r * 4, counts, fc.reshape(-1)[C + 1:], 5 * C + 1, prob, nimg, r, C, im,
                                         cfg, var, shared_deltas=False, records=True)
    _check_det(got, refs, 300, records=True)
    assert got[3][2] == 0


def test_frcnn_detections_two_phase_class_lists():
    """post_nms_top_n = 5000: 2 x 80 class lists of 5000 candidates take the two-phase path.  The highest-probability
    rows cluster, so most lists keep few boxes among their first 2048 and phase 2 appends the rest."""
    nimg, r, C = 2, 5000, 80
    im, var = (600, 1024), [0.1, 0.2]
    cfg = {'class_max_detections': 100, 'class_nms_threshold': 0.5, 'total_max_detections': 300,
           'min_prob_threshold': 0.0}
    props, fc, prob = _frcnn_inputs(8, nimg, r, C, clustered=True)
    assert ops().nms_path(nimg * C, r, 0.5) == TWO_PHASE
    counts = [r, r]
    refs = _frcnn_oracle(props, fc, prob, counts, C, im, cfg, var)
    work = 0
    for i in range(nimg):
        rows = slice(i * r, (i + 1) * r)
        for lst in _class_lists(props[i], fc[rows, C + 1:], prob[rows], C, im, cfg, var):
            k1, surv = two_phase_stats(lst, 0.5, 100)
            work += k1 < 100 and len(surv) > 0
    print('FRCNN two-phase class lists with phase-2 work: %d of %d' % (work, nimg * C))
    assert work >= nimg * C // 2
    got = ops().class_detections_batched(props, r * 4, counts, fc.reshape(-1)[C + 1:], 5 * C + 1, prob, nimg, r, C, im,
                                         cfg, var, shared_deltas=False)
    _check_det(got, refs, 300)


@pytest.mark.parametrize('min_prob', [0.0, 0.3])
def test_ssd_detections_shared_anchors(min_prob):
    """2 images x 20 classes over 8096 shared anchors (image stride 0): 40 class lists take the two-phase path.
    The anchors near two objects regress onto them and carry the foreground probability, so with min_prob 0
    most lists keep few boxes among their first 2048 candidates and phase 2 appends the rest."""
    shapes = [(37, 37), (18, 18), (9, 9), (5, 5), (3, 3), (1, 1)]
    anchors = ssd_anchors(shapes, 0.1, 0.88, [1, 0.5, 2, 0.333, 3], [4, 6, 6, 6, 4, 4], [300, 300, 3]).astype(F32)
    r, nc, nimg = anchors.shape[0], 20, 2
    assert r == 8096
    rng = np.random.default_rng(23)
    loc = (rng.standard_normal((nimg, r, 4)) * 0.5).astype(F32)
    loc[:, :, 2:] = 0
    ctr = (anchors[:, :2] + anchors[:, 2:]) / 2
    wh = anchors[:, 2:] - anchors[:, :2]
    logits = rng.standard_normal((nimg, r, nc + 1)) * 3
    for i in range(nimg):                            # like a trained head: the anchors near an object regress onto it
        hot = np.zeros(r, bool)
        for o in rng.uniform(80, 220, (2, 2)):
            near = np.hypot(*(ctr - o).T) < 70
            loc[i, near, :2] = ((o - ctr[near]) / (wh[near] * 0.1) + rng.uniform(-0.05, 0.05, (near.sum(), 2)))
            hot |= near
        logits[i, ~hot, 0] += 30                     # the rest: background by a wide margin
    prob = T.softmax(logits.astype(F32).reshape(nimg * r, nc + 1))
    cfg = {'class_max_detections': 100, 'class_nms_threshold': 0.45, 'total_max_detections': 100,
           'min_prob_threshold': min_prob}
    assert ops().nms_path(nimg * nc, r, 0.45) == TWO_PHASE
    refs, work, nvalid = [], 0, []
    for i in range(nimg):
        p_i, l_i = prob[i * r:(i + 1) * r], loc[i]
        ref = ossd.ssd_proposal(p_i, l_i, anchors, (300.0, 300.0), nc, cfg, [0.1, 0.2])
        refs.append({'proposal_label': ref['labels'], 'proposal_label_prob': ref['probs'], 'objects': ref['objects']})
        for c in range(nc):
            p = p_i[:, c + 1]
            ok = p >= F32(min_prob)
            b = clip_boxes(decode(anchors[ok], l_i[ok], [0.1, 0.2]), (300.0, 300.0))
            a = (np.maximum(b[:, 2] - b[:, 0], F32(0)) * np.maximum(b[:, 3] - b[:, 1], F32(0))) > 0
            b, p = b[a], p[ok][a]
            lst = b[np.argsort(-p, kind='stable')]
            nvalid.append(len(lst))
            k1, surv = two_phase_stats(lst, 0.45, 100)
            work += k1 < 100 and len(surv) > 0
    print('SSD min_prob %g: class-list nvalid %d..%d (median %d), %d of %d lists with phase-2 work' % (
        min_prob, min(nvalid), max(nvalid), int(np.median(nvalid)), work, nimg * nc))
    if min_prob == 0.0:
        assert work >= nimg * nc // 2
    got = ops().class_detections_batched(anchors, 0, None, loc, 4, prob, nimg, r, nc, (300, 300), cfg, [0.1, 0.2],
                                         shared_deltas=True, records=True)
    _check_det(got, refs, 100, records=True)
