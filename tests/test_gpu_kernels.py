"""Per-kernel parity: every CUDA stage, called through the C ABI, against the CPU
oracle on the same seeded inputs (`-m gpu`, needs an H100).

Tolerances: integer / index outputs bit-exact; floating point within the
north-star's 1e-3 on box coordinates (px) and fp32-class (<= 2e-5 of the output
scale) on convolution activations -- the fp16x2 split carries 22 mantissa bits.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import tf_ops as T
from oracle import fasterrcnn as ofr
from oracle import ssd as ossd
from oracle.bbox import encode


def ops():
    import gpu_ops
    return gpu_ops


def assert_close(y, ref, rel=2e-5, what=''):
    assert y.shape == ref.shape, (what, y.shape, ref.shape)
    scale = max(1.0, float(np.abs(ref).max()))
    err = float(np.abs(y.astype(np.float64) - ref.astype(np.float64)).max())
    assert err <= rel * scale, '%s: max abs err %.3e > %.1e * %.3g' % (what, err, rel, scale)


def _bn_fold(rng, c):
    return rng.uniform(0.5, 1.5, c).astype(np.float32), rng.standard_normal(c).astype(np.float32) * 0.1


def _ref_conv(x, w, stride, rate, padding, scale, bias, residual, act):
    if padding == 'SLIM':
        y = T.conv2d_same(x, w, stride, rate)
    else:
        y = T.conv2d(x, w, stride, padding, rate)
    if scale is not None:
        y = y * scale
    if bias is not None:
        y = y + bias
    if residual is not None:
        y = y + residual
    if act == 1:
        y = T.relu(y)
    elif act == 2:
        y = T.relu6(y)
    return y.astype(np.float32)


CONV_CASES = [
    # name, n, h, w, cin, cout, k, stride, rate, padding, residual, act
    ('stem7x7s2', 2, 45, 61, 3, 64, 7, 2, 1, 'SLIM', False, 1),
    ('1x1_64_256', 2, 19, 32, 64, 256, 1, 1, 1, 'SAME', True, 1),
    ('3x3_64_64', 2, 19, 32, 64, 64, 3, 1, 1, 'SAME', False, 1),
    ('3x3s2_slim', 1, 38, 65, 64, 64, 3, 2, 1, 'SLIM', False, 1),
    ('3x3_rate6', 1, 18, 18, 128, 128, 3, 1, 6, 'SAME', False, 1),
    ('3x3_valid', 2, 5, 5, 128, 256, 3, 1, 1, 'VALID', False, 1),
    ('3x3s2_same', 2, 18, 18, 64, 128, 3, 2, 1, 'SAME', False, 1),
    ('rpn_heads_72', 1, 12, 16, 128, 72, 1, 1, 1, 'SAME', False, 0),
    ('relu6', 1, 12, 16, 128, 128, 3, 1, 1, 'SAME', False, 2),
    ('fc_401', 37, 1, 1, 256, 401, 1, 1, 1, 'SAME', False, 0),
    ('roi_7x7', 5, 7, 7, 128, 128, 3, 1, 1, 'SAME', True, 1),
    ('wide_256', 1, 38, 64, 256, 256, 3, 1, 1, 'SAME', False, 1),
    ('1x1_1024_256', 1, 38, 64, 1024, 256, 1, 1, 1, 'SAME', False, 1),
    # enough tiles that a stream-K range holds whole tiles plus a head and a tail piece
    ('sk_many_tiles', 2, 64, 96, 128, 256, 3, 1, 1, 'SAME', True, 1),
    ('sk_1x1_512_128', 3, 40, 64, 512, 128, 1, 1, 1, 'SAME', False, 1),
    # short-K 1x1 layers of the bottlenecks (the 16-epilogue-warp kernels): residual / no residual / subsampled
    ('b1_conv3_64_256_res', 2, 38, 64, 64, 256, 1, 1, 1, 'SAME', True, 1),
    ('b1_shortcut_64_256', 2, 38, 64, 64, 256, 1, 1, 1, 'SAME', False, 0),
    ('b2_conv3_128_512_res', 3, 19, 32, 128, 512, 1, 1, 1, 'SAME', True, 1),
    ('b3_shortcut_512_1024', 1, 38, 64, 512, 1024, 1, 1, 1, 'SAME', False, 0),
    # the block3 endpoint at its production size (several waves of tiles per CTA)
    ('b3_conv3_endpoint', 8, 38, 64, 256, 1024, 1, 1, 1, 'SAME', True, 1),
    # 3x3 stride-1 layers for the halo-patch kernels: 13-row tiles; C_out = 64 with three channel slices, a ragged last
    # tile column and a ragged last tile row; an odd number of M tiles (the CTA-pair kernel's idle half) with two N tiles
    ('halo_38x64_128', 2, 38, 64, 128, 128, 3, 1, 1, 'SAME', False, 1),
    ('halo_23x61_192_64', 1, 23, 61, 192, 64, 3, 1, 1, 'SAME', False, 1),
    ('halo_75x20_64_256', 3, 75, 20, 64, 256, 3, 1, 1, 'SAME', False, 0),
]


@pytest.mark.parametrize('impl', ['simt', 'tc', 'tc_streamk', 'tc_split', 'tc_split_epi16', 'tc_split_epi16_streamk', 'tc_split_cta2', 'tc_split_cta2_streamk',
                                  'tc_split_halo', 'tc_split_halo_streamk', 'tc_split_halo_cta2', 'tc_split_halo_cta2_streamk'])
@pytest.mark.parametrize('case', CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv2d_matches_oracle(case, impl):
    name, n, h, w, cin, cout, k, stride, rate, padding, use_res, act = case
    if impl != 'simt' and cin % 64 != 0:
        pytest.skip('layer shape runs on the SIMT kernel by design')
    if impl.startswith('tc_split') and cout % 32 != 0:
        pytest.skip('split-plane outputs exist for cout % 32 == 0 (head layers write fp32)')
    if 'halo' in impl and not (k == 3 and stride == 1 and rate == 1 and padding == 'SAME' and not use_res):
        pytest.skip('the halo-patch kernels exist for 3x3 / stride 1 / rate 1 / SAME layers without residual')
    import zlib
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = (rng.standard_normal((n, h, w, cin)) * 2).astype(np.float32)
    wt = (rng.standard_normal((k, k, cin, cout)) * np.sqrt(2.0 / (k * k * cin))).astype(np.float32)
    scale, bias = _bn_fold(rng, cout)
    ref0 = _ref_conv(x, wt, stride, rate, padding, scale, bias, None, 0)
    res = rng.standard_normal(ref0.shape).astype(np.float32) if use_res else None
    ref = _ref_conv(x, wt, stride, rate, padding, scale, bias, res, act)
    y = ops().conv2d(x, wt, stride, rate, padding, scale, bias, res, act, impl)
    assert_close(y, ref, 2e-5, '%s/%s' % (name, impl))


def test_conv_tc_equals_simt_on_large_k():
    """RPN-sized reduction (K = 9216): both CUDA paths agree to fp32-class accuracy."""
    rng = np.random.default_rng(7)
    x = np.abs(rng.standard_normal((1, 20, 30, 1024))).astype(np.float32)
    wt = (rng.standard_normal((3, 3, 1024, 128)) * 0.01).astype(np.float32)
    b = rng.standard_normal(128).astype(np.float32) * 0.01
    a = ops().conv2d(x, wt, 1, 1, 'SAME', None, b, None, 2, 'simt')
    c = ops().conv2d(x, wt, 1, 1, 'SAME', None, b, None, 2, 'tc')
    ref = _ref_conv(x, wt, 1, 1, 'SAME', None, b, None, 2)
    assert_close(a, ref, 2e-5, 'simt')
    assert_close(c, ref, 2e-5, 'tc')


@pytest.mark.parametrize('h0,w0,nh,nw,dtype', [(375, 500, 600, 800, np.uint8), (1200, 1600, 768, 1024, np.uint8),
                                               (333, 517, 300, 300, np.uint8), (64, 48, 64, 48, np.uint8),
                                               (97, 131, 600, 810, np.float32)])
def test_resize_bilinear_bit_exact(h0, w0, nh, nw, dtype):
    """utils/image.py:94-97,139-142 (tf.image.resize_images BILINEAR, TF1 legacy kernel): the GPU kernel follows the
    oracle's float32 operation order without FMA contraction -- identical bits."""
    rng = np.random.default_rng(h0 + nw)
    img = rng.integers(0, 256, (h0, w0, 3)).astype(dtype)
    if dtype == np.float32:
        img = img + rng.uniform(0, 1, img.shape).astype(np.float32)
    ref = T.resize_bilinear(img.astype(np.float32), nh, nw)
    got = ops().resize_bilinear(img, nh, nw)
    np.testing.assert_array_equal(got, ref)


@pytest.mark.parametrize('k,stride,padding,h,w', [(3, 2, 'SAME', 300, 512), (2, 2, 'VALID', 75, 75),
                                                    (3, 1, 'SAME', 18, 18), (2, 2, 'VALID', 14, 14)])
def test_max_pool(k, stride, padding, h, w):
    rng = np.random.default_rng(3)
    x = rng.standard_normal((2, h, w, 64)).astype(np.float32)
    assert_close(ops().max_pool(x, k, stride, padding), T.max_pool(x, k, stride, padding), 1e-6, 'max_pool')


def test_roi_pool_reference_goldens():
    """models/fasterrcnn/roi_pool_test.py:56-175 on the GPU kernel (C padded to 8)."""
    a = np.ones((5, 5))
    m = np.block([[a * 1, a * 2], [a * 3, a * 4]])[None, :, :, None].astype(np.float32)
    fmap = np.repeat(m, 8, axis=3)
    r = ops().roi_pool(fmap, np.array([[1, 1, 4, 4], [6, 1, 9, 4], [1, 6, 4, 9], [6, 6, 9, 9]], np.float32), (10, 10), 2, 2)
    for i in range(4):
        np.testing.assert_array_equal(r[i, :, :, 0], np.ones((2, 2)) * (i + 1))
    r = ops().roi_pool(fmap, np.array([[3, 1, 6, 4], [1, 3, 4, 7], [5, 3, 9, 7], [3, 6, 6, 9]], np.float32), (10, 10), 2, 2)[..., 0]
    np.testing.assert_array_equal(r[0], [[1, 2], [1, 2]])
    np.testing.assert_array_equal(r[1], [[1, 1], [3, 3]])
    np.testing.assert_array_equal(r[2], [[2, 2], [4, 4]])
    np.testing.assert_array_equal(r[3], [[3, 4], [3, 4]])


def test_roi_pool_random_matches_oracle():
    rng = np.random.default_rng(5)
    fmap = rng.standard_normal((1, 38, 64, 256)).astype(np.float32)
    n = 97
    c = rng.uniform(-50, 1050, (n, 2)); s = rng.uniform(4, 600, (n, 2))
    rois = np.concatenate([c, c + s], 1).astype(np.float32)
    rois[:, [0, 2]] = np.clip(rois[:, [0, 2]], 0, 1023); rois[:, [1, 3]] = np.clip(rois[:, [1, 3]], 0, 599)
    rois[0] = [0, 0, 1023, 599]; rois[1] = [10, 10, 10, 10]
    ref = ofr.roi_pool(rois, fmap, (600, 1024), 7, 7)['roi_pool']
    y = ops().roi_pool(fmap, rois, (600, 1024), 7, 7)
    assert_close(y, ref, 2e-6, 'roi_pool')


@pytest.mark.parametrize('n', [1, 2, 63, 64, 65, 1000, 8192, 12000, 29184, 40000])
def test_sort_desc_exact_with_ties(n):
    rng = np.random.default_rng(n)
    s = rng.uniform(0, 1, n).astype(np.float32)
    s[rng.integers(0, n, max(1, n // 7))] = s[0]          # exact ties -> lower index first
    idx = ops().sort_desc(s)
    np.testing.assert_array_equal(idx, np.argsort(-s, kind='stable').astype(np.int32))


def _random_boxes(rng, n, size=600.0):
    c = rng.uniform(0, size, (n, 2)); s = rng.uniform(8, size / 3, (n, 2))
    return np.concatenate([c, c + s], 1).astype(np.float32)


@pytest.mark.parametrize('n,thr,max_out', [(1, 0.5, 10), (64, 0.5, 64), (65, 0.3, 10), (500, 0.7, 500),
                                             (3000, 0.7, 300), (12000, 0.7, 2000), (777, 0.0, 777), (300, 1.0, 300)])
def test_nms_bitmask_identical_keep_set(n, thr, max_out):
    rng = np.random.default_rng(n + int(thr * 100))
    boxes = _random_boxes(rng, n)
    if n > 10:
        boxes[5] = boxes[4]; boxes[9] = [10, 10, 10, 50]       # duplicate + zero-area box
    scores = np.arange(n, 0, -1).astype(np.float32)            # already sorted
    ref = T.non_max_suppression(boxes[:, [1, 0, 3, 2]], scores, max_out, thr)
    got = ops().nms_sorted(boxes, thr, max_out)
    np.testing.assert_array_equal(got, ref)


def test_nms_ratio_exactly_at_threshold_takes_the_exact_path():
    """IoU == threshold is NOT suppressed (tf.image.non_max_suppression uses a strict >).  The mask kernel decides
    almost every pair with a +-2^-20 margin test and only divides inside the margin: these pairs sit exactly on
    it, one ulp below it and one ulp above it."""
    a = [0, 0, 2, 2]; b = [0, 0, 2, 1]                       # inter 2, union 4 -> IoU 0.5 exactly
    c = [10, 10, 12, 11]; d = [11, 10, 13, 11]               # inter 1, union 3 -> IoU RN(1/3)
    third = np.float32(1.0) / np.float32(3.0)
    for boxes, thr in (([a, b], np.float32(0.5)), ([c, d], third)):
        boxes = np.array(boxes, np.float32)
        for t in (thr, np.nextafter(thr, np.float32(0)), np.nextafter(thr, np.float32(1))):
            ref = T.non_max_suppression(boxes[:, [1, 0, 3, 2]], np.array([2, 1], np.float32), 2, float(t))
            got = ops().nms_sorted(boxes, float(t), 2)
            np.testing.assert_array_equal(got, ref)
        assert len(ops().nms_sorted(boxes, float(thr), 2)) == 2                               # equal: both kept
        assert len(ops().nms_sorted(boxes, float(np.nextafter(thr, np.float32(0))), 2)) == 1  # one ulp lower: suppressed


def test_nms_all_duplicates_and_all_degenerate():
    boxes = np.tile(np.array([[5, 5, 50, 60]], np.float32), (300, 1))
    np.testing.assert_array_equal(ops().nms_sorted(boxes, 0.7, 300), [0])
    flat = np.tile(np.array([[5, 5, 5, 60]], np.float32), (130, 1))          # zero area: IoU 0, nothing suppressed
    ref = T.non_max_suppression(flat[:, [1, 0, 3, 2]], np.arange(130, 0, -1).astype(np.float32), 130, 0.7)
    np.testing.assert_array_equal(ops().nms_sorted(flat, 0.7, 130), ref)


RPN_CFG = {'pre_nms_top_n': 4, 'post_nms_top_n': 3, 'nms_threshold': 1, 'min_size': 0, 'clip_after_nms': False,
           'filter_outside_anchors': False, 'apply_nms': True, 'min_prob_threshold': 0.0}


def _rpn_both(anchors, prob, cfg, gt=None, pred=None, im=(40, 40)):
    anchors = np.array(anchors, np.float32)
    prob = np.array(prob, np.float32)
    pred = encode(anchors, np.array(gt, np.float32)) if pred is None else np.array(pred, np.float32)
    ref = ofr.rpn_proposal(prob, pred, anchors, im, cfg)
    p, s = ops().rpn_proposals(prob, pred, anchors, im, cfg)
    return ref, p, s


def test_rpn_proposals_reference_goldens_on_gpu():
    """models/fasterrcnn/rpn_proposal_test.py:61-500 -- same inputs through the CUDA chain."""
    gt = [[10, 10, 26, 36], [10, 10, 20, 22], [10, 11, 20, 21], [19, 30, 33, 38]]
    anchors = [[11, 13, 34, 31], [10, 10, 20, 22], [11, 13, 34, 28], [21, 29, 34, 37]]
    prob = [[0.8, 0.2], [0.1, 0.9], [0.4, 0.6], [0.2, 0.8]]
    for thr, n_exp, sc in ((0.0, 2, [0.9, 0.8]), (0.3, 3, [0.9, 0.8, 0.2]), (0.6, 3, [0.9, 0.8, 0.2]),
                           (0.8, 3, [0.9, 0.8, 0.2]), (1.0, 4, None)):
        ref, p, s = _rpn_both(anchors, prob, dict(RPN_CFG, post_nms_top_n=4, nms_threshold=thr), gt=gt)
        assert p.shape == (n_exp, 4)
        if sc:
            np.testing.assert_allclose(s, sc)
        np.testing.assert_allclose(p, ref['proposals'], atol=1e-3)
    gt = [[10, 10, 20, 22], [10, 10, 20, 22], [10, 10, 20, 50], [10, 10, 20, 22]]
    anchors = [[11, 13, 34, 31], [10, 10, 20, 22], [11, 13, 34, 40], [7, 13, 34, 30]]
    prob = [[0.3, 0.7], [0.4, 0.6], [0.9, 0.1], [0.8, 0.2]]
    for over, n_exp, sc in (({}, 3, [0.7, 0.6, 0.2]), ({'post_nms_top_n': 2}, 2, [0.7, 0.6]),
                            ({'post_nms_top_n': 3, 'pre_nms_top_n': 2}, 2, [0.7, 0.6]),
                            ({'post_nms_top_n': 1, 'pre_nms_top_n': 2}, 1, [0.7])):
        ref, p, s = _rpn_both(anchors, prob, dict(RPN_CFG, **over), gt=gt)
        assert p.shape == (n_exp, 4)
        np.testing.assert_allclose(s, sc)
    # negative areas (NaN deltas) are filtered
    gt = [[10, 10, 20, 3], [10, 10, 20, 22], [10, 10, 8, 22], [10, 10, 20, 22]]
    anchors = [[11, 13, 12, 16], [10, 10, 20, 22], [11, 13, 12, 19], [7, 13, 34, 30]]
    with np.errstate(invalid='ignore'):
        ref, p, s = _rpn_both(anchors, prob, RPN_CFG, gt=gt)
    assert p.shape == (2, 4)
    # clipping before / after NMS
    anchors = [[-20, -10, 12, 6], [2, -10, 20, 20], [0, 0, 12, 16], [2, -10, 20, 2]]
    prob = [[0.3, 0.7], [0.4, 0.6], [0.3, 0.7], [0.1, 0.9]]
    for after in (False, True):
        ref, p, s = _rpn_both(anchors, prob, dict(RPN_CFG, clip_after_nms=after), pred=np.zeros((4, 4)))
        assert (p >= 0).all() and (p < 40).all()
        np.testing.assert_allclose(p, ref['proposals'], atol=1e-3)
    # outside-anchor filter
    gt = [[0, 0, 10, 12], [10, 10, 20, 22], [10, 10, 20, 22], [30, 25, 39, 39], [30, 25, 39, 39]]
    anchors = [[-20, -10, 12, 6], [2, 10, 20, 20], [0, 0, 50, 16], [2, -10, 20, 50], [25, 30, 27, 33]]
    prob = [[0.3, 0.7], [0.4, 0.6], [0.3, 0.7], [0.1, 0.9], [0.2, 0.8]]
    ref, p, s = _rpn_both(anchors, prob, dict(RPN_CFG, filter_outside_anchors=True, pre_nms_top_n=5, post_nms_top_n=5), gt=gt)
    assert p.shape == ref['proposals'].shape == (2, 4)


def test_rpn_proposals_full_size_matches_oracle():
    """29 184 anchors (38x64x12), default thresholds: identical selection, boxes within 1e-3 px."""
    from oracle.anchors import fasterrcnn_anchors
    rng = np.random.default_rng(11)
    anchors = fasterrcnn_anchors(38, 64, 256, [0.5, 1, 2], [0.25, 0.5, 1, 2], 16).astype(np.float32)
    na = anchors.shape[0]
    logits = rng.standard_normal((na, 2)).astype(np.float32)
    prob = T.softmax(logits)
    pred = (rng.standard_normal((na, 4)) * 0.2).astype(np.float32)
    pred[:, 2:] = 0      # exp(0) == 1 on both sides: decode is bit-reproducible, so the keep set must be IDENTICAL
    cfg = {'pre_nms_top_n': 12000, 'post_nms_top_n': 2000, 'nms_threshold': 0.7, 'min_prob_threshold': 0.0,
           'clip_after_nms': False, 'filter_outside_anchors': False, 'apply_nms': True}
    ref = ofr.rpn_proposal(prob, pred, anchors, (600, 1024), cfg)
    p, s = ops().rpn_proposals(prob, pred, anchors, (600, 1024), cfg)
    assert p.shape == ref['proposals'].shape
    np.testing.assert_array_equal(s, ref['scores'])
    np.testing.assert_array_equal(p, ref['proposals'])


def test_rpn_proposals_with_size_deltas():
    """exp() path: CUDA expf vs numpy differ by <= 1 ulp -> boxes within 1e-3 px."""
    rng = np.random.default_rng(12)
    from oracle.anchors import fasterrcnn_anchors
    anchors = fasterrcnn_anchors(6, 8, 256, [0.5, 1, 2], [0.25, 0.5, 1, 2], 16).astype(np.float32)
    na = anchors.shape[0]
    prob = T.softmax(rng.standard_normal((na, 2)).astype(np.float32))
    pred = (rng.standard_normal((na, 4)) * 0.3).astype(np.float32)
    cfg = {'pre_nms_top_n': 400, 'post_nms_top_n': 100, 'nms_threshold': 0.7, 'min_prob_threshold': 0.1,
           'clip_after_nms': False, 'filter_outside_anchors': False, 'apply_nms': True}
    ref = ofr.rpn_proposal(prob, pred, anchors, (96, 128), cfg)
    p, s = ops().rpn_proposals(prob, pred, anchors, (96, 128), cfg)
    np.testing.assert_array_equal(s, ref['scores'])
    np.testing.assert_allclose(p, ref['proposals'], atol=1e-3)


def test_class_detections_rcnn_reference_golden():
    """models/fasterrcnn/rcnn_proposal_test.py:198-242 testBboxPred (exact boxes + order, atol 1e-3)."""
    proposed = np.array([(200, 315, 400, 370), (56, 0, 106, 4), (15, 15, 20, 20)], np.float32)
    gt = [[(0, 0, 1, 1)], [(5, 5, 10, 10)], [(15, 15, 20, 20)]]
    bbox_pred = np.concatenate([encode(proposed, np.array(g * 3, np.float32)) for g in gt], axis=1)
    cls_prob = np.array([(0., 1., 0., 0.), (.2, .25, .3, .25), (.45, 0., 0., .55)], np.float32)
    cfg = {'class_max_detections': 100, 'class_nms_threshold': 0.6, 'total_max_detections': 300, 'min_prob_threshold': 0.0}
    obj, lab, prob = ops().class_detections(proposed, bbox_pred, cls_prob, (900, 1440), 3, cfg, None)
    objects = np.array([g[0] for g in gt], np.float32)
    order = cls_prob[:, 1:].max(axis=1).argsort()[::-1]
    np.testing.assert_allclose(obj, objects[order], atol=1e-3)
    ref = ofr.rcnn_proposal(proposed, bbox_pred, cls_prob, (900, 1440), 3, cfg)
    np.testing.assert_array_equal(lab, ref['proposal_label'])
    np.testing.assert_array_equal(prob, ref['proposal_label_prob'])


@pytest.mark.parametrize('r,nc,min_prob', [(300, 80, 0.0), (2000, 20, 0.05), (50, 3, 0.5)])
def test_class_detections_rcnn_random(r, nc, min_prob):
    rng = np.random.default_rng(r + nc)
    props = _random_boxes(rng, r, 800.0)
    deltas = (rng.standard_normal((r, 4 * nc)) * 0.5).astype(np.float32)
    if r > 100:          # large cases: dw = dh = 0 keeps decode bit-reproducible (see the RPN full-size test)
        deltas.reshape(r, nc, 4)[:, :, 2:] = 0
    prob = T.softmax((rng.standard_normal((r, nc + 1)) * 2).astype(np.float32))
    cfg = {'class_max_detections': 100, 'class_nms_threshold': 0.5, 'total_max_detections': 300,
           'min_prob_threshold': min_prob}
    ref = ofr.rcnn_proposal(props, deltas, prob, (600, 1024), nc, cfg, variances=[0.1, 0.2])
    obj, lab, p = ops().class_detections(props, deltas, prob, (600, 1024), nc, cfg, [0.1, 0.2])
    np.testing.assert_array_equal(lab, ref['proposal_label'])
    np.testing.assert_array_equal(p, ref['proposal_label_prob'])
    np.testing.assert_allclose(obj, ref['objects'], atol=1e-3)


def test_class_detections_ssd_random():
    from oracle.anchors import ssd_anchors
    rng = np.random.default_rng(21)
    shapes = [(37, 37), (18, 18), (9, 9), (5, 5), (3, 3), (1, 1)]
    anchors = ssd_anchors(shapes, 0.1, 0.88, [1, 0.5, 2, 0.333, 3], [4, 6, 6, 6, 4, 4], [300, 300, 3])
    r = anchors.shape[0]
    assert r == 8096
    nc = 20
    loc = (rng.standard_normal((r, 4)) * 0.5).astype(np.float32)
    loc[:, 2:] = 0
    prob = T.softmax((rng.standard_normal((r, nc + 1)) * 3).astype(np.float32))
    cfg = {'class_max_detections': 100, 'class_nms_threshold': 0.45, 'total_max_detections': 100, 'min_prob_threshold': 0.3}
    ref = ossd.ssd_proposal(prob, loc, anchors, (300.0, 300.0), nc, cfg, [0.1, 0.2])
    obj, lab, p = ops().class_detections(anchors, loc, prob, (300, 300), nc, cfg, [0.1, 0.2], ssd=True)
    np.testing.assert_array_equal(lab, ref['labels'])
    np.testing.assert_array_equal(p, ref['probs'])
    np.testing.assert_allclose(obj, ref['objects'], atol=1e-3)
