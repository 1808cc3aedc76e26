"""Property tests that pin the ORACLE's third-party-op restatements (oracle/tf_ops.py) on independent, deliberately
naive scalar implementations written from the TF-1.x op semantics of SURVEY Appendix A -- the part of the path the
reference's own tests cannot pin because the arithmetic lives in TensorFlow (SURVEY 8c, mitigation iv)."""
import math

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

from luminoth_b200 import default_config, synth
from oracle import fasterrcnn as ofr
from oracle import tf_ops as T

SET = settings(max_examples=25, deadline=None)


def _same(in_size, k, stride, rate):
    k_eff = k + (k - 1) * (rate - 1)
    out = -(-in_size // stride)
    total = max((out - 1) * stride + k_eff - in_size, 0)
    return out, total // 2


@SET
@given(st.integers(1, 9), st.integers(1, 9), st.sampled_from([1, 3]), st.sampled_from([1, 2]), st.sampled_from([1, 2]),
       st.sampled_from(['SAME', 'VALID']), st.integers(0, 2 ** 31 - 1))
def test_conv2d_matches_scalar_loops(h, w, k, stride, rate, padding, seed):
    k_eff = k + (k - 1) * (rate - 1)
    if padding == 'VALID' and (h < k_eff or w < k_eff):
        return
    rng = np.random.default_rng(seed)
    cin, cout = 2, 3
    x = rng.standard_normal((1, h, w, cin))
    wt = rng.standard_normal((k, k, cin, cout))
    if padding == 'SAME':
        ho, pt = _same(h, k, stride, rate); wo, pl = _same(w, k, stride, rate)
    else:
        ho, pt = (h - k_eff) // stride + 1, 0; wo, pl = (w - k_eff) // stride + 1, 0
    ref = np.zeros((1, ho, wo, cout))
    for oy in range(ho):
        for ox in range(wo):
            for r in range(k):
                for s in range(k):
                    iy, ix = oy * stride + r * rate - pt, ox * stride + s * rate - pl
                    if 0 <= iy < h and 0 <= ix < w:
                        ref[0, oy, ox] += x[0, iy, ix] @ wt[r, s]
    got = T.conv2d(x, wt, stride, padding, rate)
    assert got.shape == ref.shape
    np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-10)


@SET
@given(st.integers(1, 10), st.integers(1, 10), st.sampled_from([2, 3]), st.sampled_from([1, 2]),
       st.sampled_from(['SAME', 'VALID']), st.integers(0, 2 ** 31 - 1))
def test_max_pool_matches_scalar_loops(h, w, k, stride, padding, seed):
    if padding == 'VALID' and (h < k or w < k):
        return
    x = np.random.default_rng(seed).standard_normal((1, h, w, 2))
    if padding == 'SAME':
        ho, pt = _same(h, k, stride, 1); wo, pl = _same(w, k, stride, 1)
    else:
        ho, pt, wo, pl = (h - k) // stride + 1, 0, (w - k) // stride + 1, 0
    ref = np.full((1, ho, wo, 2), -np.inf)
    for oy in range(ho):
        for ox in range(wo):
            for r in range(k):
                for s in range(k):
                    iy, ix = oy * stride + r - pt, ox * stride + s - pl
                    if 0 <= iy < h and 0 <= ix < w:              # TF ignores padded cells
                        ref[0, oy, ox] = np.maximum(ref[0, oy, ox], x[0, iy, ix])
    np.testing.assert_array_equal(T.max_pool(x, k, stride, padding), ref)


@SET
@given(st.integers(2, 7), st.integers(2, 7), st.integers(1, 5), st.integers(1, 5), st.integers(0, 2 ** 31 - 1))
def test_crop_and_resize_matches_scalar_kernel(H, W, ch, cw, seed):
    """tf.image.crop_and_resize (bilinear): in_y = y1 (H-1) + i (y2-y1)(H-1)/(ch-1) (midpoint when ch == 1), samples
    outside [0, H-1] give the extrapolation value, top/bottom = floor/ceil, horizontal lerp first."""
    rng = np.random.default_rng(seed)
    img = rng.standard_normal((1, H, W, 2))
    boxes = rng.uniform(-0.3, 1.3, (3, 4))
    got = T.crop_and_resize(img, boxes, np.zeros(3, np.int64), ch, cw, 0.0)
    for b, (y1, x1, y2, x2) in enumerate(boxes):
        for i in range(ch):
            in_y = y1 * (H - 1) + i * ((y2 - y1) * (H - 1) / (ch - 1)) if ch > 1 else 0.5 * (y1 + y2) * (H - 1)
            for j in range(cw):
                in_x = x1 * (W - 1) + j * ((x2 - x1) * (W - 1) / (cw - 1)) if cw > 1 else 0.5 * (x1 + x2) * (W - 1)
                if in_y < 0 or in_y > H - 1 or in_x < 0 or in_x > W - 1:
                    want = np.zeros(2)
                else:
                    t, bo = math.floor(in_y), math.ceil(in_y)
                    l, r = math.floor(in_x), math.ceil(in_x)
                    top = img[0, t, l] + (img[0, t, r] - img[0, t, l]) * (in_x - l)
                    bot = img[0, bo, l] + (img[0, bo, r] - img[0, bo, l]) * (in_x - l)
                    want = top + (bot - top) * (in_y - t)
                np.testing.assert_allclose(got[b, i, j], want, rtol=1e-10, atol=1e-12)


def _iou_tf(a, b):
    """TF's IOU on (y1,x1,y2,x2) boxes: coordinates normalised with min/max, no +1, 0 when an area is <= 0."""
    ya1, xa1, ya2, xa2 = min(a[0], a[2]), min(a[1], a[3]), max(a[0], a[2]), max(a[1], a[3])
    yb1, xb1, yb2, xb2 = min(b[0], b[2]), min(b[1], b[3]), max(b[0], b[2]), max(b[1], b[3])
    area_a, area_b = (ya2 - ya1) * (xa2 - xa1), (yb2 - yb1) * (xb2 - xb1)
    if area_a <= 0 or area_b <= 0:
        return 0.0
    ih = max(min(ya2, yb2) - max(ya1, yb1), 0.0); iw = max(min(xa2, xb2) - max(xa1, xb1), 0.0)
    inter = ih * iw
    return inter / (area_a + area_b - inter)


@SET
@given(st.integers(1, 40), st.floats(0.0, 1.0), st.integers(1, 40), st.integers(0, 2 ** 31 - 1))
def test_nms_matches_greedy_definition(n, thr, max_out, seed):
    """tf.image.non_max_suppression: visit boxes by descending score (ties: lower index first), keep a box unless
    its IoU with an already kept box is strictly greater than the threshold, stop at max_output_size."""
    rng = np.random.default_rng(seed)
    c = rng.integers(0, 12, (n, 2)).astype(np.float64); s = rng.integers(0, 8, (n, 2)).astype(np.float64)
    boxes = np.concatenate([c, c + s], 1)                         # integer grid: duplicates, zero areas, exact ties
    scores = rng.integers(0, 6, n).astype(np.float64)
    order = sorted(range(n), key=lambda i: (-scores[i], i))
    keep = []
    for i in order:
        if len(keep) >= max_out:
            break
        if all(not (_iou_tf(boxes[i], boxes[j]) > thr) for j in keep):
            keep.append(i)
    got = T.non_max_suppression(boxes, scores, max_out, thr)
    assert list(got) == keep


@SET
@given(st.integers(1, 60), st.integers(1, 60), st.integers(0, 2 ** 31 - 1))
def test_top_k_is_stable_descending(n, k, seed):
    v = np.random.default_rng(seed).integers(0, 5, n).astype(np.float32)
    k = min(k, n)
    vals, idx = T.top_k(v, k)
    want = sorted(range(n), key=lambda i: (-v[i], i))[:k]
    assert list(idx) == want and list(vals) == [v[i] for i in want]


@SET
@given(st.integers(1, 9), st.integers(1, 9), st.integers(1, 12), st.integers(1, 12), st.integers(0, 2 ** 31 - 1))
def test_resize_bilinear_matches_scalar_kernel(H, W, nh, nw, seed):
    """TF 1.x legacy bilinear resize: src = dst * (in / out), lower = floor(src), upper = min(lower + 1, in - 1)."""
    img = np.random.default_rng(seed).uniform(0, 255, (H, W, 3))
    got = T.resize_bilinear(img, nh, nw)
    for y in range(nh):
        fy = y * (H / nh); y0 = math.floor(fy); y1 = min(y0 + 1, H - 1)
        for x in range(nw):
            fx = x * (W / nw); x0 = math.floor(fx); x1 = min(x0 + 1, W - 1)
            top = img[y0, x0] + (img[y0, x1] - img[y0, x0]) * (fx - x0)
            bot = img[y1, x0] + (img[y1, x1] - img[y1, x0]) * (fx - x0)
            np.testing.assert_allclose(got[y, x], top + (bot - top) * (fy - y0), rtol=1e-12, atol=1e-9)


@pytest.mark.parametrize('arch,with_rcnn', [('resnet_v1_50', True), ('resnet_v1_101', True), ('resnet_v1_50', False)],
                         ids=['r50', 'r101', 'r50_rpn_only'])
def test_forward_on_an_image_without_proposals(arch, with_rcnn):
    """With filter_outside_anchors no anchor (the smallest is 64 px high) lies inside an image under 55 px high, so a
    40x640 image has no proposals.  The reference still runs its RCNN head on the empty list: tf.contrib.layers.flatten
    reshapes with the known inner size (rcnn.py:192) and the forward returns no detections.  At 55 px the anchors of
    the first row fit and the image has proposals again."""
    cfg = default_config('fasterrcnn', ['model.base_network.architecture=' + arch, 'model.network.num_classes=20',
                                        'model.rpn.proposals.post_nms_top_n=200',
                                        'model.rcnn.proposals.min_prob_threshold=0.05',
                                        'model.rpn.proposals.filter_outside_anchors=true',
                                        'model.network.with_rcnn=%s' % str(with_rcnn).lower()])
    wts = synth.make_weights(cfg, seed=1)
    out = ofr.forward(synth.make_images(1, 40, 640, seed=2)[0], wts, cfg)
    assert out['rpn_prediction']['proposals'].shape == (0, 4)
    if with_rcnn:
        det = out['classification_prediction']
        assert det['objects'].shape == (0, 4) and len(det['labels']) == 0 and len(det['probs']) == 0
        assert out['rcnn']['cls_prob'].shape == (0, 21) and out['rcnn']['bbox_offsets'].shape == (0, 80)
    else:
        assert 'classification_prediction' not in out
    assert len(ofr.forward(synth.make_images(1, 55, 640, seed=2)[0], wts, cfg)['rpn_prediction']['proposals']) > 0
