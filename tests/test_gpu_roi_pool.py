"""The ROI crop-and-pool kernels and the RCNN head stages around them, at the engine's batched layout, against a
float64 reference (`-m gpu`, needs an H100).

Reference.  The sample tables follow TF's crop_and_resize arithmetic in float32, exactly as the kernels and the
oracle compute them (box / image size, then (hi - lo) * (D - 1) / (crop - 1) and lo * (D - 1) + k * step, each
rounded): a float64 coordinate can move a sample across a cell boundary.  The taps, the bilinear interpolation with
those float32 weights, the 2x2 max and the mean are then float64.

Bound.  u = 2^-24.  Let M be the largest |tap| of one sample.  A kernel lerp h = fmaf(r - l, t, l) rounds twice:
|h^ - h| <= u |r - l| t + u |h| (1 + 2u) <= 3uM (1 + u).  The vertical lerp v = fmaf(b - t, ly, t) of two such values
carries their error (<= 3uM (1 + u), a convex combination) and adds u |b^ - t^| ly + u |v^| <= 3uM (1 + 3u).  So a
sample is within 6uM (1 + 4u) of the exact bilinear value; doing the same with separate operations, as the fp32 oracle
does, would round up to three times per lerp and needs 10uM.  A max is exact, so a pooled cell is within E = 6u (1 + 4u)
max M over its four samples (plus 2^-50 M for the float64 reference itself).  The mean adds the fp32 sum of the ncell
cells in any order, <= 1.01 (ncell - 1) u sum |p| (first order in u, ncell <= 256), and the division, u |m|.  Every
output then goes through the fp16x2 split (DESIGN section 2): |x - (hi + lo)| <= 2^-22 |x| + 2^-25.  One wrong tap or
weight moves a value by about |tap difference| * weight, orders of magnitude beyond this.

Every kernel instance runs every case whose shape it takes; the instances that refuse a case must be exactly those
whose preconditions fail.  All instances lerp horizontally, then vertically, with the same fmaf and take exact
maxima, so their pooled outputs must be bit-identical; their means sum in different orders and are held to the
bound only.  Padded rows (r >= counts[img]) get NaN and huge coordinates and must come out exactly 0, and the split
planes start as NaN, so a skipped write cannot pass.  LUMI_ROI_REPORT=<path> writes the largest err / bound ratio of
every check and the kernels each case ran as JSON.
"""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from luminoth_b200 import default_config, synth
from luminoth_b200.engine import Engine
from oracle import fasterrcnn as ofr

F32 = np.float32
U = 2.0 ** -24
ROWS6, ROWS5, ROWS4, COLS4, COLS8, CELLS844, CELLS848, CELLS818, CELLS418 = range(9)
CODES = range(9)
NAMES = ['rows<minb6>', 'rows<minb5>', 'rows<minb4>', 'cols<4>', 'cols<8>', 'cells<8,4,4>', 'cells<8,4,8>',
         'cells<8,1,8>', 'cells<4,1,8>']

REPORT = {}


def _report(key, **vals):
    REPORT[key] = vals
    path = os.environ.get('LUMI_ROI_REPORT')
    if path:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, 'w') as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)


def ops():
    import gpu_ops
    return gpu_ops


def fits(k, c, ph, pw):
    """The shape preconditions of instance k (roi.cu: roi_kernel_fits): crop_h = 2 pw, samples = 2 (ph + pw)."""
    if c % 8 or ph < 1 or pw < 1 or 2 * (ph + pw) > 64:
        return False
    ch, ns = 2 * pw, 2 * (ph + pw)
    return {ROWS6: ch <= 16 and ns <= 32, ROWS5: ch <= 16 and ns <= 32, ROWS4: ch <= 16 and ns <= 32,
            COLS4: ns <= 32, COLS8: ns <= 32, CELLS844: ns <= 32, CELLS848: True, CELLS818: True,
            CELLS418: True}[k]


def split_err(a):
    return 2.0 ** -22 * a + 2.0 ** -25


# ---------------------------------------------------------------- reference
def axis_table(lo_px, hi_px, im_len, D, crop):
    """One axis of TF's crop_and_resize sample table, in float32: (low index, high index, weight, inside) [R, crop]."""
    lo_n = lo_px.astype(F32) / F32(im_len)
    hi_n = hi_px.astype(F32) / F32(im_len)
    dm1 = F32(D - 1)
    step = (hi_n - lo_n) * dm1 / F32(crop - 1)                       # crop = 2 * pooled >= 2
    pos = (lo_n * dm1)[:, None] + np.arange(crop, dtype=F32)[None, :] * step[:, None]
    ok = ~((pos < 0) | (pos > dm1))
    pos = np.where(ok, pos, F32(0))
    lo = np.floor(pos).astype(np.int64)
    hi = np.ceil(pos).astype(np.int64)
    t = (pos - lo.astype(F32)).astype(F32)
    return lo, hi, t.astype(np.float64), ok


def reference(fmap, rois, counts, im_shape, ph, pw):
    """fmap [n, fh, fw, c] float32, rois [n, rmax, 4] (x1, y1, x2, y2) px.  Returns float64 (pooled, pooled bound,
    mean, mean bound) over the n * rmax rows; rows past counts[img] are NaN."""
    n, fh, fw, c = fmap.shape
    rmax = rois.shape[1]
    ch, cw, ncell = 2 * pw, 2 * ph, pw * ph
    pooled = np.full((n * rmax, pw, ph, c), np.nan)
    pbound = np.full_like(pooled, np.nan)
    mean = np.full((n * rmax, c), np.nan)
    mbound = np.full_like(mean, np.nan)
    chunk = max(1, int(4e6 // (ch * cw * c)))
    for img in range(n):
        live = rmax if counts is None else int(counts[img])
        fm = fmap[img].astype(np.float64)
        for r0 in range(0, live, chunk):
            rr = rois[img, r0:min(live, r0 + chunk)]
            R = rr.shape[0]
            ylo, yhi, yt, yok = axis_table(rr[:, 1], rr[:, 3], im_shape[0], fh, ch)
            xlo, xhi, xt, xok = axis_table(rr[:, 0], rr[:, 2], im_shape[1], fw, cw)
            tl = fm[ylo[:, :, None], xlo[:, None, :]]                  # [R, ch, cw, c]
            tr = fm[ylo[:, :, None], xhi[:, None, :]]
            bl = fm[yhi[:, :, None], xlo[:, None, :]]
            br = fm[yhi[:, :, None], xhi[:, None, :]]
            xw, yw = xt[:, None, :, None], yt[:, :, None, None]
            top = tl + (tr - tl) * xw
            bot = bl + (br - bl) * xw
            ok = (yok[:, :, None] & xok[:, None, :])[..., None]
            val = np.where(ok, top + (bot - top) * yw, 0.0)            # extrapolation_value = 0
            M = np.where(ok, np.maximum(np.maximum(np.abs(tl), np.abs(tr)), np.maximum(np.abs(bl), np.abs(br))), 0.0)
            p = val.reshape(R, pw, 2, ph, 2, c).max(axis=(2, 4))
            E = (6 * U * (1 + 4 * U) + 2.0 ** -50) * M.reshape(R, pw, 2, ph, 2, c).max(axis=(2, 4))
            rows = slice(img * rmax + r0, img * rmax + r0 + R)
            pooled[rows] = p
            pbound[rows] = E + split_err(np.abs(p) + E)
            m = p.mean(axis=(1, 2))
            e_sum = (E.sum(axis=(1, 2)) + 1.01 * (ncell - 1) * U * (np.abs(p) + E).sum(axis=(1, 2))) / ncell
            e = e_sum + U * (np.abs(m) + e_sum)
            mean[rows] = m
            mbound[rows] = e + split_err(np.abs(m) + e)
    return pooled, pbound, mean, mbound


def live_mask(n, rmax, counts):
    live = np.ones((n, rmax), bool)
    if counts is not None:
        live &= np.arange(rmax)[None, :] < np.asarray(counts)[:, None]
    return live.reshape(-1)


def err_ratio(got, ref, bound):
    assert np.isfinite(got).all(), 'non-finite output (a skipped write leaves the NaN sentinel)'
    return float((np.abs(got.astype(np.float64) - ref) / bound).max()) if got.size else 0.0


# ---------------------------------------------------------------- cases
def random_rois(rng, n, rmax, im_h, im_w):
    """Boxes of 1..im size, some reaching past the image, some inverted, a few degenerate (x1 == x2)."""
    cy, cx = rng.uniform(-0.1, 1.1, (n, rmax)) * im_h, rng.uniform(-0.1, 1.1, (n, rmax)) * im_w
    hh, hw = rng.uniform(0.5, 0.6 * im_h, (n, rmax)), rng.uniform(0.5, 0.6 * im_w, (n, rmax))
    rois = np.stack([cx - hw, cy - hh, cx + hw, cy + hh], -1)
    flip = rng.random((n, rmax)) < 0.1
    rois[flip] = rois[flip][:, [2, 3, 0, 1]]
    rois[:, 0] = [0, 0, im_w, im_h]                                    # the whole image: first / last row and column
    if rmax > 2:
        rois[:, 1] = [im_w * 0.3, im_h * 0.3, im_w * 0.3, im_h * 0.7]  # zero width
    return rois.astype(F32)


def pad_rows(rois, counts):
    """Rows past counts[img]: NaN and huge coordinates, which a live row would turn into NaN or far-off taps."""
    if counts is None:
        return rois
    rois = rois.copy()
    for img, k in enumerate(counts):
        rois[img, k:] = [np.nan, -3e38, 3e38, np.nan] if img % 2 else [1e30, 1e30, -1e30, 1e30]
    return rois


def aligned_rois(ph, pw, im, fh):
    """Boxes on a map of fh x fh cells over an im x im image (fh - 1 a power of two dividing im): with box corners on
    cell multiples, every sample coordinate lies on an integer (t = 0, the high tap read with weight 0), and the row /
    column steps of 1/4, 1/2, 1, 2 and 3 cells exercise reuse, one-row advance and reload.  Boxes end on the last row /
    column, start above / left of the map (outside rows, then inside ones), end below / right of it, and run inverted."""
    px = im / (fh - 1)                                                  # pixels per cell
    sy, sx = (2 * pw - 1) * px, (2 * ph - 1) * px                       # box height / width of a one-cell step
    out = []
    for s in (0.25, 0.5, 1.0, 2.0, 3.0):
        for y0, x0 in ((0, 0), (2, 1), (None, None)):
            if y0 is None:                                              # end exactly on the last row / column
                out.append([im - s * sx, im - s * sy, im, im])
            else:
                out.append([x0 * px, y0 * px, x0 * px + s * sx, y0 * px + s * sy])
    out += [[-3 * px, -5 * px, -3 * px + sx, -5 * px + 2 * sy],        # prefix of rows / columns outside the map
            [im - 2 * px, im - 3 * px, im - 2 * px + 2 * sx, im - 3 * px + sy],  # suffix outside
            [-2 * px, -2 * px, im + 2 * px, im + 2 * px],               # both
            [im, im, 0, 0], [5 * px + sx, 4 * px, 5 * px, 4 * px + sy],  # inverted
            [-20 * px, -20 * px, -10 * px, -10 * px]]                   # wholly outside: every sample extrapolated
    return np.asarray(out, F32)


# name: (n, fh, fw, c, rmax, counts, ph, pw, outputs, features, rois, engine's code, seed)
CASES = {
    'p7_c256_3img': (3, 12, 17, 256, 24, [24, 0, 5], 7, 7, 'both', 'randn', 'random', ROWS6, 1),
    'p7_c1024_2img': (2, 9, 14, 1024, 8, [8, 3], 7, 7, 'both', 'randn', 'random', ROWS6, 2),
    'p7_c136_pooled_only': (2, 10, 10, 136, 12, [5, 12], 7, 7, 'pooled', 'randn', 'random', ROWS6, 3),
    'p7_c264_mean_only': (3, 10, 13, 264, 10, [10, 0, 2], 7, 7, 'mean', 'randn', 'random', ROWS6, 4),
    'p2_c8': (1, 10, 10, 8, 16, None, 2, 2, 'both', 'randn', 'random', ROWS6, 5),
    'p8_c136': (2, 11, 13, 136, 12, [12, 7], 8, 8, 'both', 'randn', 'random', ROWS6, 6),
    'p7x9_c264': (3, 12, 15, 264, 10, [10, 0, 3], 9, 7, 'both', 'randn', 'random', ROWS6, 7),
    'p9x7_c264': (3, 12, 15, 264, 10, [10, 0, 3], 7, 9, 'both', 'randn', 'random', CELLS844, 8),
    'p5x3_c136': (2, 9, 9, 136, 12, [12, 4], 3, 5, 'both', 'randn', 'random', ROWS6, 9),
    'p9x5_c1024': (2, 9, 14, 1024, 8, [8, 3], 5, 9, 'both', 'randn', 'random', CELLS844, 10),
    'p9x5_c256_mean_only': (2, 9, 14, 256, 8, [6, 8], 5, 9, 'mean', 'randn', 'random', CELLS844, 11),
    'p16_c256': (2, 14, 18, 256, 6, [6, 2], 16, 16, 'both', 'randn', 'random', CELLS848, 12),
    'p31x1_c8': (1, 12, 12, 8, 10, [7], 1, 31, 'both', 'randn', 'random', CELLS848, 13),
    'p1x31_c8': (1, 12, 12, 8, 10, [7], 31, 1, 'both', 'randn', 'random', CELLS848, 14),
    'fh1_c136': (2, 1, 9, 136, 10, [10, 4], 7, 7, 'both', 'randn', 'random', ROWS6, 15),
    'fw1_c136': (2, 9, 1, 136, 10, [10, 4], 7, 7, 'both', 'randn', 'random', ROWS6, 16),
    'fh1_fw1_p9x5': (1, 1, 1, 264, 6, None, 5, 9, 'both', 'randn', 'random', CELLS844, 17),
    'aligned_p7_negative': (2, 33, 33, 136, 21, [21, 9], 7, 7, 'both', 'negative', 'aligned', ROWS6, 18),
    'aligned_p9x5_negative': (1, 33, 33, 264, 21, None, 5, 9, 'both', 'negative', 'aligned', CELLS844, 19),
    'aligned_p5x3_negative': (1, 17, 17, 8, 21, None, 3, 5, 'both', 'negative', 'aligned', ROWS6, 20),
    'aligned_p8_mixed': (1, 33, 33, 256, 21, [15], 8, 8, 'both', 'randn', 'aligned', ROWS6, 21),
}
# each instance must run at least this many cases (a refusal cannot hollow out the matrix)
MIN_RUNS = {ROWS6: 13, ROWS5: 13, ROWS4: 13, COLS4: 18, COLS8: 18, CELLS844: 18, CELLS848: 21, CELLS818: 21,
            CELLS418: 21}
RUNS = {k: [] for k in CODES}
IDENTICAL = {}


def build_case(name):
    n, fh, fw, c, rmax, counts, ph, pw, outputs, feats, kind, _, seed = CASES[name]
    rng = np.random.default_rng(seed)
    fmap = rng.standard_normal((n, fh, fw, c)).astype(F32)
    if feats == 'negative':               # resnet_v2 endpoints are pre-activation sums: the max can be below 0
        fmap = -np.abs(fmap) - F32(0.25)
    if kind == 'aligned':
        im = 512 if fh == 33 else 256
        one = aligned_rois(ph, pw, im, fh)
        assert one.shape[0] == rmax
        rois = np.stack([one] * n)
        im_shape = (im, im)
    else:
        im_shape = (16 * fh + 5, 16 * fw - 3)
        rois = random_rois(rng, n, rmax, *im_shape)
    return fmap, pad_rows(rois, counts), counts, im_shape, ph, pw, outputs


@pytest.mark.parametrize('name', list(CASES))
def test_roi_pool_every_instance(name):
    fmap, rois, counts, im_shape, ph, pw, outputs = build_case(name)
    n, fh, fw, c = fmap.shape
    rmax = rois.shape[1]
    want_code = CASES[name][11]
    assert ops().roi_kernel(c, ph, pw) == want_code, 'the engine would run %s' % NAMES[ops().roi_kernel(c, ph, pw)]
    ref_p, bnd_p, ref_m, bnd_m = reference(fmap, rois, counts, im_shape, ph, pw)
    live = live_mask(n, rmax, counts)
    first, ran, worst_p, worst_m = None, [], 0.0, 0.0
    for k in CODES:
        if not fits(k, c, ph, pw):
            with pytest.raises(RuntimeError, match='does not take'):
                ops().roi_pool_batched(fmap, rois, counts, im_shape, ph, pw, kernel=k)
            continue
        y, m = ops().roi_pool_batched(fmap, rois, counts, im_shape, ph, pw, kernel=k,
                                      pooled=outputs != 'mean', mean=outputs != 'pooled')
        y = y.cpu().numpy() if y is not None else None
        m = m.cpu().numpy() if m is not None else None
        if y is not None:
            assert (y[~live] == 0).all(), '%s: padded pooled rows are not 0' % NAMES[k]
            r = err_ratio(y[live], ref_p[live], bnd_p[live])
            assert r <= 1, '%s: pooled err / bound %.3g' % (NAMES[k], r)
            worst_p = max(worst_p, r)
            if first is None:
                first = (k, y)
            else:
                assert np.array_equal(y, first[1]), '%s and %s pooled outputs differ: max %.3g' % (
                    NAMES[first[0]], NAMES[k], np.abs(y - first[1]).max())
        if m is not None:
            assert (m[~live] == 0).all(), '%s: padded mean rows are not 0' % NAMES[k]
            r = err_ratio(m[live], ref_m[live], bnd_m[live])
            assert r <= 1, '%s: mean err / bound %.3g' % (NAMES[k], r)
            worst_m = max(worst_m, r)
        ran.append(k)
        RUNS[k].append(name)
    IDENTICAL[name] = first is not None and len(ran) > 1
    _report('case/' + name, engine_kernel=NAMES[want_code], kernels=[NAMES[k] for k in ran],
            pooled_err_over_bound=worst_p, mean_err_over_bound=worst_m,
            pooled_bit_identical_across=len(ran) if first is not None else 0)


def test_every_instance_ran_enough_cases():
    """Runs after the case matrix (file order): each instance ran at least MIN_RUNS cases."""
    if len(set().union(*RUNS.values())) < len(CASES):
        pytest.skip('needs the whole case matrix in this session')
    short = {NAMES[k]: len(v) for k, v in RUNS.items() if len(v) < MIN_RUNS[k]}
    assert not short, 'instances that ran too few cases: %s' % short
    assert sum(IDENTICAL.values()) >= 18
    _report('instances', **{NAMES[k]: len(v) for k, v in RUNS.items()})


def test_roi_pool_production_size():
    """2 images x 2000 rois on a 38 x 64 x 1024 map (a 600 x 1024 image at stride 16), the second image with 1700 live
    rows: every instance bit-identical to the row-walk kernel, a sample of 96 rows against the reference."""
    rng = np.random.default_rng(40)
    n, fh, fw, c, rmax, counts, im_shape = 2, 38, 64, 1024, 2000, [2000, 1700], (600, 1024)
    fmap = rng.standard_normal((n, fh, fw, c)).astype(F32)
    rois = pad_rows(random_rois(rng, n, rmax, *im_shape), counts)
    assert ops().roi_kernel(c, 7, 7) == ROWS6
    live = live_mask(n, rmax, counts)
    sample = np.stack([rng.choice(k, 48, replace=False) for k in counts])          # [n, 48] live rows
    ref_p, bnd_p, ref_m, bnd_m = reference(fmap, np.stack([rois[i, sample[i]] for i in range(n)]), None, im_shape, 7, 7)
    rows = (np.arange(n)[:, None] * rmax + sample).reshape(-1)
    rows_d = torch.from_numpy(rows).cuda()
    fd, rd = torch.from_numpy(fmap).cuda(), torch.from_numpy(rois).cuda()
    y0, m0 = ops().roi_pool_batched(fd, rd, counts, im_shape, 7, 7, kernel=ROWS6)
    pad = torch.from_numpy(~live).cuda()
    assert bool((y0[pad] == 0).all()) and bool((m0[pad] == 0).all())
    rp = err_ratio(y0[rows_d].cpu().numpy(), ref_p, bnd_p)
    rm = err_ratio(m0[rows_d].cpu().numpy(), ref_m, bnd_m)
    assert rp <= 1 and rm <= 1, (rp, rm)
    worst_m = rm
    for k in CODES[1:]:
        y, m = ops().roi_pool_batched(fd, rd, counts, im_shape, 7, 7, kernel=k)
        assert torch.equal(y, y0), '%s pooled differs from rows<minb6>' % NAMES[k]
        assert bool((m[pad] == 0).all())
        r = err_ratio(m[rows_d].cpu().numpy(), ref_m, bnd_m)
        assert r <= 1, '%s: mean err / bound %.3g' % (NAMES[k], r)
        worst_m = max(worst_m, r)
        del y, m
    _report('production_2x2000_c1024', pooled_err_over_bound=rp, mean_err_over_bound=worst_m,
            pooled_bit_identical_across=len(CODES))


# ---------------------------------------------------------------- RCNN head stages
def split_join(x):
    """The fp32 value the engine's split planes hold for x (hi = fp16(x), lo = fp16(x - hi))."""
    hi = x.astype(np.float16)
    lo = (x - hi.astype(F32)).astype(np.float16)
    return hi.astype(F32) + lo.astype(F32)


@pytest.mark.parametrize('r,h,w,c', [(24, 7, 7, 2048), (40, 1, 1, 1024), (16, 5, 9, 264), (8, 16, 16, 136)])
def test_spatial_mean(r, h, w, c):
    """The engine's mean after the resnet_v1_101 tail: fp32 sum of h*w split-plane values, divided, split again."""
    rng = np.random.default_rng(r * c + h)
    x = (rng.standard_normal((r, h, w, c)) * rng.choice([1e-3, 1.0, 30.0], (r, 1, 1, c))).astype(F32)
    xs = split_join(x).astype(np.float64)
    ref = xs.mean(axis=(1, 2))
    hw = h * w
    e = 1.01 * (hw - 1) * U * np.abs(xs).sum(axis=(1, 2)) / hw
    e = e + U * (np.abs(ref) + e)
    bound = e + split_err(np.abs(ref) + e)
    got = ops().spatial_mean(x)
    ratio = err_ratio(got, ref, bound)
    _report('spatial_mean/%dx%dx%dx%d' % (r, h, w, c), err_over_bound=ratio)
    assert ratio <= 1, ratio


@pytest.mark.parametrize('cols', [2, 21, 81, 91])
def test_softmax_rows(cols):
    """Softmax over the C + 1 class logits of fc rows 5C + 1 wide (C = cols - 1), logits up to +-1e4 and rows of equal
    logits, against float64.

    Bound, per element, with d = x - max: fl(d) is within u |d| of d, so exp(fl(d)) within u |d| (relative, first order)
    of exp(d), and expf adds at most 2 ulp (4u relative).  The sum s runs ceil(cols / 32) - 1 adds per lane plus 5
    shuffle levels over positive terms, each e_k already off by (|d_k| + 4) u: relative error <= (depth + 1) u +
    sum e_k (|d_k| + 4) u / sum e_k.  The division adds u.  Below 2^-126 an expf result is subnormal: 2^-147 absolute."""
    rng = np.random.default_rng(cols)
    rows, stride = 64, 5 * (cols - 1) + 1
    x = rng.standard_normal((rows, stride)).astype(F32)
    x[:16, :cols] *= F32(10.0)
    x[16:32, :cols] *= F32(1e4)                                        # one logit dominates; others underflow
    x[32:40, :cols] = F32(3.5)                                         # all equal
    x[40:44, :cols] = F32(-1e4)
    x[44:48, :cols] = rng.choice([-1e4, 1e4], (4, cols)).astype(F32)
    x[48:56, :cols] = (rng.standard_normal((8, cols)) * 60).astype(F32)   # values near the underflow edge
    x[:, cols:] = np.nan                                               # bbox columns of the fc row: never read
    got = ops().softmax_rows(x, cols)
    xl = x[:, :cols].astype(np.float64)
    d = xl - xl.max(axis=1, keepdims=True)
    e = np.exp(d)
    ref = e / e.sum(axis=1, keepdims=True)
    depth = -(-cols // 32) - 1 + 5
    s_rel = (depth + 1) * U + (e * (np.abs(d) + 4) * U).sum(axis=1, keepdims=True) / e.sum(axis=1, keepdims=True)
    rel = (np.abs(d) + 4) * U + s_rel + U
    bound = 1.01 * rel * ref + 2.0 ** -147
    ratio = err_ratio(got, ref, bound)
    _report('softmax_rows/%d' % cols, err_over_bound=ratio)
    assert ratio <= 1, ratio
    np.testing.assert_array_equal(got[32:40], np.full((8, cols), F32(1.0) / F32(cols)))


# ---------------------------------------------------------------- engine level
def frcnn_cfg(extra=()):
    return default_config('fasterrcnn', ['model.base_network.architecture=resnet_v1_50', 'model.network.num_classes=20',
                                         'model.rpn.proposals.post_nms_top_n=600'] + list(extra))


def run_engine(cfg, seed, h=96, w=128):
    """Two images small enough that every count stays below post_nms_top_n (6 x 8 cells x 12 anchors = 576 < 600)."""
    wts = synth.make_weights(cfg, seed=seed)
    imgs = synth.make_images(2, h, w, seed=seed + 1)
    eng = Engine(cfg, max_batch=2, max_h=h, max_w=w)
    eng.load_weights(wts).finalize()
    eng.set_debug_taps(True)
    eng.predict_raw(imgs)
    taps = {k: eng.get_tensor(k) for k in ('conv_feature_map', 'proposals', 'proposal_counts', 'roi_pool',
                                           'rcnn_features', 'rcnn_cls_prob')}
    eng.close()
    taps['proposal_counts'] = taps['proposal_counts'].astype(int).reshape(-1)
    assert (taps['proposal_counts'] < 600).all() and (taps['proposal_counts'] > 0).all(), taps['proposal_counts']
    return wts, (h, w), taps


def test_engine_fused_mean_matches_its_roi_pool_tap():
    """R50 at 7 x 7: one launch writes the roi_pool tap and the fused mean.  Each rcnn_features row is the float64 mean
    of its 49 tap cells within the bound (the tap holds the split of each cell, so its own split error is added), and
    the padded rows of both are exactly 0."""
    wts, im, t = run_engine(frcnn_cfg(), seed=3)
    cnt, post = t['proposal_counts'], 600
    pooled = t['roi_pool'].reshape(2 * post, 49, 1024).astype(np.float64)
    feats = t['rcnn_features'].reshape(2 * post, 1024)
    live = live_mask(2, post, cnt)
    assert (pooled[~live] == 0).all() and (feats[~live] == 0).all()
    p = pooled[live]
    ref = p.mean(axis=1)
    pa = np.abs(p) * (1 + 2.0 ** -21) + 2.0 ** -25                   # >= |the fp32 cell value the tap holds the split of|
    e = (split_err(pa).sum(axis=1) + 1.01 * 48 * U * pa.sum(axis=1)) / 49
    e = e + U * (np.abs(ref) + e)
    bound = e + split_err(np.abs(ref) + e)
    ratio = err_ratio(feats[live], ref, bound)
    _report('engine/r50_7x7_fused_mean', err_over_bound=ratio, counts=cnt.tolist())
    assert ratio <= 1, ratio


@pytest.mark.parametrize('use_mean', [True, False])
def test_engine_pooled_9x5_runs_the_cell_kernel(use_mean):
    """pooled_width 9, pooled_height 5: crop_h 18 rules out the row walk, so the engine runs cells<8,4,4>.  The roi_pool
    tap against the reference on the engine's own feature map and proposals; cls_prob against the oracle head fed the
    oracle's roi_pool of the same proposals."""
    assert ops().roi_kernel(1024, 5, 9) == CELLS844
    cfg = frcnn_cfg(['model.rcnn.roi.pooled_width=9', 'model.rcnn.roi.pooled_height=5',
                     'model.rcnn.use_mean=%s' % use_mean])
    wts, im, t = run_engine(cfg, seed=5)
    cnt, post = t['proposal_counts'], 600
    fmap, props = t['conv_feature_map'], t['proposals'].reshape(2, post, 4)
    pooled = t['roi_pool'].reshape(2 * post, 9, 5, 1024)
    live = live_mask(2, post, cnt)
    assert (pooled[~live] == 0).all()
    ref_p, bnd_p, _, _ = reference(fmap, props, cnt, im, 5, 9)
    ratio = err_ratio(pooled[live], ref_p[live], bnd_p[live])
    worst_prob = 0.0
    for i in range(2):
        k = int(cnt[i])
        roi_ref = ofr.roi_pool(props[i, :k], fmap[i][None], im, 9, 5)['roi_pool']
        head = ofr.rcnn_head(roi_ref, wts, cfg['model']['rcnn'], 'resnet_v1_50')
        dp = float(np.abs(t['rcnn_cls_prob'][i, :k] - head['cls_prob']).max())
        worst_prob = max(worst_prob, dp)
    _report('engine/r50_9x5_use_mean_%s' % use_mean, roi_pool_err_over_bound=ratio, cls_prob_abs=worst_prob,
            counts=cnt.tolist())
    assert ratio <= 1, ratio
    assert worst_prob <= 3e-5, worst_prob
