"""Conv kernels at the edges of the fp16x2 split, held to a per-element error bound (`-m gpu`, needs an H100).

Every case runs through `lumi_op_conv2d_io` on the SIMT kernel (impl 0: fp32 outputs, 13: split planes) and the
tensor-core kernel (1 / 2: fp32 outputs, whole tiles / stream-K; 3 / 4 / 5: split planes through the slot epilogue,
two consumer warpgroups / four allowed up to the engine's 16 K slices / four + stream-K; 12: the register epilogue;
6 / 7: 2-CTA clusters), all on the engine's single-buffered mainloop, and is compared with a float64 reference
computed from the fp32 inputs.  test_gpu_conv_engine_layers runs the engine's own launch (codes 16-19) of every
production layer against the same bound, evaluated at sampled pixels (`reference(..., at=...)`).

The bound
---------
Per output element,  |y - ref| <= alpha * S + beta * W + V + delta,  with
  S = |s| * sum |x||w| + |b| + |r|      (T.conv2d(|x|, |w|) over the taps inside the map)
  W = |s| * sum |w|                     (T.conv2d(ones, |w|): the same taps)
  V = (2^-25 |s| 2^-e[c] + 2^-150 2^e[c] max|w[:, c]|) * sum |x|      (tensor cores only, T.conv2d(|x|, ones))
and the constants from the error terms, u = 2^-24 being fp32's unit roundoff:
* The activation split x^ = hi + lo (input and residual): |x^ - x| <= 2^-22 |x| while lo is a normal fp16; below
  |x| = 2^-3 lo is subnormal and the error is an absolute 2^-25.  The relative part is 2^-22 in alpha, the floor
  2^-25 * |w| per tap is beta * W with beta = 2^-25, and the residual's floor is 2^-25 in delta.
* The weight split (tensor cores): hi + lo of w * 2^e[c] keeps 2^-22 relative (alpha) with an absolute floor of
  2^-25 in units of 2^e[c], i.e. 2^-25 * 2^-e[c] per weight: the first part of V.  A clamped column (e = 126) with
  |s| < 1 has a subnormal scale_tc, off by up to 2^-150 times |acc| <= 2^e max|w| sum|x|: the second part of V.
* The dropped lo * lo product: 2^-22 |x||w| (alpha).
* The 64-deep slice chains: the tensor core's own fp32 additions are not IEEE round-to-nearest.  The bound allows
  each wgmma's addition 2^-21 of the magnitudes it sums (two ulps: the alignment of the products and the final
  rounding), for the four hi * hi wgmma of a slice that is 4 * 2^-21 = 8 * 2^-22 of the slice's sum |x||w| (the eight
  cross-term wgmma act on 2^-10 of that and are absorbed in the 1 % slack below).
* The K / 64 fp32 folds of the slice tiles into the running sum (and the stream-K partial sums: a tree of the same
  number of additions): ceil(K / 64) * u of sum |x||w|.  On the SIMT kernel the whole K-deep fp32 FMA chain instead:
  K * u.
* The epilogue: fmaf(acc, s, b) and the residual's two additions, 3 u of S; the output's own split (split outputs;
  added for every impl), 2^-22 of S plus an absolute 2^-25 (delta).
So alpha = 1.01 * (2^-22 * (3 + 8 + 1) + u * (ceil(K / 64) + 3)) on the tensor cores, 1.01 * (2^-22 * 2 + u * (K + 3))
on the SIMT kernel, beta = 1.01 * 2^-25, delta = 2^-25 (+ 2^-25 with a residual).  These are worst-case bounds, not
fitted to results: each case prints its largest err / bound (run with -s).  On an H100 the largest ratios are about
0.44 (channel scales from 1e-4 to 1e4), 0.3 (the pre-activation output) and 0.18 (1e-3 activations, where the split
floor decides); long-K cases sit near 1e-3, the linear chain terms being far above the typical random-walk error.

The pre-activation output p = relu(fmaf(x^, ps, pb)) is held to |ps| * bound(x) + (u + 2^-22) (|ps| |x| + |pb|)
+ 2^-25: the error of the x it reads, its own fmaf and its own split.
"""
import ctypes
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import gpu_ops as G
from luminoth_b200.engine import LUMI_EOVERFLOW
from oracle import tf_ops as T

f16, f32, f64 = np.float16, np.float32, np.float64
U = 2.0 ** -24

FP32_IMPLS = [0, 1, 2]
SPLIT_IMPLS = [13, 3, 4, 5, 12, 6, 7]
IMPLS = [0, 13, 1, 2, 3, 4, 5, 12, 6, 7]
PREACT_IMPLS = SPLIT_IMPLS            # 13: the SIMT kernel writing split planes

PAD = {'VALID': 0, 'SAME': 1, 'SLIM': 2}


def conv_io(x, w, stride=1, padding='SAME', scale=None, bias=None, residual=None, res_stride=1, act=0, impl=0,
            pre=None, want_x=True):
    """lumi_op_conv2d_io -> (rc, y or None, p or None); rc == LUMI_EOVERFLOW returns no outputs."""
    import torch
    lib = G._lib()
    n, h, wd, cin = x.shape
    kh, kw, _, cout = w.shape
    xd, wdv = G._dev(x, f32), G._dev(w, f32)
    sd = G._dev(scale, f32) if scale is not None else None
    bd = G._dev(bias, f32) if bias is not None else None
    rd = G._dev(residual, f32) if residual is not None else None
    rh, rw = (residual.shape[1], residual.shape[2]) if residual is not None else (0, 0)
    psd, pbd = (G._dev(pre[0], f32), G._dev(pre[1], f32)) if pre is not None else (None, None)
    ho, wo = ctypes.c_int(), ctypes.c_int()
    args = [G._p(xd), n, h, wd, cin, G._p(wdv), kh, kw, cout, stride, 1, PAD[padding], G._p(sd), G._p(bd), G._p(rd),
            rh, rw, res_stride, act, impl, G._p(psd), G._p(pbd)]
    G._check(lib.lumi_op_conv2d_io(*args, None, None, ctypes.byref(ho), ctypes.byref(wo), None))
    shape = (n, ho.value, wo.value, cout)
    y = torch.empty(shape, dtype=torch.float32, device='cuda') if want_x else None
    p = torch.empty(shape, dtype=torch.float32, device='cuda') if pre is not None else None
    rc = lib.lumi_op_conv2d_io(*args, G._p(y), G._p(p), ctypes.byref(ho), ctypes.byref(wo), None)
    if rc == LUMI_EOVERFLOW:
        return rc, None, None
    G._check(rc)
    torch.cuda.synchronize()
    return rc, (y.cpu().numpy() if y is not None else None), (p.cpu().numpy() if p is not None else None)


def _conv64(x, w, stride, padding):
    x, w = np.asarray(x, f64), np.asarray(w, f64)
    return T.conv2d_same(x, w, stride) if padding == 'SLIM' else T.conv2d(x, w, stride, padding)


def pack_exponent(w):
    """e[c] of the tensor-core weight packing (DESIGN section 2), and max|w[:, c]|."""
    mx = np.abs(w.reshape(-1, w.shape[-1]).astype(f64)).max(0)
    e = np.zeros(mx.shape, np.int64)
    ok = (mx > 0) & np.isfinite(mx)
    e[ok] = np.clip(14 - np.frexp(mx[ok])[1], -126, 126)
    return e, mx


def out_geometry(h, w, k, stride, rate, padding, kw=None):
    """(ho, wo, pad_top, pad_left) of the layer, as lumi_op_conv2d and the engine's run_conv derive them: a k x k
    kernel, or k x kw (SLIM pads both sides by the kernel's height, as conv2d_same's square kernels need)."""
    keff = k + (k - 1) * (rate - 1)
    kweff = keff if kw is None else kw + (kw - 1) * (rate - 1)
    if padding == 'SAME' or (padding == 'SLIM' and stride == 1):
        ho, wo = -(-h // stride), -(-w // stride)
        return ho, wo, max(0, (ho - 1) * stride + keff - h) // 2, max(0, (wo - 1) * stride + kweff - w) // 2
    if padding == 'SLIM':
        p = (keff - 1) // 2
        return (h - 1) // stride + 1, (w - 1) // stride + 1, p, p
    return (h - keff) // stride + 1, (w - kweff) // stride + 1, 0, 0


def _sampled_sums(x, w, stride, padding, rate, at):
    """float64 sum x w, sum |x||w|, sum |w| and sum |x| over the taps inside the map, at output pixels
    at = (img, oy, ox): [P, C_out] each ([P, 1] for sum |x|).  Only the sampled input patches are gathered."""
    n, h, wd, cin = x.shape
    kh, kw, _, cout = w.shape
    _, _, pt, pl = out_geometry(h, wd, kh, stride, rate, padding, kw=kw)
    img, oy, ox = (np.asarray(a, np.int64) for a in at)
    w64 = w.astype(f64).reshape(kh * kw, cin, cout)
    aw = np.abs(w64)
    acc = np.zeros((len(img), cout))
    sxw = np.zeros((len(img), cout))
    sw = np.zeros((len(img), cout))
    sx = np.zeros((len(img), 1))
    for t in range(kh * kw):
        iy = oy * stride - pt + (t // kw) * rate
        ix = ox * stride - pl + (t % kw) * rate
        inside = (iy >= 0) & (iy < h) & (ix >= 0) & (ix < wd)
        xt = x[img, iy.clip(0, h - 1), ix.clip(0, wd - 1)].astype(f64) * inside[:, None]
        acc += xt @ w64[t]
        axt = np.abs(xt)
        sxw += axt @ aw[t]
        sw += inside[:, None] * aw[t].sum(0)
        sx += axt.sum(1, keepdims=True)
    return acc, sxw, sw, sx


def reference(x, w, stride, padding, scale, bias, residual, res_stride, act, impl, rate=1, at=None, k_fold=None):
    """float64 reference of the layer and the per-element bound of the module docstring: at every output element
    ([n, ho, wo, C_out]) or, with at = (img, oy, ox) index arrays, at those output pixels only ([P, C_out]).
    k_fold: the K whose 64-deep slices the tensor-core kernel folds, when a packed layout runs more than kh kw C_in."""
    cout = w.shape[-1]
    s = np.ones(cout, f64) if scale is None else scale.astype(f64)
    b = np.zeros(cout, f64) if bias is None else bias.astype(f64)
    if at is None:
        assert rate == 1
        acc = _conv64(x, w, stride, padding)
        ax, aw = np.abs(x.astype(f64)), np.abs(w.astype(f64))
        sxw, sw = _conv64(ax, aw, stride, padding), _conv64(np.ones_like(ax), aw, stride, padding)
        sx = _conv64(ax, np.ones(w.shape[:3] + (1,)), stride, padding)
    else:
        acc, sxw, sw, sx = _sampled_sums(x, w, stride, padding, rate, at)
    r = None
    if residual is not None:
        if at is None:
            r = residual.astype(f64)[:, ::res_stride, ::res_stride][:, :acc.shape[1], :acc.shape[2]]
        else:
            r = residual[at[0], np.asarray(at[1]) * res_stride, np.asarray(at[2]) * res_stride].astype(f64)
        assert r.shape == acc.shape
    ref = acc * s + b + (r if r is not None else 0.0)
    if act == 1:
        ref = np.maximum(ref, 0.0)
    elif act == 2:
        ref = np.clip(ref, 0.0, 6.0)
    S = np.abs(s) * sxw + np.abs(b) + (np.abs(r) if r is not None else 0.0)
    W = np.abs(s) * sw
    K = w.shape[0] * w.shape[1] * w.shape[2] if k_fold is None else k_fold
    if impl in (0, 13):
        alpha = 1.01 * (2.0 ** -22 * 2 + U * (K + 3))
        V = 0.0
    else:
        alpha = 1.01 * (2.0 ** -22 * 12 + U * (math.ceil(K / 64) + 3))
        e, mx = pack_exponent(w)
        fw = 2.0 ** -25 * np.abs(s) * 2.0 ** -e.astype(f64) + 2.0 ** -150 * 2.0 ** e.astype(f64) * mx
        V = fw * sx
    delta = 2.0 ** -25 * (2 if r is not None else 1)
    return ref, alpha * S + 1.01 * 2.0 ** -25 * W + V + delta


def preact_reference(ref, bound, ps, pb):
    ps, pb = ps.astype(f64), pb.astype(f64)
    p = np.maximum(ref * ps + pb, 0.0)
    pbound = np.abs(ps) * bound + 1.01 * (U + 2.0 ** -22) * (np.abs(ps) * (np.abs(ref) + bound) + np.abs(pb)) + 2.0 ** -25
    return p, pbound


def check(name, got, ref, bound):
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    err = np.abs(got.astype(f64) - ref)
    ok = err <= bound                                   # NaN fails
    ratio = float(np.max(np.where(np.isfinite(err), err / bound, np.inf)))
    print('%-60s max err/bound %.3f' % (name, ratio))
    if not ok.all():
        i = np.unravel_index(np.argmin(np.where(ok, np.inf, -err / bound)), err.shape)
        raise AssertionError('%s: %d elements over the bound; worst at %s: got %r, ref %r, bound %.3e'
                             % (name, int((~ok).sum()), i, float(got[i]), float(ref[i]), float(bound[i])))
    return ratio


def run_case(name, x, w, impl, stride=1, padding='SAME', scale=None, bias=None, residual=None, res_stride=1, act=0):
    rc, y, _ = conv_io(x, w, stride, padding, scale, bias, residual, res_stride, act, impl)
    assert rc == 0, '%s: LUMI_EOVERFLOW' % name
    ref, bound = reference(x, w, stride, padding, scale, bias, residual, res_stride, act, impl)
    check('%s/impl%d' % (name, impl), y, ref, bound)
    return y, ref


def he(rng, k, cin, cout, gain=1.0):
    return (rng.standard_normal((k, k, cin, cout)) * gain * np.sqrt(2.0 / (k * k * cin))).astype(f32)


def signed_uniform(rng, lo, hi, n):
    return (rng.uniform(lo, hi, n) * rng.choice([-1.0, 1.0], n)).astype(f32)


# ---------------------------------------------------------------------------------------------- weight columns
@pytest.mark.parametrize('act', [0, 1])
@pytest.mark.parametrize('impl', IMPLS)
def test_weight_column_magnitudes(impl, act):
    """Column maxima from 2^-40 to 2^40 (BN scale 2^-k keeps the outputs O(1), so e[c] spans 80 binades), an all-zero
    column, a column at 2^-120 (below the exponent clamp) and a column with a single nonzero weight.  The zero and
    tiny columns are bias only: they must equal act(bias) exactly (relu would turn a NaN into 0, not into b)."""
    rng = np.random.default_rng(100 + act)
    n, h, wd, cin, cout = 2, 9, 13, 64, 96
    x = rng.standard_normal((n, h, wd, cin)).astype(f32)
    ks = np.round(np.linspace(-40, 40, cout - 3)).astype(int)
    w = he(rng, 3, cin, cout)
    w[..., :cout - 3] *= (2.0 ** ks).astype(f32)
    w[..., cout - 3] = 0.0
    w[..., cout - 2] = (rng.uniform(-1, 1, (3, 3, cin)) * 2.0 ** -120).astype(f32)
    w[..., cout - 1] = 0.0
    w[1, 1, 5, cout - 1] = 0.37
    scale = np.ones(cout, f32)
    scale[:cout - 3] = (2.0 ** -ks).astype(f32) * rng.uniform(0.5, 1.5, cout - 3).astype(f32)
    bias = signed_uniform(rng, 0.01, 1.0, cout)
    bias[cout - 3:cout - 1] = [0.25, 0.5]
    y, _ = run_case('weight_columns/act%d' % act, x, w, impl, scale=scale, bias=bias, act=act)
    for c in (cout - 3, cout - 2):
        want = bias[c] if act == 0 else max(bias[c], f32(0))
        np.testing.assert_array_equal(y[..., c], np.full(y.shape[:3], want, f32), err_msg='column %d' % c)


# ---------------------------------------------------------------------------------------------- channel scale
@pytest.mark.parametrize('impl', IMPLS)
def test_channel_scale_range(impl):
    """BN scales from 1e-4 to 1e4 (both signs), and every eighth channel dominated by a large bias."""
    rng = np.random.default_rng(200)
    n, h, wd, cin, cout = 2, 11, 14, 128, 128
    x = rng.standard_normal((n, h, wd, cin)).astype(f32)
    w = he(rng, 3, cin, cout, 0.35)
    scale = (10.0 ** np.linspace(-4, 4, cout)).astype(f32) * rng.choice([-1, 1], cout).astype(f32)
    rng.shuffle(scale)
    bias = (rng.standard_normal(cout) * 0.1).astype(f32)
    bias[::8] = signed_uniform(rng, 1e2, 1e3, cout // 8)
    scale[::8] = np.abs(scale[::8]).clip(max=1.0) * 1e-3
    run_case('channel_scale', x, w, impl, scale=scale, bias=bias, act=0)


# ---------------------------------------------------------------------------------------------- activation magnitude
@pytest.mark.parametrize('kind', ['small_1e-3', 'mixed_1e-4_1e2'])
@pytest.mark.parametrize('impl', IMPLS)
def test_activation_magnitude(impl, kind):
    """Input maps at 1e-3 scale, where the split's 2^-25 floor (subnormal lo) decides the error, and maps whose
    channels alternate between 1e-4 and 1e2 scale."""
    rng = np.random.default_rng(300)
    n, h, wd, cin, cout = 2, 10, 15, 64, 64
    x = rng.standard_normal((n, h, wd, cin))
    if kind == 'small_1e-3':
        x = x * 1e-3
        bias = (rng.standard_normal(cout) * 1e-4).astype(f32)
    else:
        x = x * np.where(np.arange(cin) % 2 == 0, 1e-4, 1e2)
        bias = (rng.standard_normal(cout) * 0.1).astype(f32)
    x = x.astype(f32)
    w = he(rng, 3, cin, cout)
    scale = rng.uniform(0.5, 1.5, cout).astype(f32)
    run_case('activation/%s' % kind, x, w, impl, scale=scale, bias=bias, act=0)


# ---------------------------------------------------------------------------------------------- shapes
# name, n, h, w, cin, cout, k, residual: short K (1x1, 64 channels: the four-consumer kernel), long K (3x3, 1024
# channels), C_out 64 (BN = 64), 96 and 160 (channel boxes TMA clips), 256, and a multi-image tile (5x6 maps: four
# images per tile, the last tile ragged)
SHAPES = [
    ('short_k_1x1_64_256', 2, 13, 21, 64, 256, 1, True),
    ('long_k_3x3_1024_64', 2, 14, 18, 1024, 64, 3, False),
    ('cout64_3x3', 2, 11, 17, 128, 64, 3, True),
    ('cout96_1x1', 3, 9, 14, 64, 96, 1, True),
    ('cout160_3x3', 2, 9, 11, 128, 160, 3, False),
    ('cout256_3x3', 1, 12, 20, 128, 256, 3, True),
    ('multi_image_5x6', 7, 5, 6, 64, 128, 3, True),
]


@pytest.mark.parametrize('shape', SHAPES, ids=[s[0] for s in SHAPES])
@pytest.mark.parametrize('impl', IMPLS)
def test_shapes(impl, shape):
    name, n, h, wd, cin, cout, k, with_res = shape
    rng = np.random.default_rng(400 + SHAPES.index(shape))
    x = (rng.standard_normal((n, h, wd, cin)) * 2).astype(f32)
    w = he(rng, k, cin, cout)
    scale = rng.uniform(0.5, 1.5, cout).astype(f32)
    bias = (rng.standard_normal(cout) * 0.1).astype(f32)
    res = rng.standard_normal((n, h, wd, cout)).astype(f32) if with_res else None
    run_case(name, x, w, impl, scale=scale, bias=bias, residual=res, act=1)


# ---------------------------------------------------------------------------------------------- overflow threshold
def pick_tile(n, ho, wo):
    """The conv kernel's M-tile choice (conv.cu pick_tile): (nb, th, tw)."""
    best, nb, th, tw = -1.0, 1, 1, 1
    for w_ in range(1, min(128, wo) + 1):
        for h_ in range(1, min(128 // w_, ho) + 1):
            b_ = max(1, min(n, 128 // (h_ * w_))) if (h_ == ho and w_ == wo) else 1
            tiles = -(-n // b_) * -(-ho // h_) * -(-wo // w_)
            eff = n * ho * wo / (tiles * 128.0)
            if eff > best + 1e-9 or (eff > best - 1e-9 and w_ > tw):
                best, nb, th, tw = eff, b_, h_, w_
    return nb, th, tw


F16_MAX = f32(65504.0)
THRESHOLDS = [F16_MAX, np.nextafter(F16_MAX, f32(np.inf)), f32(65519.996), f32(65520.0)]
OVF_N, OVF_H, OVF_W, OVF_CIN, OVF_COUT = 3, 11, 19, 64, 96


def _last_pixel_is_in_a_ragged_tile():
    nb, th, tw = pick_tile(OVF_N, OVF_H, OVF_W)
    return OVF_N % nb != 0 or OVF_H % th != 0 or OVF_W % tw != 0


@pytest.mark.parametrize('sign', [1, -1])
@pytest.mark.parametrize('target', THRESHOLDS, ids=['65504', 'next_after_65504', '65519.996', '65520'])
@pytest.mark.parametrize('impl', SPLIT_IMPLS)
def test_overflow_threshold(impl, target, sign):
    """Zero weights, a bias and a residual that put one element -- the last valid pixel (in a ragged last tile), last
    real channel -- exactly at +-target: every split output raises LUMI_EOVERFLOW iff |v| > 65504, whatever its hi
    plane rounds to (65504.004 and 65519.996 round to a finite 65504)."""
    assert _last_pixel_is_in_a_ragged_tile()
    n, h, wd, cin, cout = OVF_N, OVF_H, OVF_W, OVF_CIN, OVF_COUT
    x = np.random.default_rng(500).standard_normal((n, h, wd, cin)).astype(f32)
    w = np.zeros((1, 1, cin, cout), f32)
    bias = np.zeros(cout, f32)
    bias[-1] = sign * (target - f32(32768.0))                          # exact in fp32, and v = b + 32768 exactly
    assert bias[-1] + f32(sign * 32768.0) == f32(sign) * target
    res = np.zeros((n, h, wd, cout), f32)
    res[-1, -1, -1, -1] = sign * 32768.0
    rc, y, _ = conv_io(x, w, bias=bias, residual=res, impl=impl)
    if target > F16_MAX:
        assert rc == LUMI_EOVERFLOW, 'impl %d: %r did not raise' % (impl, float(sign * target))
    else:
        assert rc == 0, 'impl %d: %r raised' % (impl, float(sign * target))
        assert y[-1, -1, -1, -1] == sign * F16_MAX
        np.testing.assert_array_equal(y[:-1, ..., -1], np.full(y[:-1, ..., -1].shape, bias[-1]))


@pytest.mark.parametrize('want_x', [True, False], ids=['x_and_p', 'p_only'])
@pytest.mark.parametrize('target', THRESHOLDS, ids=['65504', 'next_after_65504', '65519.996', '65520'])
@pytest.mark.parametrize('impl', PREACT_IMPLS)
def test_preact_overflow_threshold(impl, target, want_x):
    """The same threshold on the pre-activation output p = relu(fmaf(x^, ps, pb)): x = -1 or +1 at the chosen element
    (x^ exact), ps = -target or +target on its channel, so p is exactly target there and 0 everywhere else."""
    n, h, wd, cin, cout = OVF_N, OVF_H, OVF_W, OVF_CIN, OVF_COUT
    x = np.random.default_rng(501).standard_normal((n, h, wd, cin)).astype(f32)
    w = np.zeros((1, 1, cin, cout), f32)
    for sign in (1, -1):
        res = np.zeros((n, h, wd, cout), f32)
        res[-1, -1, -1, -1] = sign
        ps = np.zeros(cout, f32)
        ps[-1] = sign * target
        rc, y, p = conv_io(x, w, residual=res, impl=impl, pre=(ps, np.zeros(cout, f32)), want_x=want_x)
        if target > F16_MAX:
            assert rc == LUMI_EOVERFLOW, 'impl %d: p = %r did not raise' % (impl, float(target))
        else:
            assert rc == 0, 'impl %d: p = %r raised' % (impl, float(target))
            assert p[-1, -1, -1, -1] == F16_MAX and np.count_nonzero(p) == 1
            if want_x:
                np.testing.assert_array_equal(y, res)


# ---------------------------------------------------------------------------------------------- subsampled residual
# name, layer, residual resolution (h, w), cout: the residual has the resolution of the layer's input map for the
# stride-2 3x3 layer, and of the unit's input (twice the layer's) for the conv3-like 1x1 layer; the layer reads
# residual[:, ::2, ::2] (slim's `subsample`)
SUBSAMPLE = [
    ('1x1_odd_256', '1x1', (13, 21), 256),
    ('1x1_even_64', '1x1', (14, 20), 64),
    ('3x3s2_odd_64', '3x3s2', (13, 19), 64),
    ('3x3s2_even_256', '3x3s2', (12, 22), 256),
]
SUB_MODES = [(i, 'plain') for i in IMPLS] + [(i, m) for i in PREACT_IMPLS for m in ('x_and_p', 'p_only')]


@pytest.mark.parametrize('impl,mode', SUB_MODES, ids=['%d-%s' % m for m in SUB_MODES])
@pytest.mark.parametrize('case', SUBSAMPLE, ids=[c[0] for c in SUBSAMPLE])
def test_subsampled_residual(case, impl, mode):
    name, layer, (rh, rw), cout = case
    rng = np.random.default_rng(600 + SUBSAMPLE.index(case))
    n, cin = 3, 64
    if layer == '1x1':
        h, wd, k, stride, padding = -(-rh // 2), -(-rw // 2), 1, 1, 'SAME'
    else:
        h, wd, k, stride, padding = rh, rw, 3, 2, 'SLIM'
    x = (rng.standard_normal((n, h, wd, cin)) * 2).astype(f32)
    w = he(rng, k, cin, cout)
    scale = rng.uniform(0.5, 1.5, cout).astype(f32)
    bias = (rng.standard_normal(cout) * 0.1).astype(f32)
    res = rng.standard_normal((n, rh, rw, cout)).astype(f32)
    ref, bound = reference(x, w, stride, padding, scale, bias, res, 2, 0, impl)
    assert ref.shape[1:3] == (-(-rh // 2), -(-rw // 2))
    tag = 'subsample/%s/impl%d/%s' % (name, impl, mode)
    if mode == 'plain':
        rc, y, _ = conv_io(x, w, stride, padding, scale, bias, res, 2, 0, impl)
        assert rc == 0
        check(tag, y, ref, bound)
        return
    ps = rng.uniform(-1.5, 1.5, cout).astype(f32)
    pb = (rng.standard_normal(cout) * 0.2).astype(f32)
    rc, y, p = conv_io(x, w, stride, padding, scale, bias, res, 2, 0, impl, pre=(ps, pb), want_x=mode == 'x_and_p')
    assert rc == 0
    if y is not None:
        check(tag + '/x', y, ref, bound)
    pref, pbound = preact_reference(ref, bound, ps, pb)
    check(tag + '/p', p, pref, pbound)
