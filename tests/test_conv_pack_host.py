"""The tensor-core weight packing of a conv layer (`lumi_pack_conv_weights`, host only, no GPU).

Per output channel c the packing stores the fp16 split (hi, lo) of w[:, c] * 2^e[c] and scale_tc[c] = s[c] * 2^-e[c],
with e[c] = 14 - ex, max|w[:, c]| = f * 2^ex (f in [0.5, 1)), clamped to [-126, 126] so that 2^e and 2^-e are normal
fp32.  What the conv kernel multiplies is (hi + lo) * scale_tc, and that must reconstruct w * s:

* hi + lo keeps 23 bits of v = w * 2^e (|v - hi - lo| <= 2^-23 |v| while lo is a normal fp16; a subnormal lo costs at
  most 2^-25 absolute, 2^-38 * max|w[:, c]| once scaled back for an unclamped column, and nothing for a clamped one,
  whose v are multiples of 2^-23);
* scale_tc is s * 2^-e rounded once (2^-24 relative).
Together: |(hi + lo) * scale_tc - w * s| <= 2^-22 * max|w[:, c]| * |s| for every element.  The one floor: where
|s| * 2^-e < 2^-126, scale_tc is a subnormal fp32 (absolute error 2^-150), which adds 2^-150 * |hi + lo| < 2^-136.
"""
import ctypes

import numpy as np
import pytest

from luminoth_b200 import engine

f16, f32 = np.float16, np.float32
EXP_MAX = 126


def pack(w, scale=None):
    """w: [kdim, cout] fp32 -> hi, lo [cout, kdim] fp16, scale_tc [cout] fp32."""
    lib = engine.load_library()
    w = np.ascontiguousarray(w, f32)
    kdim, cout = w.shape
    hi = np.zeros((cout, kdim), f16)
    lo = np.zeros((cout, kdim), f16)
    sct = np.zeros(cout, f32)
    s = None if scale is None else np.ascontiguousarray(scale, f32)
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p) if a is not None else None
    rc = lib.lumi_pack_conv_weights(vp(w), kdim, cout, vp(s), vp(hi), vp(lo), vp(sct))
    assert rc == 0, lib.lumi_op_last_error().decode()
    return hi, lo, sct


def exponent(mx):
    """e[c] as documented: 0 for an all-zero column."""
    if not (mx > 0 and np.isfinite(mx)):
        return 0
    return int(np.clip(14 - np.frexp(np.float64(mx))[1], -EXP_MAX, EXP_MAX))


def columns():
    """[kdim, cout] weights: column maxima 2^k over all of fp32 (subnormals included), then the edge columns."""
    rng = np.random.default_rng(0)
    kdim = 96
    cols, names = [], []
    for k in range(-149, 128):
        c = rng.uniform(-1, 1, kdim) * 2.0 ** k
        c[rng.integers(kdim)] = 2.0 ** k * rng.choice([-1, 1])
        cols.append(c)
        names.append('max 2^%d' % k)
    for k in (-140, -126, -114, -113, -112, -60, 0, 60, 126):         # maxima that are not powers of two
        c = rng.uniform(-1, 1, kdim) * 2.0 ** k
        c[5] = 1.9999 * 2.0 ** k
        cols.append(c)
        names.append('max 1.9999 * 2^%d' % k)
    cols.append(np.zeros(kdim))
    names.append('all zero')
    c = np.zeros(kdim)
    c[17] = -0.37
    cols.append(c)
    names.append('single nonzero')
    for k in (-120, -100, 0, 40, 100):                                 # one weight 2^-30 of the column max
        c = rng.uniform(-1, 1, kdim) * 2.0 ** k
        c[3] = 2.0 ** k
        c[4] = 2.0 ** (k - 30)
        cols.append(c)
        names.append('2^-30 weight, max 2^%d' % k)
    w = np.stack(cols, 1).astype(f32)
    return w, names


def scales(cout, rng):
    s = (10.0 ** rng.uniform(-4, 4, cout)) * rng.choice([-1, 1], cout)
    s[::7] = 1.0
    return s.astype(f32)


@pytest.mark.parametrize('with_scale', [False, True])
def test_pack_reconstructs_every_column(with_scale):
    w, names = columns()
    s = scales(w.shape[1], np.random.default_rng(1)) if with_scale else np.ones(w.shape[1], f32)
    hi, lo, sct = pack(w, s if with_scale else None)
    assert np.isfinite(hi).all() and np.isfinite(lo).all() and np.isfinite(sct).all()
    hi64, lo64 = hi.astype(np.float64), lo.astype(np.float64)
    recon = (hi64 + lo64) * sct.astype(np.float64)[:, None]                   # [cout, kdim]
    exact = w.T.astype(np.float64) * s.astype(np.float64)[:, None]
    bad = []
    for c, name in enumerate(names):
        mx = float(np.abs(w[:, c]).max())
        e = exponent(mx)
        # the documented formula, bit for bit (numpy's fp16 conversion rounds to nearest even, subnormals included)
        v = (w[:, c] * f32(2.0 ** e)).astype(f32)
        np.testing.assert_array_equal(hi[c], v.astype(f16), err_msg=name)
        np.testing.assert_array_equal(lo[c], (v - hi[c].astype(f32)).astype(f16), err_msg=name)
        assert sct[c] == f32(np.float64(s[c]) * 2.0 ** -e), name
        tol = 2.0 ** -22 * mx * abs(float(s[c]))
        if abs(float(sct[c])) < 2.0 ** -126:                                  # subnormal scale_tc
            tol += 2.0 ** -150 * float(np.abs(hi64[c] + lo64[c]).max())
        err = float(np.abs(recon[c] - exact[c]).max())
        if not err <= tol:
            bad.append('%s: err %.3e > %.3e' % (name, err, tol))
        if mx == 0:
            assert not hi[c].any() and not lo[c].any() and e == 0, name      # exact zeros
            continue
        packed = np.abs(hi64[c] + lo64[c]).max()
        if 14 - np.frexp(np.float64(mx))[1] <= EXP_MAX:                       # unclamped: the max lands in [2^13, 2^14)
            assert 2.0 ** 13 <= packed < 2.0 ** 14, (name, packed)
            assert 2.0 ** 13 <= np.abs(hi64[c]).max() <= 2.0 ** 14, name    # hi itself may round up to 2^14
        else:                                                                 # clamped: e = 126, below 2^13
            assert e == EXP_MAX and packed < 2.0 ** 13, (name, packed)
    assert not bad, '\n'.join(bad)


def test_pack_clamps_tiny_columns():
    """A column below 2^-113 would need e >= 127: 2^e overflows to inf there (inf weights, NaN for the zeros) and
    2^-e is subnormal.  The clamp keeps every output finite and the column's own scale exact."""
    kdim = 64
    w = np.zeros((kdim, 4), f32)
    w[3, 0] = 4e-35                  # e would be 128
    w[:, 1] = np.linspace(-1, 1, kdim) * 2.0 ** -120
    w[7, 2] = 2.0 ** -149            # the smallest subnormal
    w[:, 3] = np.linspace(-1, 1, kdim) * 2.0 ** -113
    s = np.array([1.0, 3.0, 0.5, 1e-4], f32)
    hi, lo, sct = pack(w, s)
    assert np.isfinite(hi).all() and np.isfinite(lo).all()
    np.testing.assert_array_equal(sct, (s.astype(np.float64) * 2.0 ** -126).astype(f32))
    recon = (hi.astype(np.float64) + lo.astype(np.float64)) * sct.astype(np.float64)[:, None]
    exact = w.T.astype(np.float64) * s.astype(np.float64)[:, None]
    assert (np.abs(recon - exact) <= 2.0 ** -136).all()
    assert (recon[w.T == 0] == 0).all()                                     # zero weights stay zero, never NaN
