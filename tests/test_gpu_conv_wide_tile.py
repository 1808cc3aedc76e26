"""The conv kernel's 128 x 256 tile (`lumi_op_conv2d` impl 14: whole tiles, 15: stream-K forced) for split-output
layers with C_out padded to a multiple of 256.  Each slice runs as two 128-column halves with the BN = 128 kernel's
MMA chain and fold order, so on whole tiles the outputs are byte-identical to the BN = 128 slot-epilogue kernel
(impl 3).  Stream-K adds the partial sums of a tile in another order and is held to the per-element bound of
test_gpu_conv_numerics."""
import os
import shutil
import subprocess
import zlib

import numpy as np
import pytest

from test_gpu_conv_epilogue import SLOT, _conv, _inputs
from test_gpu_conv_numerics import check, conv_io, he, reference
from test_gpu_kernels import CONV_CASES

WIDE, WIDE_STREAMK = 14, 15

# name, n, h, w, cin, cout, k, stride, rate, padding, residual, act
WIDE_CASES = [c for c in CONV_CASES if c[4] % 64 == 0 and c[5] % 256 == 0] + [
    ('ragged_3x3_256_res', 3, 23, 61, 128, 256, 3, 1, 1, 'SAME', True, 1),      # ragged tile rows, columns, images
    ('3x3s2_256_res', 2, 37, 63, 128, 256, 3, 2, 1, 'SAME', True, 1),
    ('relu6_512', 1, 12, 16, 128, 512, 3, 1, 1, 'SAME', False, 2),
    # C_out = 256 + 3 x 64, padded to 512: the last 64-column group lies outside the tensor (TMA clips the stores)
    ('cout448_res', 2, 19, 40, 128, 448, 1, 1, 1, 'SAME', True, 1),
    ('cout448_3x3', 1, 13, 21, 192, 448, 3, 1, 1, 'SAME', False, 1),
    ('rpn_like_1024_512', 1, 19, 32, 1024, 512, 3, 1, 1, 'SAME', False, 1),   # 144 K slices
]


@pytest.mark.gpu
@pytest.mark.parametrize('case', WIDE_CASES, ids=[c[0] for c in WIDE_CASES])
def test_wide_tile_is_byte_identical_to_bn128(case):
    args = _inputs(case)
    wide = _conv(*args, WIDE)
    ref = _conv(*args, SLOT)
    assert wide.tobytes() == ref.tobytes(), '%s: max abs diff %.3e' % (case[0], float(np.abs(wide - ref).max()))


# name, layer, residual (h, w), cout: the layer reads residual[:, ::2, ::2] (slim's `subsample`)
SUBSAMPLED = [('1x1_odd_256', '1x1', (13, 21), 256), ('3x3s2_even_512', '3x3s2', (12, 22), 512)]


def _subsampled_inputs(case):
    name, layer, (rh, rw), cout = case
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    n, cin = 3, 128
    if layer == '1x1':
        h, wd, k, stride, padding = -(-rh // 2), -(-rw // 2), 1, 1, 'SAME'
    else:
        h, wd, k, stride, padding = rh, rw, 3, 2, 'SLIM'
    x = (rng.standard_normal((n, h, wd, cin)) * 2).astype(np.float32)
    w = he(rng, k, cin, cout)
    scale = rng.uniform(0.5, 1.5, cout).astype(np.float32)
    bias = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    res = rng.standard_normal((n, rh, rw, cout)).astype(np.float32)
    return x, w, stride, padding, scale, bias, res


@pytest.mark.gpu
@pytest.mark.parametrize('case', SUBSAMPLED, ids=[c[0] for c in SUBSAMPLED])
def test_wide_tile_subsampled_residual_is_byte_identical(case):
    x, w, stride, padding, scale, bias, res = _subsampled_inputs(case)
    rc_w, wide, _ = conv_io(x, w, stride, padding, scale, bias, res, 2, 1, WIDE)
    rc_n, ref, _ = conv_io(x, w, stride, padding, scale, bias, res, 2, 1, SLOT)
    assert rc_w == 0 and rc_n == 0
    assert wide.tobytes() == ref.tobytes(), '%s: max abs diff %.3e' % (case[0], float(np.abs(wide - ref).max()))


# name, n, h, w, cin, cout, k, residual: enough K slices per CTA that every stream-K range splits tiles
STREAMK_CASES = [
    ('3x3_256_res', 2, 38, 64, 256, 256, 3, True),
    ('1x1_1024_256', 2, 38, 64, 1024, 256, 1, False),
    ('3x3_1024_512', 1, 19, 32, 1024, 512, 3, False),
    ('cout448_3x3_res', 2, 19, 40, 128, 448, 3, True),
]


@pytest.mark.gpu
@pytest.mark.parametrize('case', STREAMK_CASES, ids=[c[0] for c in STREAMK_CASES])
def test_wide_tile_streamk_within_bound(case):
    name, n, h, wd, cin, cout, k, with_res = case
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = (rng.standard_normal((n, h, wd, cin)) * 2).astype(np.float32)
    w = he(rng, k, cin, cout)
    scale = rng.uniform(0.5, 1.5, cout).astype(np.float32)
    bias = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    res = rng.standard_normal((n, h, wd, cout)).astype(np.float32) if with_res else None
    rc, y, _ = conv_io(x, w, 1, 'SAME', scale, bias, res, 1, 1, WIDE_STREAMK)
    assert rc == 0
    ref, bound = reference(x, w, 1, 'SAME', scale, bias, res, 1, 1, WIDE_STREAMK)
    check('wide_streamk/%s' % name, y, ref, bound)


@pytest.mark.gpu
def test_wide_tile_rejects_narrow_cout():
    x, wt, stride, rate, padding, scale, bias, res, act = _inputs(('cout128', 1, 8, 8, 64, 128, 1, 1, 1, 'SAME',
                                                                   False, 1))
    with pytest.raises(RuntimeError, match='multiple of 256'):
        _conv(x, wt, stride, rate, padding, scale, bias, res, act, WIDE)


def test_wide_tile_kernel_has_no_local_memory_sass():
    """The 128 x 256 instance is built, and its register budget holds: no local-memory loads or stores anywhere."""
    from luminoth_b200 import build as B
    exe = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(exe) or not os.path.exists(B.LIB):
        pytest.skip('cuobjdump or the built library is not available')
    sass = subprocess.run([exe, '-sass', B.LIB], capture_output=True, text=True).stdout
    wide = [f for f in sass.split('Function : ')[1:] if f.startswith('_ZN4lumi14conv_tc_kernelILi256E')]
    assert len(wide) == 1, 'expected one 128 x 256 conv_tc_kernel instance, found %d' % len(wide)
    assert 'HGMMA' in wide[0]
    assert not any(op in wide[0] for op in ('STL', 'LDL')), 'local-memory traffic in the 128 x 256 kernel'
