"""The conv kernel's shared-memory slot epilogue (residual prefetched by TMA into a slot, split output planes written
over it and bulk-stored by TMA) against the register epilogue it replaces: the same arithmetic, so bit-identical
outputs on every split-output conv case, plus a case whose channel count TMA clips (C_out = 96)."""
import os
import shutil
import subprocess
import zlib

import numpy as np
import pytest

from test_gpu_kernels import CONV_CASES, _bn_fold, _ref_conv, assert_close

# lumi_op_conv2d impl codes: split planes through the slot epilogue (two consumer warpgroups / four allowed up to the
# engine's 16 K slices / four + stream-K), and the generic kernel with the register epilogue forced; all run the
# engine's single-buffered mainloop
SLOT, SLOT_EPI16, SLOT_EPI16_STREAMK, REGISTER = 3, 4, 5, 12

# name, n, h, w, cin, cout, k, stride, rate, padding, residual, act: the second 64-channel box of the tile is half
# outside the tensor, on the residual load and on the stores
CLIPPED_CASE = ('cout96_res', 2, 19, 40, 128, 96, 1, 1, 1, 'SAME', True, 1)
SPLIT_CASES = [c for c in CONV_CASES if c[4] % 64 == 0 and c[5] % 32 == 0] + [CLIPPED_CASE]


def _conv(x, w, stride, rate, padding, scale, bias, residual, act, impl):
    import ctypes
    import torch
    import gpu_ops as G
    lib = G._lib()
    n, h, wd, cin = x.shape
    kh, kw, _, cout = w.shape
    pad = {'VALID': 0, 'SAME': 1, 'SLIM': 2}[padding]
    xd, wdv, sd, bd = G._dev(x, np.float32), G._dev(w, np.float32), G._dev(scale, np.float32), G._dev(bias, np.float32)
    rd = G._dev(residual, np.float32) if residual is not None else None
    ho, wo = ctypes.c_int(), ctypes.c_int()
    G._check(lib.lumi_op_conv2d(G._p(xd), n, h, wd, cin, G._p(wdv), kh, kw, cout, stride, rate, pad, G._p(sd),
                                G._p(bd), G._p(rd), act, impl, None, ctypes.byref(ho), ctypes.byref(wo), None))
    y = torch.empty((n, ho.value, wo.value, cout), dtype=torch.float32, device='cuda')
    G._check(lib.lumi_op_conv2d(G._p(xd), n, h, wd, cin, G._p(wdv), kh, kw, cout, stride, rate, pad, G._p(sd),
                                G._p(bd), G._p(rd), act, impl, G._p(y), ctypes.byref(ho), ctypes.byref(wo), None))
    torch.cuda.synchronize()
    return y.cpu().numpy()


def _inputs(case):
    name, n, h, w, cin, cout, k, stride, rate, padding, use_res, act = case
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = (rng.standard_normal((n, h, w, cin)) * 2).astype(np.float32)
    wt = (rng.standard_normal((k, k, cin, cout)) * np.sqrt(2.0 / (k * k * cin))).astype(np.float32)
    scale, bias = _bn_fold(rng, cout)
    ref0 = _ref_conv(x, wt, stride, rate, padding, scale, bias, None, 0)
    res = rng.standard_normal(ref0.shape).astype(np.float32) if use_res else None
    return x, wt, stride, rate, padding, scale, bias, res, act


@pytest.mark.gpu
@pytest.mark.parametrize('case', SPLIT_CASES, ids=[c[0] for c in SPLIT_CASES])
def test_slot_epilogue_is_bit_identical_to_register_epilogue(case):
    args = _inputs(case)
    slot = _conv(*args, SLOT)
    reg = _conv(*args, REGISTER)
    assert slot.tobytes() == reg.tobytes(), '%s: max abs diff %.3e' % (case[0], float(np.abs(slot - reg).max()))


@pytest.mark.gpu
@pytest.mark.parametrize('impl', [SLOT, SLOT_EPI16, SLOT_EPI16_STREAMK, REGISTER])
def test_clipped_channel_box_matches_oracle(impl):
    x, wt, stride, rate, padding, scale, bias, res, act = _inputs(CLIPPED_CASE)
    ref = _ref_conv(x, wt, stride, rate, padding, scale, bias, res, act)
    assert_close(_conv(x, wt, stride, rate, padding, scale, bias, res, act, impl), ref, 2e-5, 'cout96/%d' % impl)


def test_conv_kernel_has_tma_stores_sass():
    """The slot epilogue is built: the conv kernels carry 4-D TMA tensor stores."""
    from luminoth_b200 import build as B
    exe = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if not os.path.exists(exe) or not os.path.exists(B.LIB):
        pytest.skip('cuobjdump or the built library is not available')
    sass = subprocess.run([exe, '-sass', B.LIB], capture_output=True, text=True).stdout
    conv = [f for f in sass.split('Function : ')[1:] if f.startswith('_ZN4lumi14conv_tc_kernel')]
    assert conv, 'no conv_tc_kernel in the library'
    assert any('UTMASTG.4D' in f for f in conv), 'no TMA tensor store in the conv kernels'
