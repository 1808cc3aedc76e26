"""Every distinct conv launch of the production workloads, at production size, through the kernels the engine runs.

LAYERS holds one row per distinct conv launch of
* resnet_v1_50 to the block3 endpoint at bench's shape (pipelined halves of 4 images at 600x1024; the stem is tested
  through its tap below), the RPN conv and heads, and the RCNN heads on 2000 proposals x 4 images;
* resnet_v1_101's block4 tail on the pooled ROI maps of 300 proposals x 4 images (bench's frcnn_r101);
* resnet_v2_50's conv3 layers, which write the next unit's pre-activation (x and p, or p only);
* block3 of resnet_v1_50 at output_stride 8 (rate 2 on 75x128 maps);
* every conv of the default SSD but conv1_1 (tested through its tap) on halves of a batch of 32 at 300x300.
The geometry follows the TF padding arithmetic, as the engine's layer table derives it.

* Parity: each row runs through lumi_op_conv2d_io as the engine launches it (impl 16 / 17: split outputs on all SMs
  and with the pipelined half-batch's SMs reserved; 18 / 19 the same with fp32 outputs), and is held to the
  per-element bound of test_gpu_conv_numerics at sampled output pixels (every border pixel of each image and one
  random pixel per 16 consecutive ones, all channels): a float64 conv of the big layers is out of a CPU's reach.
  Inputs are drawn as the engine sees them: non-negative after a ReLU, BN-folded scales, a residual of the scale of
  the layer's output.  Run with -s for each row's largest err / bound.
* Mainloops: the single-buffered mainloop the engine runs and the double-buffered one (impl | 32, LUMI_CONV_PIPE=1)
  give byte-identical outputs on every row, on whole tiles and on forced stream-K, and so do whole engines.
* The Toeplitz-view convs (the ResNet stem over its space-to-depth staging, SSD's conv1_1 over its packed pixels),
  through the `stem` and `conv1_1` debug taps, against float64 at sampled pixels with the packed K.
"""
import collections
import ctypes
import zlib

import numpy as np
import pytest

import gpu_ops as G
from test_gpu_conv_numerics import PAD, check, out_geometry, preact_reference, reference

f32, f64 = np.float32, np.float64

# lumi_op_conv2d codes (include/luminoth_b200.h)
WHOLE, WHOLE_EPI16, STREAMK_EPI16, F32_WHOLE, F32_STREAMK = 3, 4, 5, 1, 2
ENGINE, ENGINE_RESERVE, ENGINE_F32, ENGINE_F32_RESERVE = 16, 17, 18, 19
PIPE = 32                 # | on codes 1-12: the double-buffered mainloop
EPI16_K_SLICES = 16       # CONV_EPI16_DEFAULT: the four-warpgroup kernel's K-slice bound

BASE_DEPTH = (64, 128, 256, 512)
BLOCK_STRIDE = (2, 2, 2, 1)
R50_UNITS = (3, 4, 6, 3)
RELU, RELU6 = 1, 2

# res: None or (res_h, res_w, res_stride, res_nonneg); pre: None, 'x_and_p' or 'p_only'; x_nonneg: the layer reads a
# ReLU output; parts: the C_out of each weight variable a fused conv concatenates
Row = collections.namedtuple('Row', 'name n h w cin cout k stride rate padding res act f32 pre x_nonneg bn parts')


def _row(name, n, h, w, cin, cout, k=1, stride=1, rate=1, padding='SAME', res=None, act=0, fp32=False, pre=None,
         x_nonneg=True, bn=True, parts=None):
    return Row(name, n, h, w, cin, cout, k, stride, rate, padding, res, act, fp32, pre, x_nonneg, bn,
               tuple(parts or (cout,)))


def unit_stride_rate(units, output_stride, b, u):
    """conv2 stride and rate of unit (b, u) as slim's stack_blocks_dense sets them at output_stride."""
    target, current, r = output_stride // 4, 1, 1
    for bb in range(b + 1):
        for uu in range(units[bb]):
            s = BLOCK_STRIDE[bb] if uu == units[bb] - 1 else 1
            atrous = current == target
            if (bb, uu) == (b, u):
                return (1, r) if atrous else (s, 1)
            if atrous:
                r *= s
            else:
                current *= s


def resnet_rows(tag, n, h, w, units=R50_UNITS, output_stride=16, blocks=(0, 1, 2), v2=False, hw=None):
    """The bottleneck convs of `blocks`; hw: the first block's input resolution (default: after the stem and pool)."""
    if hw is None:
        ho, wo, _, _ = out_geometry(h, w, 7, 2, 1, 'SLIM')
        hw = (-(-ho // 2), -(-wo // 2))                              # pool1 3x3/2 SAME
    rows = []
    for b in blocks:
        bd, depth = BASE_DEPTH[b], BASE_DEPTH[b] * 4
        for u in range(units[b]):
            cin = depth if u else (BASE_DEPTH[b - 1] * 4 if b else 64)
            st, rt = (1, 1) if b == 3 and tag.endswith('tail') else unit_stride_rate(units, output_stride, b, u)
            s = '%s/block%d/unit_%d/' % (tag, b + 1, u + 1)
            ho, wo, _, _ = out_geometry(hw[0], hw[1], 3, st, rt, 'SLIM')
            project = cin != depth
            if project and not v2:
                rows.append(_row(s + 'shortcut', n, hw[0], hw[1], cin, depth, stride=st))
            if not v2:
                rows.append(_row(s + 'conv1', n, hw[0], hw[1], cin, bd, act=RELU))
                rows.append(_row(s + 'conv2', n, hw[0], hw[1], bd, bd, 3, st, rt, 'SLIM', act=RELU))
            # conv3's residual: the projection at the output's resolution, or the unit's input subsampled by st
            res = (ho, wo, 1, False) if project else (hw[0], hw[1], st, not v2)
            if v2:
                last = b == blocks[-1] and u == units[b] - 1
                nxt_projects = u == units[b] - 1
                pre = None if last else ('p_only' if nxt_projects else 'x_and_p')
                if pre:
                    rows.append(_row(s + 'conv3', n, ho, wo, bd, depth, res=res, pre=pre, bn=False))
            else:
                rows.append(_row(s + 'conv3', n, ho, wo, bd, depth, res=res, act=RELU))
            hw = (ho, wo)
    return rows, hw


def frcnn_heads(tag, n, hw, depth, classes=80, anchors=12, post=2000):
    return [_row(tag + '/rpn/conv', n, hw[0], hw[1], depth, 512, 3, act=RELU6, bn=False),
            _row(tag + '/rpn/heads', n, hw[0], hw[1], 512, 6 * anchors, fp32=True, bn=False,
                 parts=(2 * anchors, 4 * anchors)),
            _row(tag + '/rcnn/heads', n * post, 1, 1, depth, 5 * classes + 1, fp32=True, bn=False,
                 parts=(classes + 1, 4 * classes))]


def ssd_rows(n=16, size=300, classes=20, anchors=(4, 6, 6, 6, 4, 4)):
    rows, hw, cin, fmaps = [], size, 64, []
    for b, (reps, ch) in enumerate(zip((2, 2, 3, 3, 3), (64, 128, 256, 512, 512))):
        for r in range(reps):
            if (b, r) != (0, 0):                                     # conv1_1: the packed Toeplitz view
                rows.append(_row('ssd/conv%d_%d' % (b + 1, r + 1), n, hw, hw, cin, ch, 3, act=RELU, bn=False))
            cin = ch
        if b == 3:
            fmaps.append((hw, 512))
        if b < 4:
            hw = (hw - 2) // 2 + 1                                   # 2x2/2 VALID
    extras = [('conv6', 3, 1024, 1, 6, 'SAME'), ('conv7', 1, 1024, 1, 1, 'SAME'), ('conv8_1', 1, 256, 1, 1, 'SAME'),
              ('conv8_2', 3, 512, 2, 1, 'SAME'), ('conv9_1', 1, 128, 1, 1, 'SAME'), ('conv9_2', 3, 256, 2, 1, 'SAME'),
              ('conv10_1', 1, 128, 1, 1, 'SAME'), ('conv10_2', 3, 256, 1, 1, 'VALID'),
              ('conv11_1', 1, 128, 1, 1, 'SAME'), ('conv11_2', 3, 256, 1, 1, 'VALID')]
    for i, (name, k, cout, st, rt, pad) in enumerate(extras):
        rows.append(_row('ssd/' + name, n, hw, hw, cin, cout, k, st, rt, pad, act=RELU, bn=False))
        hw = out_geometry(hw, hw, k, st, rt, pad)[0]
        cin = cout
        if i in (1, 3, 5, 7, 9):
            fmaps.append((hw, cout))
    for i, ((s, ch), a) in enumerate(zip(fmaps, anchors)):
        rows.append(_row('ssd/MultiBox_%d' % i, n, s, s, ch, a * (5 + classes), 3, fp32=True, bn=False,
                         parts=(4 * a, (classes + 1) * a)))
    return rows


def _dedupe(rows):
    """One row per distinct launch: rows that differ only in name are the same launch."""
    seen, out = set(), []
    for r in rows:
        key = r[1:]
        if key not in seen:
            seen.add(key)
            out.append(r)
    return out


def _layers():
    rows, hw = resnet_rows('r50', 4, 600, 1024)
    rows += frcnn_heads('r50', 4, hw, 1024)
    tail, _ = resnet_rows('r101_tail', 1200, 0, 0, blocks=(3,), hw=(7, 7))
    rows += tail + frcnn_heads('r101', 4, hw, 2048, post=300)[2:]
    rows += resnet_rows('r50_v2', 4, 600, 1024, v2=True)[0]
    _, hw8 = resnet_rows('r50_os8', 4, 600, 1024, output_stride=8, blocks=(0, 1))
    rows += resnet_rows('r50_os8', 4, 600, 1024, output_stride=8, blocks=(2,), hw=hw8)[0]
    rows += ssd_rows()
    return _dedupe(rows)


LAYERS = _layers()
IDS = [r.name for r in LAYERS]


# ---------------------------------------------------------------------------------------------- inputs and launches
def _inputs(row):
    rng = np.random.default_rng(zlib.crc32(row.name.encode()))
    x = rng.standard_normal((row.n, row.h, row.w, row.cin), dtype=f32)
    if row.x_nonneg:
        np.abs(x, out=x)
    w = (rng.standard_normal((row.k, row.k, row.cin, row.cout)) * np.sqrt(2.0 / (row.k * row.k * row.cin))).astype(f32)
    if row.bn:                                                       # gamma / sqrt(var + eps), beta - mean * scale
        scale = rng.uniform(0.5, 1.5, row.cout).astype(f32)
        bias = (rng.standard_normal(row.cout) * 0.1).astype(f32)
    else:
        scale, bias = None, (rng.standard_normal(row.cout) * 0.05).astype(f32)
    res = None
    if row.res:
        rh, rw, _, nonneg = row.res
        res = rng.standard_normal((row.n, rh, rw, row.cout), dtype=f32)
        if nonneg:
            np.abs(res, out=res)
    pre = None
    if row.pre:
        pre = (rng.uniform(0.5, 1.5, row.cout).astype(f32), (rng.standard_normal(row.cout) * 0.1).astype(f32))
    return x, w, scale, bias, res, pre


class Launch(object):
    """The row's inputs on the device; run(impl) -> (x output, pre-activation output) as CUDA float32 tensors."""

    def __init__(self, row, inputs):
        self.row = row
        self.x, self.w, self.scale, self.bias, self.res, self.pre = inputs
        self.d = [G._dev(a, f32) if a is not None else None for a in (self.x, self.w, self.scale, self.bias, self.res)]
        self.dpre = [G._dev(a, f32) for a in self.pre] if self.pre else [None, None]

    def run(self, impl):
        import torch
        r = self.row
        rh, rw, rs = (r.res[0], r.res[1], r.res[2]) if r.res else (0, 0, 1)
        xd, wd, sd, bd, rd = self.d
        args = [G._p(xd), r.n, r.h, r.w, r.cin, G._p(wd), r.k, r.k, r.cout, r.stride, r.rate, PAD[r.padding],
                G._p(sd), G._p(bd), G._p(rd), rh, rw, rs, r.act, impl, G._p(self.dpre[0]), G._p(self.dpre[1])]
        ho, wo = ctypes.c_int(), ctypes.c_int()
        lib = G._lib()
        G._check(lib.lumi_op_conv2d_io(*args, None, None, ctypes.byref(ho), ctypes.byref(wo), None))
        shape = (r.n, ho.value, wo.value, r.cout)
        y = None if r.pre == 'p_only' else torch.empty(shape, dtype=torch.float32, device='cuda')
        p = torch.empty(shape, dtype=torch.float32, device='cuda') if r.pre else None
        G._check(lib.lumi_op_conv2d_io(*args, G._p(y), G._p(p), ctypes.byref(ho), ctypes.byref(wo), None))
        torch.cuda.synchronize()
        return y, p


def sample_pixels(n, ho, wo, seed):
    """(img, oy, ox): every pixel of each image's border rows and columns, and one random pixel in every 16
    consecutive output pixels."""
    rng = np.random.default_rng(seed)
    total = n * ho * wo
    flat = np.arange(0, total, 16) + rng.integers(0, 16, -(-total // 16))
    flat = flat[flat < total]
    img, oy, ox = np.meshgrid(np.arange(n), np.arange(ho), np.arange(wo), indexing='ij', sparse=True)
    border = ((oy == 0) | (oy == ho - 1) | (ox == 0) | (ox == wo - 1)) & (img >= 0)
    flat = np.union1d(flat, np.flatnonzero(border))
    img, rem = np.divmod(flat, ho * wo)
    return img, rem // wo, rem % wo


def _gather(t, at):
    import torch
    idx = [torch.as_tensor(a, device='cuda') for a in at]
    return t[idx[0], idx[1], idx[2]].cpu().numpy()


def _four_warpgroup(row):
    return row.k * row.k * row.cin // 64 <= EPI16_K_SLICES


# ---------------------------------------------------------------------------------------------- host checks
def test_sampled_bound_matches_the_full_bound():
    """The sampled float64 reference and bound equal the full ones at every pixel (stride 1 / 2, every padding,
    square, non-square and even kernels)."""
    rng = np.random.default_rng(7)
    for k, stride, padding, res_stride in [(3, 1, 'SAME', 1), (3, 2, 'SLIM', 1), (1, 1, 'SAME', 2), (3, 1, 'VALID', 1),
                                           (7, 2, 'SLIM', 1), (3, 2, 'SAME', 1), ((5, 3), 1, 'SAME', 1),
                                           ((3, 5), 2, 'SAME', 1), ((1, 7), 1, 'VALID', 1), ((7, 1), 2, 'VALID', 1),
                                           ((2, 2), 1, 'SAME', 1), ((4, 4), 2, 'SAME', 1), ((2, 2), 2, 'VALID', 1)]:
        kh, kw = (k, k) if isinstance(k, int) else k
        x = rng.standard_normal((2, 11, 14, 8)).astype(f32)
        w = rng.standard_normal((kh, kw, 8, 5)).astype(f32)
        scale, bias = rng.uniform(0.5, 1.5, 5).astype(f32), rng.standard_normal(5).astype(f32)
        ho, wo, _, _ = out_geometry(11, 14, kh, stride, 1, padding, kw=kw)
        res = rng.standard_normal((2, ho * res_stride, wo * res_stride, 5)).astype(f32)
        at = tuple(a.ravel() for a in np.meshgrid(np.arange(2), np.arange(ho), np.arange(wo), indexing='ij'))
        for impl in (0, ENGINE):
            ref, bound = reference(x, w, stride, padding, scale, bias, res, res_stride, RELU, impl)
            assert ref.shape == (2, ho, wo, 5)
            sref, sbound = reference(x, w, stride, padding, scale, bias, res, res_stride, RELU, impl, at=at)
            np.testing.assert_allclose(sref, ref.reshape(-1, 5), rtol=1e-12, atol=1e-12)
            np.testing.assert_allclose(sbound, bound.reshape(-1, 5), rtol=1e-12)


def test_pixel_sample_covers_borders_and_every_16_pixels():
    n, ho, wo = 3, 19, 37
    img, oy, ox = sample_pixels(n, ho, wo, 1)
    flat = (img * ho + oy) * wo + ox
    assert len(np.unique(flat)) == len(flat)
    assert np.all(np.bincount(flat // 16, minlength=-(-n * ho * wo // 16)) >= 1)
    for i in range(n):
        on = set(zip(oy[img == i].tolist(), ox[img == i].tolist()))
        assert all((y, x) in on for y in (0, ho - 1) for x in range(wo))
        assert all((y, x) in on for x in (0, wo - 1) for y in range(ho))


def test_layer_table_geometry():
    """Spot checks of the derived shapes against the engine's known maps: R50 block3 at 38x64 (600x1024, output
    stride 16), 75x128 at output stride 8, SSD's feature maps 37 / 18 / 9 / 5 / 3 / 1, fc6 at rate 6."""
    by = {r.name: r for r in LAYERS}
    assert (by['r50/block3/unit_1/conv1'].h, by['r50/block3/unit_1/conv1'].w) == (38, 64)
    assert (by['r50/rpn/conv'].h, by['r50/rpn/conv'].w, by['r50/rpn/conv'].cin) == (38, 64, 1024)
    assert by['r50/block2/unit_4/conv3'].res == (75, 128, 2, True)
    os8 = by['r50_os8/block3/unit_1/conv2']
    assert (os8.h, os8.w, os8.rate, os8.stride) == (75, 128, 2, 1)
    assert [by['ssd/MultiBox_%d' % i].h for i in range(6)] == [37, 18, 9, 5, 3, 1]
    assert (by['ssd/conv6'].rate, by['ssd/conv6'].h) == (6, 18)
    assert by['r101_tail/block4/unit_1/conv1'].cin == 1024 and _four_warpgroup(by['r101_tail/block4/unit_1/conv1'])
    assert by['r50/rcnn/heads'].n == 8000 and by['r101/rcnn/heads'].n == 1200


# ---------------------------------------------------------------------------------------------- GPU: coverage
COVERED_BY_TAPS = {(7, 7, 3, 64), (3, 3, 3, 64)}     # the stem and SSD's conv1_1: test_toeplitz_view_* below


def _covered(kh, kw, cin, cout):
    return (kh, kw, cin, cout) in COVERED_BY_TAPS or any(
        (r.k, r.k, r.cin) == (kh, kw, cin) and cout in r.parts for r in LAYERS)


@pytest.mark.gpu
@pytest.mark.parametrize('mtype,params', [
    ('fasterrcnn', ['model.base_network.architecture=resnet_v1_50', 'model.network.num_classes=80']),
    ('fasterrcnn', ['model.base_network.architecture=resnet_v1_101', 'model.network.num_classes=80']),
    ('fasterrcnn', ['model.base_network.architecture=resnet_v2_50', 'model.network.num_classes=80']),
    ('fasterrcnn', ['model.base_network.architecture=resnet_v1_50', 'model.base_network.output_stride=8']),
    ('ssd', []),
], ids=['r50', 'r101', 'r50_v2', 'r50_os8', 'ssd'])
def test_layer_table_covers_every_conv_weight(mtype, params):
    """Every 4-D conv weight the engine loads for the configs has a row of its (kh, kw, C_in, C_out)."""
    from luminoth_b200 import default_config
    from luminoth_b200.engine import Engine
    eng = Engine(default_config(mtype, params))
    specs = [(name, shape) for name, shape in eng.weight_specs()
             if len(shape) == 4 and name.rsplit('/', 1)[-1] in ('weights', 'w')]
    eng.close()
    assert specs
    missing = [name for name, shape in specs if not _covered(*shape)]
    assert not missing, 'conv weights without a layer row: %s' % missing


# ---------------------------------------------------------------------------------------------- GPU: parity
@pytest.mark.gpu
@pytest.mark.parametrize('row', LAYERS, ids=IDS)
def test_engine_launch_matches_float64(row):
    """Codes 16 / 17 (18 / 19 for fp32 outputs) against float64 at the sampled pixels."""
    inputs = _inputs(row)
    x, w, scale, bias, res, pre = inputs
    launch = Launch(row, inputs)
    codes = (ENGINE_F32, ENGINE_F32_RESERVE) if row.f32 else (ENGINE, ENGINE_RESERVE)
    ho, wo, _, _ = out_geometry(row.h, row.w, row.k, row.stride, row.rate, row.padding)
    at = sample_pixels(row.n, ho, wo, zlib.crc32(row.name.encode()) + 1)
    rs = row.res[2] if row.res else 1
    ref, bound = reference(x, w, row.stride, row.padding, scale, bias, res, rs, row.act, codes[0], rate=row.rate, at=at)
    if pre:
        pref, pbound = preact_reference(ref, bound, *pre)
    for impl in codes:
        y, p = launch.run(impl)
        tag = '%s/impl%d (%d px)' % (row.name, impl, len(at[0]))
        if y is not None:
            assert y.shape == (row.n, ho, wo, row.cout)
            check(tag, _gather(y, at), ref, bound)
        if p is not None:
            check(tag + '/p', _gather(p, at), pref, pbound)


@pytest.mark.gpu
@pytest.mark.parametrize('row', LAYERS, ids=IDS)
def test_double_buffered_mainloop_is_bit_identical(row):
    """impl and impl | 32 write the same bytes, on whole tiles (the four-warpgroup kernel where the engine takes it)
    and on forced stream-K."""
    launch = Launch(row, _inputs(row))
    if row.f32:
        codes = (F32_WHOLE, F32_STREAMK)
    else:
        codes = (WHOLE_EPI16 if _four_warpgroup(row) else WHOLE, STREAMK_EPI16)
    import torch
    for impl in codes:
        one = launch.run(impl)
        two = launch.run(impl | PIPE)
        for a, b, what in zip(one, two, ('x', 'p')):
            if a is not None:
                assert a.view(torch.int32).equal(b.view(torch.int32)), \
                    '%s impl %d %s: max abs diff %.3e' % (row.name, impl, what, float((a - b).abs().max()))


@pytest.mark.gpu
def test_pipe_flag_is_rejected_off_codes_1_to_12():
    import torch
    lib = G._lib()
    x, w = G._dev(np.ones((1, 4, 4, 64), f32)), G._dev(np.ones((1, 1, 64, 256), f32))
    y = torch.empty((1, 4, 4, 256), dtype=torch.float32, device='cuda')
    for impl in (0, 13, 14, 15, ENGINE, ENGINE_RESERVE, ENGINE_F32, ENGINE_F32_RESERVE):
        rc = lib.lumi_op_conv2d(G._p(x), 1, 4, 4, 64, G._p(w), 1, 1, 256, 1, 1, 1, None, None, None, 0, impl | PIPE,
                                G._p(y), None, None, None)
        assert rc != 0, 'impl %d | 32 was accepted' % impl
        assert 'impl' in lib.lumi_op_last_error().decode()
    for impl in (1, 3, 12):
        G._check(lib.lumi_op_conv2d(G._p(x), 1, 4, 4, 64, G._p(w), 1, 1, 256, 1, 1, 1, None, None, None, 0,
                                    impl | PIPE, G._p(y), None, None, None))


# ---------------------------------------------------------------------------------------------- GPU: whole engines
def _frcnn_cfg():
    from luminoth_b200 import default_config
    return default_config('fasterrcnn', ['model.base_network.architecture=resnet_v1_50', 'model.network.num_classes=20',
                                         'model.rpn.proposals.post_nms_top_n=200',
                                         'model.rcnn.proposals.min_prob_threshold=0.05'])


def _engine_outputs(cfg, wts, imgs, taps):
    from luminoth_b200.engine import Engine
    n, h, w, _ = imgs.shape
    eng = Engine(cfg, max_batch=n, max_h=h, max_w=w)
    eng.load_weights(wts).finalize()
    out = {}
    for mode in ('off', 'always'):
        eng.set_conv_streamk(mode)
        eng.set_debug_taps(False)
        out[mode + '/pipelined'] = eng.predict_raw(imgs)
        eng.set_debug_taps(True)
        out[mode + '/taps'] = eng.predict_raw(imgs)
        for t in taps:
            out[mode + '/' + t] = (eng.get_tensor(t),)
    eng.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('model', ['r50', 'ssd'])
def test_double_buffered_engine_is_bit_identical(model, monkeypatch):
    """LUMI_CONV_PIPE=1 (read at engine creation) changes no byte of the detections or the feature maps, on whole
    tiles and on stream-K: R50 at batch 2 x 224x320, SSD at batch 3 (pipelined halves of 2 and 1)."""
    from luminoth_b200 import default_config, synth
    if model == 'r50':
        cfg, imgs, taps = _frcnn_cfg(), synth.make_images(2, 224, 320, seed=11), ['conv_feature_map', 'stem']
    else:
        cfg = default_config('ssd', ['model.proposals.min_prob_threshold=0.2'])
        imgs, taps = synth.make_images(3, 300, 300, seed=12), ['conv1_1'] + ['fmap_%d' % i for i in range(6)]
    wts = synth.make_weights(cfg, seed=13)
    monkeypatch.delenv('LUMI_CONV_PIPE', raising=False)
    single = _engine_outputs(cfg, wts, imgs, taps)
    monkeypatch.setenv('LUMI_CONV_PIPE', '1')
    double = _engine_outputs(cfg, wts, imgs, taps)
    assert sorted(single) == sorted(double)
    for key in sorted(single):
        for a, b in zip(single[key], double[key]):
            assert a.tobytes() == b.tobytes(), '%s/%s differs' % (model, key)


# ---------------------------------------------------------------------------------------------- GPU: Toeplitz views
RGB_MEANS = np.array([123.68, 116.78, 103.94], f32)


def _bn_fold(wts, scope):
    """The engine's fold (make_conv_bn): s = gamma / sqrt(var + eps) in double, rounded once; b = beta - mean * s."""
    g, b, m, v = (wts[scope + '/BatchNorm/' + k].astype(f64) for k in ('gamma', 'beta', 'moving_mean', 'moving_variance'))
    s = g / np.sqrt(v + 1e-5)
    return s.astype(f32), (b - m * s).astype(f32)


@pytest.mark.gpu
@pytest.mark.parametrize('n,h,w', [(8, 600, 1024), (1, 375, 501)], ids=['r50_8x600x1024', 'r50_375x501'])
def test_toeplitz_view_stem_matches_float64(n, h, w):
    """The stem conv (7x7/2 over image - mean as four K = 64 taps of the space-to-depth staging) per element at
    sampled pixels, K = 256 in the fold count."""
    stem_against_float64(n, h, w)


def stem_against_float64(n, h, w):
    """The `stem` tap of a batch of n h x w images against float64 at sampled pixels; returns the largest err / bound."""
    from luminoth_b200 import synth
    from luminoth_b200.engine import Engine
    cfg = _frcnn_cfg()
    wts = synth.make_weights(cfg, seed=21)
    imgs = synth.make_images(n, h, w, seed=22)
    eng = Engine(cfg, max_batch=n, max_h=h, max_w=w)
    eng.load_weights(wts).finalize()
    eng.set_debug_taps(True)
    eng.predict_raw(imgs)
    stem = eng.get_tensor('stem')
    eng.close()
    ho, wo, _, _ = out_geometry(h, w, 7, 2, 1, 'SLIM')
    assert stem.shape == (n, ho, wo, 64)
    root = 'truncated_base_network/resnet_v1_50/conv1'
    scale, bias = _bn_fold(wts, root)
    x = imgs.astype(f32) - RGB_MEANS                                   # the engine's fp32 image - mean
    at = sample_pixels(n, ho, wo, 23)
    ref, bound = reference(x, wts[root + '/weights'], 2, 'SLIM', scale, bias, None, 1, RELU, ENGINE, at=at, k_fold=256)
    return check('stem %dx%dx%d (%d px)' % (n, h, w, len(at[0])), stem[at], ref, bound)


@pytest.mark.gpu
def test_toeplitz_view_conv1_1_matches_float64():
    """SSD's conv1_1 (3x3 over the raw pixels as three K = 64 filter rows of the packed staging) at batch 32, per
    element at sampled pixels, K = 192 in the fold count."""
    from luminoth_b200 import default_config, synth
    from luminoth_b200.engine import Engine
    cfg = default_config('ssd', [])
    wts = synth.make_weights(cfg, seed=31)
    imgs = synth.make_images(32, 300, 300, seed=32)
    eng = Engine(cfg, max_batch=32)
    eng.load_weights(wts).finalize()
    eng.set_debug_taps(True)
    eng.predict_raw(imgs)
    y = eng.get_tensor('conv1_1')
    eng.close()
    assert y.shape == (32, 300, 300, 64)
    p = 'ssd/ssd_feature_extractor/vgg_16/conv1/conv1_1'
    at = sample_pixels(32, 300, 300, 33)
    ref, bound = reference(imgs, wts[p + '/weights'], 1, 'SAME', None, wts[p + '/biases'], None, 1, RELU, ENGINE, at=at,
                           k_fold=192)
    check('conv1_1 32x300x300 (%d px)' % len(at[0]), y[at], ref, bound)
