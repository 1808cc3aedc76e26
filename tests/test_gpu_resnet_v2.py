"""resnet_v1_152 and the pre-activation resnet_v2 base networks on the GPU (`-m gpu`): the pre-activation output
of the conv epilogue and of the max pool, then Faster R-CNN end to end against the CPU oracle."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import gpu_ops as G
import resnet_v2_oracle as V2
from luminoth_b200 import synth
from luminoth_b200.engine import Engine, LUMI_EOVERFLOW
from oracle import fasterrcnn as ofr
from oracle import tf_ops as T
from test_gpu_e2e import box_dev, float_bound, frcnn_cfg, rel_err, _report

f16, f32 = np.float16, np.float32

# lumi_op_conv2d_preact impl codes: 0 SIMT; split planes through the slot epilogue with two consumer warpgroups (3), four
# allowed (4), four + stream-K (5); 2-CTA clusters with the register epilogue (6, 7: + stream-K); 12: as 3 with the
# register epilogue
IMPLS = [0, 3, 4, 5, 6, 7, 12]
OP_IMPL = {0: 'simt', 3: 'tc_split', 4: 'tc_split_epi16', 5: 'tc_split_epi16_streamk', 6: 'tc_split_cta2',
           7: 'tc_split_cta2_streamk'}

# (n, h, w, cin, kh, cout, stride, padding, residual, act): a conv3-like 1x1 layer with a residual on a ragged map,
# C_out = 64 (BN = 64), C_out = 96 (channel box clipped by TMA), a stride-2 3x3
SHAPES = [
    (2, 13, 21, 64, 1, 256, 1, 'SAME', True, 0),
    (1, 11, 19, 128, 1, 64, 1, 'SAME', True, 0),
    (2, 9, 14, 64, 1, 96, 1, 'SAME', False, 1),
    (2, 17, 23, 64, 3, 128, 2, 'SLIM', False, 1),
]


def split(v):
    v = np.asarray(v, f32)
    hi = v.astype(f16)
    lo = (v - hi.astype(f32)).astype(f16)
    return hi.astype(f32) + lo.astype(f32)


def preact_ref(xhat, s, b):
    """p = relu(fmaf(x^, s, b)) rounded once to fp32; returns the three fp32 values within one ulp."""
    p = np.maximum(xhat.astype(np.float64) * s.astype(np.float64) + b.astype(np.float64), 0.0).astype(f32)
    return p, np.nextafter(p, f32(-np.inf)), np.nextafter(p, f32(np.inf))


def conv2d_preact(x, w, stride, padding, scale, bias, residual, act, impl, pre_scale, pre_bias, want_x):
    lib = G._lib()
    n, h, wd, cin = x.shape
    kh, kw, _, cout = w.shape
    pad = {'VALID': 0, 'SAME': 1, 'SLIM': 2}[padding]
    xd, wdv, sd, bd = G._dev(x, f32), G._dev(w, f32), G._dev(scale, f32), G._dev(bias, f32)
    rd = G._dev(residual, f32) if residual is not None else None
    psd, pbd = G._dev(pre_scale, f32), G._dev(pre_bias, f32)
    ho, wo = ctypes.c_int(), ctypes.c_int()
    args = [G._p(xd), n, h, wd, cin, G._p(wdv), kh, kw, cout, stride, 1, pad, G._p(sd), G._p(bd), G._p(rd), act, impl,
            G._p(psd), G._p(pbd)]
    G._check(lib.lumi_op_conv2d_preact(*args, None, None, ctypes.byref(ho), ctypes.byref(wo), None))
    import torch
    y = torch.empty((n, ho.value, wo.value, cout), dtype=torch.float32, device='cuda') if want_x else None
    p = torch.empty((n, ho.value, wo.value, cout), dtype=torch.float32, device='cuda')
    rc = lib.lumi_op_conv2d_preact(*args, G._p(y), G._p(p), ctypes.byref(ho), ctypes.byref(wo), None)
    if rc == LUMI_EOVERFLOW:
        return rc, None, None
    G._check(rc)
    torch.cuda.synchronize()
    return rc, (y.cpu().numpy() if want_x else None), p.cpu().numpy()


def _case(shape, seed):
    n, h, w, cin, kh, cout, stride, padding, with_res, act = shape
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, h, w, cin)).astype(f32)
    wt = (rng.standard_normal((kh, kh, cin, cout)) * np.sqrt(2.0 / (kh * kh * cin))).astype(f32)
    scale = rng.uniform(0.5, 1.5, cout).astype(f32)
    bias = (rng.standard_normal(cout) * 0.1).astype(f32)
    pre_scale = rng.uniform(-1.5, 1.5, cout).astype(f32)        # negative gammas too
    pre_bias = (rng.standard_normal(cout) * 0.2).astype(f32)
    pad = {'VALID': 0, 'SAME': 1, 'SLIM': 2}[padding]
    ho = (h - 1) // stride + 1 if pad else (h - kh) // stride + 1
    wo = (w - 1) // stride + 1 if pad else (w - kh) // stride + 1
    res = rng.standard_normal((n, ho, wo, cout)).astype(f32) if with_res else None
    return x, wt, stride, padding, scale, bias, res, act, pre_scale, pre_bias


@pytest.mark.parametrize('impl', IMPLS)
@pytest.mark.parametrize('si', range(len(SHAPES)))
def test_conv2d_preact_modes(impl, si):
    x, wt, stride, padding, scale, bias, res, act, ps, pb = _case(SHAPES[si], seed=10 + si)
    # code 12 (register epilogue) is bit-identical to code 3 (slot epilogue): test_gpu_conv_epilogue
    y_ref = G.conv2d(x, wt, stride=stride, padding=padding, scale=scale, bias=bias, residual=res, act=act,
                     impl=OP_IMPL[3 if impl == 12 else impl])
    if impl == 0:       # lumi_op_conv2d's SIMT path returns fp32; the engine stores the split planes
        y_ref = split(y_ref)
    rc, y, p = conv2d_preact(x, wt, stride, padding, scale, bias, res, act, impl, ps, pb, want_x=True)
    assert rc == 0
    np.testing.assert_array_equal(y, y_ref)                     # x: bit-identical to the plain conv
    cands = preact_ref(y, ps, pb)
    ok = np.zeros(p.shape, bool)
    for c in cands:
        ok |= p == split(c)
    assert ok.all(), 'p differs from relu(fmaf(x^, s, b)) by more than one fp32 ulp at %d places' % (~ok).sum()
    rc, none, p_only = conv2d_preact(x, wt, stride, padding, scale, bias, res, act, impl, ps, pb, want_x=False)
    assert rc == 0 and none is None
    np.testing.assert_array_equal(p_only, p)                    # p-only mode writes the same p
    # an fp16 overflow in p (not in x) raises LUMI_EOVERFLOW, in both modes
    big = ps.copy()
    big[3] = 1e6
    for want_x in (True, False):
        rc, _, _ = conv2d_preact(x, wt, stride, padding, scale, bias, res, act, impl, big, np.full_like(pb, 1e5),
                                 want_x=want_x)
        assert rc == LUMI_EOVERFLOW


@pytest.mark.parametrize('negative', [False, True])
def test_max_pool_preact(negative):
    """p = relu(BN(max pool)) with the batch norm after the max (negative gammas do not commute with it); an
    all-negative input checks that SAME padding never enters the max."""
    rng = np.random.default_rng(5)
    x = rng.standard_normal((2, 15, 22, 64)).astype(f32)
    if negative:
        x = -np.abs(x) - 0.5
    ps = rng.uniform(-1.5, 1.5, 64).astype(f32)
    pb = (rng.standard_normal(64) * 0.2).astype(f32)
    lib = G._lib()
    import torch
    xd, psd, pbd = G._dev(x), G._dev(ps), G._dev(pb)
    y = torch.empty((2, 8, 11, 64), dtype=torch.float32, device='cuda')
    G._check(lib.lumi_op_max_pool_preact(G._p(xd), 2, 15, 22, 64, 3, 2, 1, G._p(psd), G._p(pbd), G._p(y), None))
    got = y.cpu().numpy()
    m = T.max_pool(split(x), 3, 2, 'SAME')
    assert (m < 0).all() == negative
    ok = np.zeros(got.shape, bool)
    for c in preact_ref(split(m), ps, pb):
        ok |= got == split(c)
    assert ok.all()
    plain = G.max_pool(x, 3, 2, 'SAME')                          # the unchanged op still returns the max
    np.testing.assert_array_equal(plain, split(m))


@pytest.mark.parametrize('arch,impl', [('resnet_v1_152', 'tc'), ('resnet_v2_50', 'simt'), ('resnet_v2_50', 'tc'),
                                       ('resnet_v2_101', 'tc'), ('resnet_v2_152', 'tc')])
def test_fasterrcnn_new_archs_stages_and_detections(arch, impl):
    cfg = frcnn_cfg(arch)
    wts = synth.make_weights(cfg, seed=1)
    h, w = 224, 320
    imgs = synth.make_images(2, h, w, seed=2)
    eng = Engine(cfg, max_batch=2, max_h=h, max_w=w)
    eng.load_weights(wts).finalize()
    eng.set_conv_impl(impl)
    eng.set_debug_taps(True)
    boxes, scores, labels, counts = eng.predict_raw(imgs)
    fmap = eng.get_tensor('conv_feature_map')
    heads = eng.get_tensor('rpn_heads')
    props = eng.get_tensor('proposals')
    pcnt = eng.get_tensor('proposal_counts').astype(int)
    cls_prob = eng.get_tensor('rcnn_cls_prob')
    pooled = eng.get_tensor('roi_pool')
    for i in range(2):
        ref = V2.fasterrcnn_forward(imgs[i], wts, cfg)
        tru = V2.fasterrcnn_forward(imgs[i], wts, cfg, dtype=np.float64)
        e_fm = rel_err(fmap[i], tru['conv_feature_map'][0])
        o_fm = rel_err(ref['conv_feature_map'][0], tru['conv_feature_map'][0])
        A = 12
        rh = heads[i].reshape(-1, 6 * A)
        lg = np.concatenate([rh[:, :2 * A].reshape(-1), rh[:, 2 * A:].reshape(-1)])
        lg_t = np.concatenate([tru['rpn']['rpn_cls_score'].reshape(-1), tru['rpn']['rpn_bbox_pred'].reshape(-1)])
        lg_r = np.concatenate([ref['rpn']['rpn_cls_score'].reshape(-1), ref['rpn']['rpn_bbox_pred'].reshape(-1)])
        e_lg, o_lg = rel_err(lg, lg_t), rel_err(lg_r, lg_t)
        tp, rp = tru['rpn_prediction']['proposals'], ref['rpn_prediction']['proposals']
        assert pcnt[i] == tp.shape[0], 'proposal count %d vs %d' % (pcnt[i], tp.shape[0])
        z = np.zeros(pcnt[i], int)
        e_pr, o_pr = box_dev(props[i, :pcnt[i]], z, tp, z), box_dev(rp, z, tp, z)
        k = int(counts[i])
        tc_, rc_ = tru['classification_prediction'], ref['classification_prediction']
        e_det = box_dev(boxes[i, :k], labels[i, :k], tc_['objects'], tc_['labels'])
        o_det = box_dev(rc_['objects'], rc_['labels'], tc_['objects'], tc_['labels'])
        e_p = float(np.abs(np.sort(scores[i, :k]) - np.sort(tc_['probs'])).max()) if k else 0.0
        _report('frcnn/%s/%s/img%d' % (arch, impl, i), fmap_rel_engine=e_fm, fmap_rel_oracle32=o_fm,
                fmap_max_abs_oracle64=np.abs(tru['conv_feature_map']).max(), rpn_head_rel_engine=e_lg,
                rpn_head_rel_oracle32=o_lg, proposals_px_engine=e_pr, proposals_px_oracle32=o_pr,
                detections_px_engine=e_det, detections_px_oracle32=o_det, probs_abs_engine=e_p, detections=k)
        assert k > 0
        assert e_fm <= float_bound(o_fm, 5e-6), 'feature map: engine %.2e vs oracle32 %.2e' % (e_fm, o_fm)
        assert e_lg <= float_bound(o_lg, 1e-5), 'rpn heads: engine %.2e vs oracle32 %.2e' % (e_lg, o_lg)
        assert e_pr <= float_bound(o_pr, 1e-3), 'proposals: engine %.2e px vs oracle32 %.2e px' % (e_pr, o_pr)
        assert e_det <= float_bound(o_det, 1e-3), 'detections: engine %.2e px vs oracle32 %.2e px' % (e_det, o_det)
        assert e_p <= 2e-5
        assert (np.diff(scores[i, :k]) <= 0).all()
        roi_ref = ofr.roi_pool(props[i, :pcnt[i]], fmap[i][None], (h, w), 7, 7)['roi_pool']
        assert rel_err(pooled[i * 200:i * 200 + pcnt[i]], roi_ref) < 2e-6, 'roi_pool'
        head_ref = ofr.rcnn_head(roi_ref, wts, cfg['model']['rcnn'], arch)
        np.testing.assert_allclose(cls_prob[i, :pcnt[i]], head_ref['cls_prob'], atol=3e-5)
    eng.close()


def test_resnet_v2_taps_pipeline_and_graphs_bit_identical():
    """Under whole-tile conv scheduling the v2 forward gives the same bits with debug taps on or off, with the
    two-stream pipeline on or off, and from a CUDA-graph replay."""
    cfg = frcnn_cfg('resnet_v2_50')
    wts = synth.make_weights(cfg, seed=1)
    imgs = synth.make_images(2, 224, 320, seed=2)
    eng = Engine(cfg, max_batch=2, max_h=224, max_w=320)
    eng.load_weights(wts).finalize()
    eng.set_conv_streamk('off')
    eager = eng.predict_raw(imgs)                          # first sight of the shape: eager
    replays = []
    for _ in range(2):                                     # captured, then replayed
        for a, b in zip(eager, eng.predict_raw(imgs)):
            np.testing.assert_array_equal(a, b)
        replays.append(eng.last_graph_replays)
    assert replays[-1] > 0
    eng.set_pipeline(False)
    for a, b in zip(eager, eng.predict_raw(imgs)):
        np.testing.assert_array_equal(a, b)
    eng.set_debug_taps(True)
    for a, b in zip(eager, eng.predict_raw(imgs)):
        np.testing.assert_array_equal(a, b)
    assert eng.get_tensor('conv_feature_map').shape == (2, 14, 20, 1024)
    assert int(eager[3].sum()) > 0
    eng.close()
