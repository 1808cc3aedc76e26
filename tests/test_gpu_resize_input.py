"""Images at their original sizes: the bilinear resize fused into the input staging (`-m gpu`).

``lumi_predict_resize`` takes n source images of any sizes and one target size, and its staging kernels sample each
pixel of the target image from its source with the operation sequence of ``lumi_op_resize_bilinear``.  So it must give
the same bytes as resizing every image with ``lumi_op_resize_bilinear`` and feeding the float32 batch to
``lumi_predict_f32`` -- the path ``PredictorNetwork`` took before.  That path is rebuilt here, and its resized images
are also checked against the host restatement of the TF kernel (oracle/tf_ops.py), so an error in the sampling shared
by both paths still fails.
"""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import gpu_ops as G
import resnet_v2_oracle as V2
from luminoth_b200 import synth
from luminoth_b200.engine import Engine, LUMI_EINVAL
from luminoth_b200.predicting import PredictorNetwork, target_size
from oracle import tf_ops as T
from test_gpu_e2e import box_dev, float_bound, frcnn_cfg, rel_err, ssd_parity, _report
from test_ssd_config_host import ssd_cfg

# (h0, w0) of the sources of one call.  Upscale, three sizes that map to one target (160x224, 150x210, 200x280 to
# 224x320), the identity size, a 1-pixel-high source and downscales; odd counts, so the pipeline halves differ.
FRCNN_SOURCES = [(160, 224), (150, 210), (200, 280), (224, 320), (1, 300), (300, 420), (97, 131)]
FRCNN_TARGET = (224, 320)
SSD_SOURCES = [(375, 500), (300, 300), (1, 40), (120, 90), (480, 640)]
SSD_TARGET = (300, 300)


def sources(sizes, f32, seed):
    """uint8 images, or float32 images with non-integer pixels, of the given sizes."""
    rng = np.random.default_rng(seed)
    out = []
    for h0, w0 in sizes:
        im = rng.integers(0, 256, size=(h0, w0, 3), dtype=np.uint8)
        if f32:
            im = (im.astype(np.float32) + rng.random((h0, w0, 3), dtype=np.float32)).astype(np.float32)
        out.append(im)
    return out


def resized_batch(srcs, h, w):
    """The resize of the old path: lumi_op_resize_bilinear per image, checked bit-equal to the host TF restatement."""
    out = []
    for im in srcs:
        r = G.resize_bilinear(im, h, w)
        np.testing.assert_array_equal(r, T.resize_bilinear(im.astype(np.float32), h, w),
                                      err_msg='lumi_op_resize_bilinear vs host, %s' % (im.shape,))
        out.append(r)
    return np.stack(out)


def on_device(srcs):
    import torch
    return [torch.from_numpy(im).cuda() for im in srcs]


def make_engine(cfg, wts, n, h, w, impl):
    eng = Engine(cfg, max_batch=n, max_h=h, max_w=w)
    eng.load_weights(wts).finalize()
    eng.set_conv_impl(impl)
    return eng


def assert_same(a, b, what):
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y, err_msg=what)


CASES = [('frcnn', 'resnet_v1_50', 'tc'), ('frcnn', 'resnet_v1_50', 'simt'), ('frcnn', 'resnet_v2_50', 'tc'),
         ('ssd', 'vgg_16', 'tc'), ('ssd', 'vgg_16', 'simt')]


def _case(kind, arch):
    if kind == 'frcnn':
        cfg = frcnn_cfg(arch)
        return cfg, synth.make_weights(cfg, seed=1), FRCNN_SOURCES, FRCNN_TARGET, ['stem', 'conv_feature_map']
    cfg = ssd_cfg(300, 300)
    cfg['model']['proposals']['min_prob_threshold'] = 0.2
    return cfg, synth.make_weights(cfg, seed=5), SSD_SOURCES, SSD_TARGET, ['conv1_1', 'fmap_0']


@pytest.mark.parametrize('kind,arch,impl', CASES, ids=['-'.join(c) for c in CASES])
def test_fused_resize_matches_resize_then_predict(kind, arch, impl):
    """uint8 and float32 sources, on the host and on the device: detections and counts of predict_resize (eager, then
    captured) equal resize -> predict_raw(float32) on the production path, and so do the taps, byte for byte."""
    cfg, wts, sizes, (h, w), taps = _case(kind, arch)
    n = len(sizes)
    eng = make_engine(cfg, wts, n, h, w, impl)
    dbg = make_engine(cfg, wts, n, h, w, impl)
    dbg.set_debug_taps(True)
    for f32 in (False, True):
        srcs = sources(sizes, f32, seed=11 + f32)
        batch = resized_batch(srcs, h, w)
        want = eng.predict_raw(batch)
        assert int(want[3].sum()) > 0, 'the comparison must not be vacuous'
        for where, feed in (('host', srcs), ('device', on_device(srcs))):
            tag = '%s %s %s' % (kind, 'f32' if f32 else 'u8', where)
            for call in range(2):
                assert_same(want, eng.predict_resize(feed, h, w), '%s call %d' % (tag, call))
            want_dbg = dbg.predict_raw(batch)            # one stream: other stream-K split points than `want`
            want_taps = [dbg.get_tensor(t) for t in taps]
            assert_same(want_dbg, dbg.predict_resize(feed, h, w), tag + ' taps run')
            for name, ref in zip(taps, want_taps):
                np.testing.assert_array_equal(dbg.get_tensor(name), ref, err_msg='%s tap %s' % (tag, name))
    eng.close()
    dbg.close()


def test_graph_replay_reads_new_sources():
    """A, A again (captured), then B with the same target and other source sizes: a replay of A's graph that must read
    B's table.  Then C with larger sources: the source arena grows and the graphs are dropped.  B and C equal the
    eager results of a second engine with graphs off."""
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=1)
    h, w = FRCNN_TARGET
    a = sources([(160, 224), (150, 210), (200, 280)], False, seed=21)
    b = sources([(120, 168), (224, 320), (90, 100)], False, seed=22)
    c = sources([(480, 640), (300, 420), (600, 900)], False, seed=23)
    eng = make_engine(cfg, wts, 3, h, w, 'tc')
    ref = make_engine(cfg, wts, 3, h, w, 'tc')
    ref.set_graphs(False)
    replays = []
    outs = []
    for srcs in (a, a, b, c):
        outs.append(eng.predict_resize(srcs, h, w))
        replays.append(eng.last_graph_replays)
    assert replays[0] == 0 and replays[1] == 2 and replays[2] == 2 and replays[3] == 0, replays
    assert_same(outs[0], outs[1], 'A captured vs A eager')
    for name, srcs, got in (('B', b, outs[2]), ('C', c, outs[3])):
        want = ref.predict_resize(srcs, h, w)
        assert int(want[3].sum()) > 0
        assert_same(want, got, name)
        assert_same(want, ref.predict_raw(resized_batch(srcs, h, w)), name + ' vs resize -> predict_raw')
    eng.close()
    ref.close()


def test_fasterrcnn_fused_resize_against_oracle():
    """Two sources of different sizes resized to 224x320 in the engine: feature map, RPN heads, proposals and
    detections against the float64 oracle fed the host-resized image, with the rule of tests/test_gpu_float_input.py."""
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=1)
    h, w = FRCNN_TARGET
    srcs = sources([(150, 210), (300, 420)], False, seed=31)
    imgs = [T.resize_bilinear(im.astype(np.float32), h, w) for im in srcs]
    eng = make_engine(cfg, wts, 2, h, w, 'tc')
    eng.set_debug_taps(True)
    boxes, scores, labels, counts = eng.predict_resize(srcs, h, w)
    fmap = eng.get_tensor('conv_feature_map')
    heads = eng.get_tensor('rpn_heads')
    props = eng.get_tensor('proposals')
    pcnt = eng.get_tensor('proposal_counts').astype(int)
    A = 12
    for i in range(2):
        ref = V2.fasterrcnn_forward(imgs[i], wts, cfg)
        tru = V2.fasterrcnn_forward(imgs[i], wts, cfg, dtype=np.float64)
        e_fm = rel_err(fmap[i], tru['conv_feature_map'][0])
        o_fm = rel_err(ref['conv_feature_map'][0], tru['conv_feature_map'][0])
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
        _report('resize_input/frcnn/img%d' % i, fmap_rel_engine=e_fm, fmap_rel_oracle32=o_fm,
                rpn_head_rel_engine=e_lg, rpn_head_rel_oracle32=o_lg, proposals_px_engine=e_pr,
                proposals_px_oracle32=o_pr, detections_px_engine=e_det, detections_px_oracle32=o_det,
                probs_abs_engine=e_p, detections=k)
        assert k > 0
        assert e_fm <= float_bound(o_fm, 5e-6), 'feature map: engine %.2e vs oracle32 %.2e' % (e_fm, o_fm)
        assert e_lg <= float_bound(o_lg, 1e-5), 'rpn heads: engine %.2e vs oracle32 %.2e' % (e_lg, o_lg)
        assert e_pr <= float_bound(o_pr, 1e-3), 'proposals: engine %.2e px vs oracle32 %.2e px' % (e_pr, o_pr)
        assert e_det <= float_bound(o_det, 1e-3), 'detections: engine %.2e px vs oracle32 %.2e px' % (e_det, o_det)
        assert e_p <= 2e-5
    eng.close()


def test_ssd_fused_resize_against_oracle():
    """375x500 and 480x640 sources resized to 300x300 in the engine: SSD's taps and detections against the float64
    oracle fed the host-resized images."""
    cfg, wts, _, (h, w), _ = _case('ssd', 'vgg_16')
    srcs = sources([(375, 500), (480, 640)], False, seed=41)
    imgs = np.stack([T.resize_bilinear(im.astype(np.float32), h, w) for im in srcs])
    eng = make_engine(cfg, wts, 2, h, w, 'tc')
    eng.set_debug_taps(True)
    out = eng.predict_resize(srcs, h, w)
    ssd_parity('resize_input/ssd', eng, imgs, wts, cfg, out)
    eng.close()


def test_predictor_one_engine_call_per_chunk():
    """predict_batch_raw on a mixed list -- uint8 and float32 images, several source sizes per target size, an
    untouched bucket -- gives the bytes of the old path (resize each image, then predict_raw per chunk) and makes one
    engine call per chunk."""
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=7)
    rng = np.random.default_rng(51)
    u8 = lambda h0, w0: rng.integers(0, 256, size=(h0, w0, 3), dtype=np.uint8)
    images = [u8(300, 400), u8(480, 640), u8(600, 800).astype(np.float32) + np.float32(0.25), u8(375, 500),
              u8(500, 500), u8(600, 600), u8(600, 600), u8(600, 900), u8(600, 900), u8(600, 900)]
    net = PredictorNetwork(cfg, weights=wts, max_batch=2)
    net.engine.set_conv_streamk('off')
    calls = []
    eng = net.engine
    real_raw, real_resize = eng.predict_raw, eng.predict_resize
    eng.predict_raw = lambda *a: calls.append('raw') or real_raw(*a)
    eng.predict_resize = lambda *a: calls.append('resize') or real_resize(*a)
    got = net.predict_batch_raw(images)
    del eng.predict_raw, eng.predict_resize
    # the old path, chunk by chunk
    sizes = [target_size(im.shape, cfg) for im in images]
    buckets = {}
    for i, (nh, nw, _) in enumerate(sizes):
        buckets.setdefault((nh, nw), []).append(i)
    assert len(buckets) == 3
    want_calls = []
    for (nh, nw), idxs in buckets.items():
        untouched = all(images[i].dtype == np.uint8 and images[i].shape[:2] == (nh, nw) for i in idxs)
        for s in range(0, len(idxs), 2):
            chunk = idxs[s:s + 2]
            if untouched:
                want_calls.append('raw')
                boxes, scores, labels, counts = real_raw(np.stack([images[i] for i in chunk]))
            else:
                want_calls.append('resize')
                boxes, scores, labels, counts = real_raw(resized_batch([images[i] for i in chunk], nh, nw))
            for j, i in enumerate(chunk):
                k = int(counts[j])
                for x, y in zip(got[i][:3], (boxes[j, :k], labels[j, :k], scores[j, :k])):
                    np.testing.assert_array_equal(x, y, err_msg='image %d' % i)
                assert got[i][3] == sizes[i][2]
    assert calls == want_calls and 'raw' in calls, calls
    assert sum(len(g[0]) for g in got) > 0
    net.engine.close()


def test_bad_inputs_are_refused():
    """Sizes below 1, mixed dtypes or host and device images in one call, n > max_batch, an empty target and SSD at
    another size are ValueErrors; the engine serves the next valid call."""
    import torch
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=1)
    h, w = FRCNN_TARGET
    eng = make_engine(cfg, wts, 2, h, w, 'tc')
    ok = sources([(100, 120), (90, 80)], False, seed=61)
    want = eng.predict_resize(ok, h, w)
    with pytest.raises(ValueError, match='sizes must be >= 1'):
        eng.predict_resize([ok[0], np.zeros((0, 5, 3), np.uint8)], h, w)
    with pytest.raises(ValueError, match='share a dtype'):
        eng.predict_resize([ok[0], ok[1].astype(np.float32)], h, w)
    with pytest.raises(ValueError, match='all numpy arrays or all CUDA'):
        eng.predict_resize([ok[0], torch.from_numpy(ok[1]).cuda()], h, w)
    with pytest.raises(ValueError, match='max_batch'):
        eng.predict_resize(ok + ok[:1], h, w)
    with pytest.raises(ValueError, match='empty image'):
        eng.predict_resize(ok, 0, w)
    # straight through the C ABI: negative sizes, a null source
    k = eng.max_detections
    outs = [np.empty(s, dt) for s, dt in (((2, k, 4), np.float32), ((2, k), np.float32), ((2, k), np.int32),
                                          ((2,), np.int32))]
    optrs = [o.ctypes.data_as(ctypes.c_void_p) for o in outs]
    ptrs = (ctypes.c_void_p * 2)(ok[0].ctypes.data, ok[1].ctypes.data)
    for bad, msg in (([100, 120, -1, 80], 'sizes must be >= 1'), ([100, 120, 90, 0], 'sizes must be >= 1')):
        sz = np.array(bad, np.int32)
        rc = eng._lib.lumi_predict_resize(eng._h, ptrs, sz.ctypes.data_as(ctypes.c_void_p), 0, 0, 2, h, w, *optrs, 0)
        assert rc == LUMI_EINVAL and msg in eng._lib.lumi_last_error(eng._h).decode()
    nul = (ctypes.c_void_p * 2)(ok[0].ctypes.data, None)
    sz = np.array([100, 120, 90, 80], np.int32)
    rc = eng._lib.lumi_predict_resize(eng._h, nul, sz.ctypes.data_as(ctypes.c_void_p), 0, 0, 2, h, w, *optrs, 0)
    assert rc == LUMI_EINVAL and 'null source' in eng._lib.lumi_last_error(eng._h).decode()
    assert_same(want, eng.predict_resize(ok, h, w), 'after the refused calls')
    eng.close()
    scfg, swts, _, _, _ = _case('ssd', 'vgg_16')
    ssd = make_engine(scfg, swts, 1, 300, 300, 'tc')
    with pytest.raises(ValueError, match='fixed size'):
        ssd.predict_resize(ok[:1], 320, 320)
    ssd.close()


def test_noncontiguous_device_sources_written_on_torch_stream():
    """Device frames written on torch's current stream behind a long kernel, then passed as permuted CHW -> HWC views
    (non-contiguous, so predict_resize copies them on that stream): three calls over one reused buffer must each give
    the results of the same frames from the host."""
    import torch
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=1)
    h, w = FRCNN_TARGET
    sizes = [(160, 224), (150, 210), (200, 280)]
    eng = make_engine(cfg, wts, 3, h, w, 'tc')
    bufs = [torch.zeros((3, h0, w0), dtype=torch.uint8, device='cuda') for h0, w0 in sizes]
    for call in range(3):
        frames = sources(sizes, False, seed=71 + call)
        want = eng.predict_resize(frames, h, w)
        assert int(want[3].sum()) > 0
        chw = [torch.from_numpy(np.ascontiguousarray(f.transpose(2, 0, 1))).pin_memory().cuda() for f in frames]
        torch.cuda.synchronize()
        torch.cuda._sleep(20_000_000)                  # the writes below land well after this call starts
        for b, c in zip(bufs, chw):
            b.copy_(c, non_blocking=True)
        views = [b.permute(1, 2, 0) for b in bufs]
        assert not any(v.is_contiguous() for v in views)
        assert_same(want, eng.predict_resize(views, h, w), 'call %d' % call)
    eng.close()


def test_device_outputs_back_to_back():
    """Three lumi_predict_resize calls with device outputs and host sources, queued without a synchronisation behind a
    long kernel on the engine's stream: each call packs its sources into the pinned buffer while the uploads of the
    calls before it are still queued.  Each must equal the host-output result of its own sources."""
    import torch
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=1)
    h, w = FRCNN_TARGET
    eng = make_engine(cfg, wts, 3, h, w, 'tc')
    # the largest sources first: neither the device arena nor the pinned buffer grows later (a growth synchronises)
    calls = [sources([(300, 420), (280, 400), (260, 380)], False, seed=81),
             sources([(160, 224), (150, 210), (200, 280)], False, seed=82),
             sources([(120, 168), (224, 320), (90, 100)], False, seed=83)]
    want = [eng.predict_resize(srcs, h, w) for srcs in calls]       # also warms up: the calls below replay graphs
    assert all(int(wt[3].sum()) > 0 for wt in want)
    k = eng.max_detections
    outs = []
    with torch.cuda.stream(torch.cuda.ExternalStream(eng.stream)):
        torch.cuda._sleep(50_000_000)
    for srcs in calls:
        o = [torch.empty(s, dtype=dt, device='cuda') for s, dt in (((3, k, 4), torch.float32), ((3, k), torch.float32),
                                                                   ((3, k), torch.int32), ((3,), torch.int32))]
        ptrs = (ctypes.c_void_p * 3)(*[s.ctypes.data for s in srcs])
        sz = np.array([s.shape[:2] for s in srcs], np.int32)
        rc = eng._lib.lumi_predict_resize(eng._h, ptrs, sz.ctypes.data_as(ctypes.c_void_p), 0, 0, 3, h, w,
                                          *[ctypes.c_void_p(t.data_ptr()) for t in o], 1)
        assert rc == 0, eng._lib.lumi_last_error(eng._h).decode()
        outs.append(o)
    eng.synchronize()
    assert eng.last_graph_replays == 2
    for i, (wt, o) in enumerate(zip(want, outs)):
        assert_same(wt, [t.cpu().numpy() for t in o], 'call %d' % i)
    eng.close()
