"""The float32 entry point (``lumi_predict_f32``) at stage precision (`-m gpu`).

``PredictorNetwork`` sends every image the preprocessing resizes through the float32 entry point, as the reference
feeds the resized float image (predicting.py:110-112): its staging kernels keep the low part of every pixel in the
second fp16 plane, which integer pixels never use.  Here the float path is held to the float64 oracle with the rule of
tests/test_gpu_e2e.py, and a uint8 image and the same image as float32 must give the same bytes through every entry
point, eager, graph capture and graph replay alike.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import gpu_ops as G
import resnet_v2_oracle as V2
from luminoth_b200 import default_config, synth
from luminoth_b200.engine import Engine
from oracle import tf_ops as T
from test_gpu_e2e import box_dev, float_bound, frcnn_cfg, rel_err, _report


def resized_float_images(n, h0, w0, h, w, seed):
    """n uint8 images of h0 x w0 resized to h x w on the GPU (the product path's resize): non-integer float pixels."""
    imgs = synth.make_images(n, h0, w0, seed=seed)
    out = np.stack([G.resize_bilinear(im, h, w) for im in imgs])
    for im, o in zip(imgs, out):
        np.testing.assert_array_equal(o, T.resize_bilinear(im.astype(np.float32), h, w))
    assert out.dtype == np.float32 and (out != np.round(out)).mean() > 0.5      # most pixels use the low plane
    return out


@pytest.mark.parametrize('arch,impl', [('resnet_v1_50', 'tc'), ('resnet_v1_50', 'simt'), ('resnet_v2_50', 'tc')])
def test_fasterrcnn_float_pixels_stages_and_detections(arch, impl):
    """160x224 images resized to 224x320 (float pixels) through predict_raw with debug taps: feature map, RPN heads,
    proposals and detections against the oracle fed the same float image."""
    cfg = frcnn_cfg(arch)
    wts = synth.make_weights(cfg, seed=1)
    h, w = 224, 320
    imgs = resized_float_images(2, 160, 224, h, w, seed=3)
    eng = Engine(cfg, max_batch=2, max_h=h, max_w=w)
    eng.load_weights(wts).finalize()
    eng.set_conv_impl(impl)
    eng.set_debug_taps(True)
    boxes, scores, labels, counts = eng.predict_raw(imgs)
    fmap = eng.get_tensor('conv_feature_map')
    heads = eng.get_tensor('rpn_heads')
    props = eng.get_tensor('proposals')
    pcnt = eng.get_tensor('proposal_counts').astype(int)
    A = 12
    for i in range(2):
        ref = V2.fasterrcnn_forward(imgs[i], wts, cfg)                          # fp32 CPU oracle
        tru = V2.fasterrcnn_forward(imgs[i], wts, cfg, dtype=np.float64)        # exact-arithmetic yardstick
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
        _report('float_input/frcnn/%s/%s/img%d' % (arch, impl, i), fmap_rel_engine=e_fm, fmap_rel_oracle32=o_fm,
                rpn_head_rel_engine=e_lg, rpn_head_rel_oracle32=o_lg, proposals_px_engine=e_pr,
                proposals_px_oracle32=o_pr, detections_px_engine=e_det, detections_px_oracle32=o_det,
                probs_abs_engine=e_p, detections=k)
        assert k > 0
        assert e_fm <= float_bound(o_fm, 5e-6), 'feature map: engine %.2e vs oracle32 %.2e' % (e_fm, o_fm)
        assert e_lg <= float_bound(o_lg, 1e-5), 'rpn heads: engine %.2e vs oracle32 %.2e' % (e_lg, o_lg)
        assert e_pr <= float_bound(o_pr, 1e-3), 'proposals: engine %.2e px vs oracle32 %.2e px' % (e_pr, o_pr)
        assert e_det <= float_bound(o_det, 1e-3), 'detections: engine %.2e px vs oracle32 %.2e px' % (e_det, o_det)
        assert e_p <= 2e-5
        assert (np.diff(scores[i, :k]) <= 0).all()
    eng.close()


def _model(kind):
    if kind == 'frcnn':
        cfg = frcnn_cfg('resnet_v1_50')
        return cfg, synth.make_weights(cfg, seed=7), synth.make_images(2, 160, 224, seed=8)
    cfg = default_config('ssd', ['model.proposals.min_prob_threshold=0.2'])
    return cfg, synth.make_weights(cfg, seed=5), synth.make_images(2, 300, 300, seed=6)


@pytest.mark.parametrize('impl', ['tc', 'simt'])
@pytest.mark.parametrize('kind', ['frcnn', 'ssd'])
def test_uint8_and_float32_pixels_give_identical_bytes(kind, impl):
    """A uint8 image converted to float32 holds the same values, so both entry points must give the same bits.  On one
    handle, on the production path (graphs on, taps off, default stream-K): float32 numpy x 3, uint8 x 3, float32 CUDA
    tensor x 2, uint8 x 2 -- each entry point runs eager, then is captured, then replayed.  Float first, so the uint8
    calls reuse the larger staging buffer and only the pixel size in the graph key keeps a float graph from being
    replayed on uint8 bytes.  A second handle runs uint8 x 3 then float32 x 3: the staging buffer grows and the graphs
    captured so far are dropped.  This is the mix PredictorNetwork gives one handle when it serves both untouched
    uint8 images and resized ones."""
    import torch
    cfg, wts, u8 = _model(kind)
    f32 = u8.astype(np.float32)
    f32_dev = torch.from_numpy(f32).cuda()
    h, w = u8.shape[1:3]
    feeds = {'f32': f32, 'u8': u8, 'f32_dev': f32_dev}

    def handle():
        eng = Engine(cfg, max_batch=2, max_h=h, max_w=w)
        eng.load_weights(wts).finalize()
        eng.set_conv_impl(impl)
        return eng

    want = None
    for order in (['f32'] * 3 + ['u8'] * 3 + ['f32_dev'] * 2 + ['u8'] * 2, ['u8'] * 3 + ['f32'] * 3):
        eng = handle()
        replays = []
        for feed in order:
            got = eng.predict_raw(feeds[feed])
            replays.append(eng.last_graph_replays)
            if want is None:
                want = got
                assert int(want[3].sum()) > 0, 'the comparison must not be vacuous'
            for a, b in zip(want, got):
                np.testing.assert_array_equal(a, b, err_msg='%s call %d (%s)' % (kind, len(replays), feed))
        # eager at the first call of each pixel type, then capture and replay of that type's own graph
        assert replays[0] == 0 and replays[2] > 0 and replays[3] == 0 and replays[5] > 0, replays
        eng.close()
