"""Faster R-CNN at model.base_network.output_stride 4, 8, 32 and null on the GPU (`-m gpu`): end-to-end parity with
the CPU oracle, bit-identity across the engine's execution modes, the dilated block3 convs on the stand-alone op, and
the RPN's top-k cut ahead of the sort against the oracle's rpn_proposal."""
import copy

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import gpu_ops as G
import resnet_v2_oracle as V2
from luminoth_b200 import synth
from luminoth_b200.engine import Engine
from oracle import fasterrcnn as ofr
from oracle import tf_ops as T
from oracle.anchors import fasterrcnn_anchors
from test_gpu_conv_epilogue import _conv
from test_gpu_e2e import box_dev, float_bound, frcnn_cfg, rel_err, _report
from test_gpu_kernels import _bn_fold, _ref_conv, assert_close


def _cfg(arch, output_stride, anchor_stride):
    extra = ['model.base_network.output_stride=%s' % output_stride]
    if anchor_stride is not None:
        extra.append('model.anchors.stride=%d' % anchor_stride)
    return frcnn_cfg(arch, extra)


def _oracle_cfg(cfg):
    """The oracle takes an integer output_stride: null builds the network of 32 (no atrous convolution)."""
    c = copy.deepcopy(cfg.to_dict())
    if c['model']['base_network']['output_stride'] is None:
        c['model']['base_network']['output_stride'] = 32
    return c


# (arch, output_stride, conv impl, model.anchors.stride or None for its default 16, h, w, pre_nms_top_n or None for
# its default 12 000).  The last case keeps 1000 of its 13 440 anchors: the RPN runs the top-k cut ahead of its sort.
E2E = [('resnet_v1_50', 8, 'tc', 8, 224, 320, None), ('resnet_v1_50', 8, 'simt', 8, 224, 320, None),
       ('resnet_v1_101', 8, 'tc', 8, 224, 320, None), ('resnet_v2_50', 8, 'tc', None, 224, 320, None),
       ('resnet_v1_50', 4, 'tc', 4, 160, 224, None), ('resnet_v1_50', 32, 'tc', 32, 225, 327, None),
       ('resnet_v1_50', 'None', 'tc', 32, 224, 320, None), ('resnet_v1_50', 8, 'tc', 8, 224, 320, 1000)]


@pytest.mark.parametrize('arch,os_,impl,astride,h,w,pre', E2E,
                         ids=['-'.join(map(str, c[:4])) + ('-pre%d' % c[6] if c[6] else '') for c in E2E])
def test_fasterrcnn_output_stride_stages_and_detections(arch, os_, impl, astride, h, w, pre):
    cfg = _cfg(arch, os_, astride)
    if pre:
        cfg['model']['rpn']['proposals']['pre_nms_top_n'] = pre
    ocfg = _oracle_cfg(cfg)
    stride = ocfg['model']['base_network']['output_stride']
    wts = synth.make_weights(cfg, seed=1)
    imgs = synth.make_images(2, h, w, seed=2)
    eng = Engine(cfg, max_batch=2, max_h=h, max_w=w)
    eng.load_weights(wts).finalize()
    eng.set_conv_impl(impl)
    eng.set_debug_taps(True)
    boxes, scores, labels, counts = eng.predict_raw(imgs)
    fmap = eng.get_tensor('conv_feature_map')
    fh, fw = -(-h // stride), -(-w // stride)
    assert fmap.shape == (2, fh, fw, 1024)
    A = 12
    anchors = eng.get_tensor('all_anchors').reshape(-1, 4)
    assert anchors.shape == (fh * fw * A, 4)
    if pre:
        assert anchors.shape[0] >= GATE * pre
    heads = eng.get_tensor('rpn_heads')
    props = eng.get_tensor('proposals')
    pcnt = eng.get_tensor('proposal_counts').astype(int)
    cls_prob = eng.get_tensor('rcnn_cls_prob')
    pooled = eng.get_tensor('roi_pool')
    for i in range(2):
        ref = V2.fasterrcnn_forward(imgs[i], wts, ocfg)
        tru = V2.fasterrcnn_forward(imgs[i], wts, ocfg, dtype=np.float64)
        np.testing.assert_array_equal(anchors, tru['all_anchors'])
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
        _report('frcnn/%s/os%s/%s/img%d' % (arch, os_, impl, i), fmap_rel_engine=e_fm, fmap_rel_oracle32=o_fm,
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
        roi_ref = ofr.roi_pool(props[i, :pcnt[i]], fmap[i][None], (h, w), 7, 7)['roi_pool']
        assert rel_err(pooled[i * 200:i * 200 + pcnt[i]], roi_ref) < 2e-6, 'roi_pool'
        head_ref = ofr.rcnn_head(roi_ref, wts, cfg['model']['rcnn'], arch)
        np.testing.assert_allclose(cls_prob[i, :pcnt[i]], head_ref['cls_prob'], atol=3e-5)
    eng.close()


def test_output_stride8_taps_pipeline_and_graphs_bit_identical():
    """At output_stride 8, under whole-tile conv scheduling, the forward gives the same bits with debug taps on or
    off, with the two-stream pipeline on or off, and from a CUDA-graph replay."""
    cfg = _cfg('resnet_v1_50', 8, 8)
    wts = synth.make_weights(cfg, seed=1)
    imgs = synth.make_images(2, 224, 320, seed=2)
    eng = Engine(cfg, max_batch=2, max_h=224, max_w=320)
    eng.load_weights(wts).finalize()
    eng.set_conv_streamk('off')
    eager = eng.predict_raw(imgs)
    replays = []
    for _ in range(2):
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
    assert eng.get_tensor('conv_feature_map').shape == (2, 28, 40, 1024)
    assert int(eager[3].sum()) > 0
    eng.close()


def test_output_stride8_predict_batch_over_two_sizes():
    """predict_batch over two image sizes (one anchor grid each, 115 200 and 72 000 anchors after the resize to the
    600-pixel short side) equals the single-image calls."""
    from luminoth_b200.predicting import PredictorNetwork
    cfg = _cfg('resnet_v1_50', 8, 8)
    wts = synth.make_weights(cfg, seed=7)
    a = synth.make_images(2, 600, 1024, seed=41)
    b = synth.make_images(2, 600, 640, seed=42)
    order = [a[0], b[0], a[1], b[1]]
    net = PredictorNetwork(cfg, weights=wts, max_batch=2)
    net.engine.set_conv_streamk('off')
    got = net.predict_batch(order)
    single = [net.predict_image(im) for im in order]
    assert got == single and all(len(g) > 0 for g in got)
    net.engine.close()


# block3's dilated 3x3 conv2 (256 -> 256, SAME, split output) at output_stride 8 (rate 2) and 4 (rate 4), on the
# SIMT kernel and the tensor-core impl codes of lumi_op_conv2d (see test_gpu_resnet_v2.IMPLS)
DILATED = [('b3_conv2_rate2', 2, 38, 64, 256, 256, 3, 1, 2, 'SAME', False, 1),
           ('b3_conv2_rate4', 1, 75, 128, 256, 256, 3, 1, 4, 'SAME', False, 1),
           ('b3_conv2_rate2_slim', 1, 29, 41, 256, 256, 3, 1, 2, 'SLIM', False, 1)]


@pytest.mark.parametrize('impl', [0, 3, 4, 5, 6, 7, 12])
@pytest.mark.parametrize('case', DILATED, ids=[c[0] for c in DILATED])
def test_dilated_block3_conv_matches_oracle(case, impl):
    import zlib
    name, n, h, w, cin, cout, k, stride, rate, padding, use_res, act = case
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = (rng.standard_normal((n, h, w, cin)) * 2).astype(np.float32)
    wt = (rng.standard_normal((k, k, cin, cout)) * np.sqrt(2.0 / (k * k * cin))).astype(np.float32)
    scale, bias = _bn_fold(rng, cout)
    ref = _ref_conv(x, wt, stride, rate, padding, scale, bias, None, act)
    assert ref.shape == (n, h, w, cout)
    assert_close(_conv(x, wt, stride, rate, padding, scale, bias, None, act, impl), ref, 2e-5, '%s/%d' % (name, impl))


def _rpn_case(fh, fw, seed, levels=None, min_prob=0.0, pre=12000):
    rng = np.random.default_rng(seed)
    anchors = fasterrcnn_anchors(fh, fw, 256, [0.5, 1, 2], [0.25, 0.5, 1, 2], 8).astype(np.float32)
    na = anchors.shape[0]
    prob = T.softmax(rng.standard_normal((na, 2)).astype(np.float32))
    if levels:                      # a few hundred distinct scores: thousands of ties straddle the k-th key
        q = np.floor(rng.uniform(0, 1, na) * levels) / levels
        prob = np.stack([1 - q, q], 1).astype(np.float32)
    pred = (rng.standard_normal((na, 4)) * 0.2).astype(np.float32)
    pred[:, 2:] = 0                 # exp(0) == 1 on both sides: the decode is bit-reproducible
    # NMS that never suppresses (IoU > 1 never holds) and room for every candidate: the output is the whole sorted
    # top-k, so the comparison sees the k-th key and which of its ties were kept
    cfg = {'pre_nms_top_n': pre, 'post_nms_top_n': pre, 'nms_threshold': 1.0, 'min_prob_threshold': min_prob,
           'clip_after_nms': False, 'filter_outside_anchors': False, 'apply_nms': True}
    return prob, pred, anchors, cfg


GATE = 4     # postproc.cu RPN_CUT_RATIO: the cut runs from GATE anchors per kept candidate on
RPN_CASES = {
    'os8_115200': dict(fh=75, fw=128, seed=21),
    'os4_460800': dict(fh=150, fw=256, seed=22),
    'ties_200_levels': dict(fh=150, fw=256, seed=23, levels=200),
    'few_valid': dict(fh=75, fw=128, seed=24, min_prob=0.93),
    # 14 400 anchors; k <= 4096 also runs the eight-warp sort of the compacted pairs
    'one_below_gate': dict(fh=30, fw=40, seed=25, pre=14400 // GATE + 1),    # na < GATE pre: the full sort
    'at_gate': dict(fh=30, fw=40, seed=26, pre=14400 // GATE),               # na == GATE pre: the cut
}


@pytest.mark.parametrize('name', sorted(RPN_CASES))
def test_rpn_proposals_with_topk_cut_match_oracle(name):
    """lumi_op_rpn_proposals at output_stride 8 and 4 anchor counts: every one of the top pre_nms_top_n proposals and
    scores, in order, identical to the oracle's."""
    prob, pred, anchors, cfg = _rpn_case(**RPN_CASES[name])
    k = cfg['pre_nms_top_n']
    valid = int((prob[:, 1] >= cfg['min_prob_threshold']).sum())
    if name == 'few_valid':
        assert 0 < valid < k
    if name == 'ties_200_levels':
        s = np.sort(prob[:, 1])[::-1]
        ties = s == s[k - 1]
        assert ties.sum() > 2000 and ties[:k].sum() > 400 and ties[k:].sum() > 1000   # ties on both sides of k
    ref = ofr.rpn_proposal(prob, pred, anchors, (600, 1024), cfg)
    p, s = G.rpn_proposals(prob, pred, anchors, (600, 1024), cfg)
    assert ref['proposals'].shape == (min(k, valid), 4)             # nothing suppressed: the whole top-k is compared
    assert p.shape == ref['proposals'].shape
    np.testing.assert_array_equal(s, ref['scores'])
    np.testing.assert_array_equal(p, ref['proposals'])
