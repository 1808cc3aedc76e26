"""Faster R-CNN from model.base_network.endpoints other than block3 on the GPU (`-m gpu`): end-to-end parity with the
CPU oracle, bit-identity across the engine's execution modes, and predict_batch over two image sizes at the stem
endpoint, whose RPN sorts 1.84 M anchors per 600x1024 image."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import endpoint_oracle as EO
from luminoth_b200 import synth
from luminoth_b200.engine import Engine
from oracle import fasterrcnn as ofr
from test_gpu_e2e import box_dev, float_bound, frcnn_cfg, rel_err, _report


def _cfg(arch, endpoint, *extra):
    return frcnn_cfg(arch, ['model.base_network.endpoint=' + endpoint] + list(extra))


# (arch, endpoint, extra overrides, conv impl, h, w, feature stride, depth)
E2E = [('resnet_v1_50', 'block4', (), 'tc', 224, 320, 16, 2048),
       ('resnet_v1_50', 'block4', (), 'simt', 224, 320, 16, 2048),
       ('resnet_v1_50', 'block4', ('model.base_network.output_stride=32',), 'tc', 225, 327, 32, 2048),
       ('resnet_v1_50', 'block2', (), 'tc', 224, 320, 16, 512),
       ('resnet_v1_50', 'block1', (), 'tc', 160, 224, 8, 256),
       ('resnet_v1_50', 'conv1', (), 'tc', 96, 128, 2, 64),
       ('resnet_v1_50', 'block3/unit_4/bottleneck_v1/conv3', (), 'tc', 224, 320, 16, 1024),
       ('resnet_v1_50', 'block2/unit_4/bottleneck_v1/conv1', (), 'tc', 160, 224, 8, 128),
       ('resnet_v1_50', 'block2/unit_1/bottleneck_v1/shortcut', (), 'tc', 160, 224, 8, 512),
       ('resnet_v1_101', 'block3/unit_12/bottleneck_v1', (), 'tc', 224, 320, 16, 1024),
       ('resnet_v1_101', 'block4', ('model.base_network.use_tail=false',), 'tc', 224, 320, 16, 2048),
       # behind v2 block4's raw sums the synthetic classifier saturates (probabilities 0.9998-0.99997, fp32 steps of
       # 6e-8), so equal fp32 scores decide which overlapping boxes the class NMS keeps: this case checks the trunk
       # and the RPN, the other block4 cases the ROI pool and head at 2048 channels
       ('resnet_v2_50', 'block4', ('model.network.with_rcnn=false',), 'tc', 224, 320, 16, 2048),
       ('resnet_v2_50', 'block2/unit_2/bottleneck_v2/conv3', (), 'tc', 160, 224, 8, 512),
       ('resnet_v2_50', 'conv1', (), 'tc', 96, 128, 2, 64),
       ('resnet_v1_50', 'block2', ('model.network.with_rcnn=false',), 'tc', 224, 320, 16, 512)]


@pytest.mark.parametrize('arch,endpoint,extra,impl,h,w,stride,depth', E2E,
                         ids=['-'.join((c[0], c[1].replace('/', '.')) + tuple(x.split('=')[-1] for x in c[2]) + (c[3],))
                              for c in E2E])
def test_fasterrcnn_endpoint_stages_and_detections(arch, endpoint, extra, impl, h, w, stride, depth):
    cfg = _cfg(arch, endpoint, *extra)
    ocfg = cfg.to_dict()
    m = ocfg['model']
    with_rcnn = m['network']['with_rcnn']
    use_tail = m['base_network']['use_tail']
    post = m['rpn']['proposals']['post_nms_top_n']
    wts = synth.make_weights(cfg, seed=1)
    imgs = synth.make_images(2, h, w, seed=2)
    eng = Engine(cfg, max_batch=2, max_h=h, max_w=w)
    eng.load_weights(wts).finalize()
    eng.set_conv_impl(impl)
    eng.set_debug_taps(True)
    boxes, scores, labels, counts = eng.predict_raw(imgs)
    fmap = eng.get_tensor('conv_feature_map')
    fh, fw = -(-h // stride), -(-w // stride)
    assert fmap.shape == (2, fh, fw, depth)
    A = 12
    anchors = eng.get_tensor('all_anchors').reshape(-1, 4)
    assert anchors.shape == (fh * fw * A, 4)
    heads = eng.get_tensor('rpn_heads')
    props = eng.get_tensor('proposals')
    pcnt = eng.get_tensor('proposal_counts').astype(int)
    if with_rcnn:
        cls_prob = eng.get_tensor('rcnn_cls_prob')
        pooled = eng.get_tensor('roi_pool')
    total = 0
    for i in range(2):
        ref = EO.fasterrcnn_forward(imgs[i], wts, ocfg)
        tru = EO.fasterrcnn_forward(imgs[i], wts, ocfg, dtype=np.float64)
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
        assert e_fm <= float_bound(o_fm, 5e-6), 'feature map: engine %.2e vs oracle32 %.2e' % (e_fm, o_fm)
        assert e_lg <= float_bound(o_lg, 1e-5), 'rpn heads: engine %.2e vs oracle32 %.2e' % (e_lg, o_lg)
        assert e_pr <= float_bound(o_pr, 1e-3), 'proposals: engine %.2e px vs oracle32 %.2e px' % (e_pr, o_pr)
        k = int(counts[i])
        total += k
        key = 'frcnn/%s/%s/%s/%s/img%d' % (arch, endpoint, '.'.join(extra), impl, i)
        if not with_rcnn:      # the detections are the proposals
            assert k == pcnt[i]
            np.testing.assert_array_equal(boxes[i, :k], props[i, :k])
            _report(key, fmap_rel_engine=e_fm, fmap_rel_oracle32=o_fm, rpn_head_rel_engine=e_lg,
                    rpn_head_rel_oracle32=o_lg, proposals_px_engine=e_pr, proposals_px_oracle32=o_pr, detections=k)
            continue
        tc_, rc_ = tru['classification_prediction'], ref['classification_prediction']
        e_det = box_dev(boxes[i, :k], labels[i, :k], tc_['objects'], tc_['labels'])
        o_det = box_dev(rc_['objects'], rc_['labels'], tc_['objects'], tc_['labels'])
        e_p = float(np.abs(np.sort(scores[i, :k]) - np.sort(tc_['probs'])).max()) if k else 0.0
        _report(key, fmap_rel_engine=e_fm, fmap_rel_oracle32=o_fm, rpn_head_rel_engine=e_lg, rpn_head_rel_oracle32=o_lg,
                proposals_px_engine=e_pr, proposals_px_oracle32=o_pr, detections_px_engine=e_det,
                detections_px_oracle32=o_det, probs_abs_engine=e_p, detections=k)
        # the SIMT cross-check kernel sums each output in one fp32 FFMA chain: across block4's K = 4608 conv2 and the
        # 2048-wide RCNN head its rounding noise is about twice the fp32 oracle's (3.4e-3 against 1.5e-3 px on
        # image 1), where the tensor-core path stays below the oracle's
        det_noise = (2.0 if impl == 'simt' else 1.0) * o_det
        assert e_det <= float_bound(det_noise, 1e-3), 'detections: engine %.2e px vs oracle32 %.2e px' % (e_det, o_det)
        assert e_p <= 2e-5
        assert (np.diff(scores[i, :k]) <= 0).all()
        roi_ref = ofr.roi_pool(props[i, :pcnt[i]], fmap[i][None], (h, w), 7, 7)['roi_pool']
        assert roi_ref.shape[-1] == depth
        assert rel_err(pooled[i * post:i * post + pcnt[i]], roi_ref) < 2e-6, 'roi_pool'
        head_ref = ofr.rcnn_head(roi_ref, wts, m['rcnn'], arch, use_tail=use_tail)
        np.testing.assert_allclose(cls_prob[i, :pcnt[i]], head_ref['cls_prob'], atol=3e-5)
    assert total > 0
    if endpoint == 'block3/unit_4/bottleneck_v1/conv3':
        assert fmap.min() < 0              # collected before the residual add and its relu
    eng.close()


def test_block4_taps_pipeline_and_graphs_bit_identical():
    """With the block4 endpoint, under whole-tile conv scheduling, the forward gives the same bits with debug taps on
    or off, with the two-stream pipeline on or off, and from a CUDA-graph replay."""
    cfg = _cfg('resnet_v1_50', 'block4')
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
    assert eng.get_tensor('conv_feature_map').shape == (2, 14, 20, 2048)
    assert int(eager[3].sum()) > 0
    eng.close()


def test_stem_endpoint_predict_batch_over_two_sizes():
    """predict_batch over two image sizes at the conv1 endpoint (stride 2: 1 843 200 and 1 152 000 anchors after the
    resize to the 600-pixel short side, through the RPN's top-k cut) equals the single-image calls."""
    from luminoth_b200.predicting import PredictorNetwork
    cfg = _cfg('resnet_v1_50', 'conv1')
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
