"""End-to-end parity through the C ABI engine vs the CPU oracle (`-m gpu`).

Stage taps are compared first (feature map, RPN head, proposals, ROI pool,
class probabilities), then the final detections: identical class assignment
after NMS and boxes within 1e-3 px (north star).  Same synthetic weights and
images on both sides (SURVEY.md section 8d).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from luminoth_b200 import default_config, synth
from luminoth_b200.engine import Engine
from luminoth_b200.predicting import PredictorNetwork
from oracle import fasterrcnn as ofr
from oracle import ssd as ossd
from oracle import predict as opredict


def rel_err(a, b):
    return float(np.abs(a.astype(np.float64) - b).max() / max(1e-12, np.abs(b).max()))


def box_dev(boxes, labels, ref_boxes, ref_labels):
    """Max |coordinate difference| after the best one-to-one matching of rows with equal labels
    (ordering may legitimately differ between two fp32 implementations when scores are near-equal)."""
    from scipy.optimize import linear_sum_assignment
    assert len(boxes) == len(ref_boxes), 'row count %d vs %d' % (len(boxes), len(ref_boxes))
    if len(boxes) == 0:
        return 0.0
    assert sorted(np.asarray(labels).tolist()) == sorted(np.asarray(ref_labels).tolist()), 'class assignment differs'
    cost = np.abs(boxes[:, None, :].astype(np.float64) - ref_boxes[None, :, :]).max(axis=2)
    cost = cost + 1e6 * (np.asarray(labels)[:, None] != np.asarray(ref_labels)[None, :])
    r, c = linear_sum_assignment(cost)
    return float(cost[r, c].max())


REPORT = {}


def _report(key, **vals):
    import json, os
    REPORT[key] = {k: float(v) for k, v in vals.items()}
    os.makedirs('gpurun_out', exist_ok=True)
    with open('gpurun_out/parity_report.json', 'w') as f:
        json.dump(REPORT, f, indent=1, sort_keys=True)


def frcnn_cfg(arch, extra=()):
    return default_config('fasterrcnn', ['model.base_network.architecture=' + arch, 'model.network.num_classes=20',
                                         'model.rpn.proposals.post_nms_top_n=200',
                                         'model.rcnn.proposals.min_prob_threshold=0.05'] + list(extra))


# Acceptance bound for float outputs.  The north star asks for 1e-3 px on box coordinates vs the reference's fp32
# CPU path.  Two fp32 evaluations of this 50-100 layer network differ by their accumulated rounding noise; the fp32
# oracle's own distance to the float64 evaluation of the same algorithm ("the noise") is 5e-4..1.2e-3 px on a 224x320
# image and ~1e-2 px in the NMS-stress configuration (it grows with box size).  The engine's conv accumulates in
# short chunks folded into an fp32 running sum (DESIGN.md section 3) to stay within that noise.  The engine
# is held to max(floor, 1.5 x noise): the floor is the north star's own number, the 1.5 a chosen margin for "one more
# fp32-class implementation" of the same arithmetic.
NOISE_FACTOR = 1.5


def float_bound(oracle32_dev, floor):
    return max(floor, NOISE_FACTOR * oracle32_dev)


@pytest.mark.parametrize('arch,impl', [('resnet_v1_50', 'simt'), ('resnet_v1_50', 'tc'), ('resnet_v1_101', 'tc')])
def test_fasterrcnn_stages_and_detections(arch, impl):
    cfg = frcnn_cfg(arch)
    wts = synth.make_weights(cfg, seed=1)
    h, w = 224, 320
    imgs = synth.make_images(2, h, w, seed=2)
    eng = Engine(cfg, max_batch=2, max_h=h, max_w=w)
    eng.load_weights(wts).finalize()
    eng.set_conv_impl(impl)
    # pipelining / fusion / taps must not change the result -- bit for bit under the whole-tile conv schedule;
    # under the default stream-K schedule the split points depend on the (half-)batch, so only to fp32 noise
    eng.set_conv_streamk('off')
    fused = eng.predict_raw(imgs)                      # production path (ROI crop+pool+mean fused for R50)
    eng.set_debug_taps(True)                           # also materialise the roi_pool tap
    for a, b in zip(fused, eng.predict_raw(imgs)):
        np.testing.assert_array_equal(a, b)
    eng.set_debug_taps(False)
    eng.set_conv_streamk('auto')
    fused = eng.predict_raw(imgs)
    eng.set_debug_taps(True)
    boxes, scores, labels, counts = eng.predict_raw(imgs)
    np.testing.assert_array_equal(fused[3], counts)
    for i in range(2):
        k = int(counts[i])
        assert box_dev(fused[0][i, :k], fused[2][i, :k], boxes[i, :k], labels[i, :k]) <= 2e-3
    fmap = eng.get_tensor('conv_feature_map')
    heads = eng.get_tensor('rpn_heads')
    props = eng.get_tensor('proposals')
    pcnt = eng.get_tensor('proposal_counts').astype(int)
    anchors = eng.get_tensor('all_anchors')
    pooled = eng.get_tensor('roi_pool')
    cls_prob = eng.get_tensor('rcnn_cls_prob')
    for i in range(2):
        img = imgs[i]
        ref = ofr.forward(img, wts, cfg)                            # fp32 CPU oracle
        tru = ofr.forward(img, wts, cfg, dtype=np.float64)          # exact-arithmetic yardstick
        np.testing.assert_array_equal(anchors, ref['all_anchors'].astype(np.float32))
        e_fm, o_fm = rel_err(fmap[i], tru['conv_feature_map'][0]), rel_err(ref['conv_feature_map'][0], tru['conv_feature_map'][0])
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
        _report('frcnn/%s/%s/img%d' % (arch, impl, i), fmap_rel_engine=e_fm, fmap_rel_oracle32=o_fm, rpn_head_rel_engine=e_lg,
                rpn_head_rel_oracle32=o_lg, proposals_px_engine=e_pr, proposals_px_oracle32=o_pr,
                detections_px_engine=e_det, detections_px_oracle32=o_det, probs_abs_engine=e_p, detections=k)
        assert e_fm <= float_bound(o_fm, 5e-6), 'feature map: engine %.2e vs oracle32 %.2e' % (e_fm, o_fm)
        assert e_lg <= float_bound(o_lg, 1e-5), 'rpn heads: engine %.2e vs oracle32 %.2e' % (e_lg, o_lg)
        assert e_pr <= float_bound(o_pr, 1e-3), 'proposals: engine %.2e px vs oracle32 %.2e px' % (e_pr, o_pr)
        assert e_det <= float_bound(o_det, 1e-3), 'detections: engine %.2e px vs oracle32 %.2e px' % (e_det, o_det)
        assert e_p <= 2e-5
        assert (np.diff(scores[i, :k]) <= 0).all()                  # tf.nn.top_k order
        # stage taps that consume the ENGINE's own proposals: compare against the oracle stage fed the same rois
        roi_ref = ofr.roi_pool(props[i, :pcnt[i]], fmap[i][None], (h, w), 7, 7)['roi_pool']
        assert rel_err(pooled[i * 200:i * 200 + pcnt[i]], roi_ref) < 2e-6, 'roi_pool'
        head_ref = ofr.rcnn_head(roi_ref, wts, cfg['model']['rcnn'], arch)
        np.testing.assert_allclose(cls_prob[i, :pcnt[i]], head_ref['cls_prob'], atol=3e-5)
    eng.close()


def test_fasterrcnn_rpn_only_mode():
    """with_rcnn: False -> proposals as objects, labels 0 (predicting.py:85-92)."""
    cfg = frcnn_cfg('resnet_v1_50', ['model.network.with_rcnn=False'])
    wts = synth.make_weights(cfg, seed=3)
    imgs = synth.make_images(1, 160, 192, seed=4)
    eng = Engine(cfg, max_batch=1, max_h=160, max_w=192)
    eng.load_weights(wts).finalize()
    boxes, scores, labels, counts = eng.predict_raw(imgs)
    tru = ofr.forward(imgs[0], wts, cfg, dtype=np.float64)['rpn_prediction']
    ref = ofr.forward(imgs[0], wts, cfg)['rpn_prediction']
    k = int(counts[0])
    assert k == tru['proposals'].shape[0]
    z = np.zeros(k, int)
    e, o = box_dev(boxes[0, :k], z, tru['proposals'], z), box_dev(ref['proposals'], z, tru['proposals'], z)
    _report('frcnn/rpn_only', proposals_px_engine=e, proposals_px_oracle32=o)
    assert e <= float_bound(o, 1e-3)
    np.testing.assert_allclose(np.sort(scores[0, :k]), np.sort(tru['scores']), atol=2e-5)
    assert (labels[0, :k] == 0).all()
    eng.close()


@pytest.mark.parametrize('impl', ['simt', 'tc'])
def test_ssd_stages_and_detections(impl):
    cfg = default_config('ssd', ['model.proposals.min_prob_threshold=0.2'])
    wts = synth.make_weights(cfg, seed=5)
    imgs = synth.make_images(2, 300, 300, seed=6)
    eng = Engine(cfg, max_batch=2)
    eng.load_weights(wts).finalize()
    eng.set_conv_impl(impl)
    eng.set_conv_streamk('off')                        # whole-tile schedule: pipelining is bit-neutral
    piped = eng.predict_raw(imgs)                      # production path: two half-batches on two streams
    eng.set_debug_taps(True)                           # single stream, taps cover the whole batch
    for a, b in zip(piped, eng.predict_raw(imgs)):
        np.testing.assert_array_equal(a, b)
    eng.set_debug_taps(False)
    eng.set_conv_streamk('auto')                       # default schedule: neutral to fp32 noise
    piped = eng.predict_raw(imgs)
    eng.set_debug_taps(True)
    boxes, scores, labels, counts = eng.predict_raw(imgs)
    np.testing.assert_array_equal(piped[3], counts)
    for i in range(2):
        k = int(counts[i])
        assert box_dev(piped[0][i, :k], piped[2][i, :k], boxes[i, :k], labels[i, :k]) <= 2e-3
    loc = eng.get_tensor('loc_pred'); prob = eng.get_tensor('cls_prob'); anchors = eng.get_tensor('all_anchors')
    for i in range(2):
        ref = ossd.forward(imgs[i], wts, cfg)
        tru = ossd.forward(imgs[i], wts, cfg, dtype=np.float64)
        np.testing.assert_array_equal(anchors, ref['all_anchors'])
        worst_e = worst_o = 0.0
        for j, fm in enumerate(tru['feature_maps'].values()):
            worst_e = max(worst_e, rel_err(eng.get_tensor('fmap_%d' % j)[i], fm[0]))
            worst_o = max(worst_o, rel_err(list(ref['feature_maps'].values())[j][0], fm[0]))
        e_loc, o_loc = rel_err(loc[i], tru['loc_pred']), rel_err(ref['loc_pred'], tru['loc_pred'])
        e_pb = float(np.abs(prob[i] - tru['cls_prob']).max()); o_pb = float(np.abs(ref['cls_prob'] - tru['cls_prob']).max())
        k = int(counts[i])
        tc_, rc_ = tru['classification_prediction'], ref['classification_prediction']
        e_det = box_dev(boxes[i, :k], labels[i, :k], tc_['objects'], tc_['labels'])
        o_det = box_dev(rc_['objects'], rc_['labels'], tc_['objects'], tc_['labels'])
        _report('ssd/%s/img%d' % (impl, i), fmap_rel_engine=worst_e, fmap_rel_oracle32=worst_o, loc_rel_engine=e_loc,
                loc_rel_oracle32=o_loc, prob_abs_engine=e_pb, prob_abs_oracle32=o_pb, detections_px_engine=e_det,
                detections_px_oracle32=o_det, detections=k)
        assert worst_e <= float_bound(worst_o, 5e-6), 'feature maps: %.2e vs %.2e' % (worst_e, worst_o)
        assert e_loc <= float_bound(o_loc, 1e-5)
        assert e_pb <= float_bound(o_pb, 2e-5)
        assert e_det <= float_bound(o_det, 1e-3), 'detections: engine %.2e px vs oracle32 %.2e px' % (e_det, o_det)
        assert (np.diff(scores[i, :k]) <= 0).all()
    eng.close()


def test_predictor_network_drop_in_schema():
    """PredictorNetwork(config).predict_image(image) -> [{'bbox','label','prob'}] == oracle predict_image.
    600x640 input: the aspect-preserving resize is the identity (scale_factor 1.0)."""
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=7)
    img = synth.make_images(1, 600, 640, seed=8)[0]
    net = PredictorNetwork(cfg, weights=wts)
    got = net.predict_image(img)
    ref = opredict.predict_image(img, wts, cfg)
    assert isinstance(got, list) and len(got) == len(ref) and len(got) > 0
    for d in got:
        assert set(d) == {'bbox', 'label', 'prob'} and len(d['bbox']) == 4 and all(isinstance(c, int) for c in d['bbox'])
    assert [d['prob'] for d in got] == sorted([d['prob'] for d in got], reverse=True)
    key = lambda d: (d['label'], d['bbox'])
    for g, r in zip(sorted(got, key=key), sorted(ref, key=key)):
        assert g['label'] == r['label'] and g['bbox'] == r['bbox'] and abs(g['prob'] - r['prob']) <= 1.01e-4
    net.engine.close()


def test_engine_fails_loudly_on_missing_weight():
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=1)
    eng = Engine(cfg, max_batch=1, max_h=64, max_w=64)
    name = 'fasterrcnn/rpn/conv/w'
    for n, _ in eng.weight_specs():
        if n != name:
            eng.set_weight(n, wts[n])
    with pytest.raises(ValueError):
        eng.finalize()
    with pytest.raises(ValueError):
        eng.set_weight(name, np.zeros((1, 1, 4, 4), np.float32))     # wrong shape
    eng.close()


@pytest.mark.parametrize('impl', ['tc', 'simt'])
def test_engine_reports_activation_overflow(impl):
    """Activations travel as fp16 hi/lo planes; a layer output beyond the fp16 range must surface as
    LUMI_EOVERFLOW (RuntimeError, code -5), never as silently wrong detections -- and the engine must
    stay usable afterwards."""
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=1)
    big = dict(wts)
    name = [n for n in wts if n.endswith('block1/unit_1/bottleneck_v1/conv1/weights')][0]
    big[name] = wts[name] * np.float32(1e7)
    imgs = synth.make_images(1, 96, 128, seed=5)
    eng = Engine(cfg, max_batch=1, max_h=96, max_w=128)
    eng.load_weights(big).finalize()
    eng.set_conv_impl(impl)
    with pytest.raises(RuntimeError, match='code -5'):
        eng.predict_raw(imgs)
    eng.close()
    eng = Engine(cfg, max_batch=1, max_h=96, max_w=128)
    eng.load_weights(wts).finalize()
    eng.set_conv_impl(impl)
    eng.predict_raw(imgs)           # sane weights: no overflow reported
    eng.close()


def test_stream_k_schedule_is_result_neutral():
    """The stream-K conv schedule only changes the fp32 summation order of split tiles: feature maps agree
    to 1e-5 relative and the detections are the same set within the box tolerance; each mode is
    deterministic (bit-identical on repeat)."""
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=3)
    h, w = 224, 320
    imgs = synth.make_images(2, h, w, seed=4)
    eng = Engine(cfg, max_batch=2, max_h=h, max_w=w)
    eng.load_weights(wts).finalize()
    eng.set_debug_taps(True)
    out = {}
    for mode in ('off', 'always'):
        eng.set_conv_streamk(mode)
        r1 = eng.predict_raw(imgs)
        fm = eng.get_tensor('conv_feature_map').copy()
        r2 = eng.predict_raw(imgs)
        for a, b in zip(r1, r2):
            np.testing.assert_array_equal(a, b)
        out[mode] = (r1, fm)
    (b0, s0, l0, c0), f0 = out['off']
    (b1, s1, l1, c1), f1 = out['always']
    assert rel_err(f1, f0.astype(np.float64)) < 1e-5
    np.testing.assert_array_equal(c0, c1)
    for i in range(2):
        k = int(c0[i])
        assert box_dev(b1[i, :k], l1[i, :k], b0[i, :k], l0[i, :k]) <= 2e-3
    eng.close()


def test_engine_capacity_is_not_part_of_the_result():
    """An engine created for (max_batch 4, 256x384) must give, for a smaller batch of smaller images, exactly
    what a tightly sized engine gives (ragged use of one handle: predicting.py serves images of any size).
    max_h x max_w is a sizing hint: an image beyond it grows the workspace instead of being refused (the
    reference's resize can exceed max_size, utils/image.py:66-86) and still gives the tight engine's result."""
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=7)
    imgs = synth.make_images(1, 160, 224, seed=8)
    big = Engine(cfg, max_batch=4, max_h=256, max_w=384)
    big.load_weights(wts).finalize()
    tight = Engine(cfg, max_batch=1, max_h=160, max_w=224)
    tight.load_weights(wts).finalize()
    a = big.predict_raw(imgs)
    b = tight.predict_raw(imgs)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x[:1], y[:1])
    # a different size on the same handle afterwards, then the first size again: no state leaks between calls
    other = synth.make_images(2, 192, 256, seed=9)
    big.predict_raw(other)
    for x, y in zip(big.predict_raw(imgs), a):
        np.testing.assert_array_equal(x, y)
    larger = synth.make_images(1, 300, 400, seed=1)                    # larger than the planned maximum
    tight2 = Engine(cfg, max_batch=1, max_h=300, max_w=400)
    tight2.load_weights(wts).finalize()
    for x, y in zip(big.predict_raw(larger), tight2.predict_raw(larger)):
        np.testing.assert_array_equal(x[:1], y[:1])
    for x, y in zip(big.predict_raw(imgs), a):                         # and the grown engine still serves the small one
        np.testing.assert_array_equal(x, y)
    big.close(); tight.close(); tight2.close()


def test_predictor_network_wide_image_beyond_max_size():
    """ADVICE r1: a 300x600 input is resized to 600x1200 (the reference multiplies its up- and down-scale factors,
    utils/image.py:66-86), wider than max_size 1024: PredictorNetwork must serve it like the reference does."""
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=7)
    img = synth.make_images(1, 300, 600, seed=31)[0]
    net = PredictorNetwork(cfg, weights=wts)
    got = net.predict_image(img)
    ref = opredict.predict_image(img, wts, cfg)
    assert len(got) == len(ref) and len(got) > 0
    free = list(ref)
    for g in got:
        hit = [r for r in free if r['label'] == g['label'] and abs(r['prob'] - g['prob']) <= 1.01e-4
               and max(abs(a - b) for a, b in zip(g['bbox'], r['bbox'])) <= 1]
        assert hit, 'no reference detection for %r' % (g,)
        free.remove(hit[0])
    net.engine.close()


def test_predict_batch_mixed_sizes_keeps_order():
    """predict_batch buckets images by preprocessed size and returns results in the caller's order; every
    entry equals the single-image call (images are independent units)."""
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=7)
    a = synth.make_images(2, 600, 640, seed=41)
    b = synth.make_images(2, 375, 500, seed=42)
    order = [a[0], b[0], a[1], b[1]]
    net = PredictorNetwork(cfg, weights=wts, max_batch=2)
    assert net.predict_batch([]) == []
    net.engine.set_conv_streamk('off')                 # batch-size independent bits (stream-K split points depend on the batch)
    got = net.predict_batch(order)
    single = [net.predict_image(im) for im in order]
    assert got == single and all(len(g) > 0 for g in got)
    net.engine.close()


def test_predictor_network_restores_a_saver_v2_checkpoint(tmp_path):
    """predicting.py:51-63 without TensorFlow: a job_dir holding `checkpoint` + model.ckpt-N.{index,data-*} (the layout
    of the reference's published checkpoints) gives exactly the detections of the same weights passed in memory."""
    from luminoth_b200 import tf_checkpoint as tfc
    from luminoth_b200.predicting import PredictorNetwork
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=11)
    run = tmp_path / 'jobs' / 'my-run'
    run.mkdir(parents=True)
    extra = dict(wts)
    extra['global_step'] = np.array(90000, np.int64)                          # things a training run also saves
    extra['fasterrcnn/rpn/conv/w/Momentum'] = np.zeros_like(wts['fasterrcnn/rpn/conv/w'])
    tfc.write_bundle(str(run / 'model.ckpt-90000'), extra)
    tfc.write_checkpoint_state(str(run), 'model.ckpt-90000')
    img = synth.make_images(1, 160, 224, seed=12)[0]
    ref_net = PredictorNetwork(frcnn_cfg('resnet_v1_50'), weights=wts)
    want = ref_net.predict_image(img)
    ref_net.engine.close()
    cfg2 = frcnn_cfg('resnet_v1_50', ['train.job_dir=' + str(tmp_path / 'jobs'), 'train.run_name=my-run'])
    net = PredictorNetwork(cfg2)
    got = net.predict_image(img)
    net.engine.close()
    assert got == want and len(got) > 0
    with pytest.raises(ValueError, match='Could not find checkpoint'):
        PredictorNetwork(frcnn_cfg('resnet_v1_50', ['train.job_dir=' + str(tmp_path / 'empty')]))


@pytest.mark.parametrize('shape', [(375, 500), (1200, 1600)])
def test_predictor_network_resized_images_match_the_reference_feed(shape):
    """Images that the dataset preprocessing resizes (utils/image.py:38-114: 375x500 -> 600x800 upscaled,
    1200x1600 -> 768x1024 downscaled) reach the network as FLOAT pixels in the reference (predicting.py:110-112).
    The product path resizes on the GPU and feeds float32; detections must match the oracle's predict_image on the
    original image (integer boxes in original-image pixels, probabilities to 1e-4)."""
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=7)
    img = synth.make_images(1, shape[0], shape[1], seed=21)[0]
    net = PredictorNetwork(cfg, weights=wts)
    got = net.predict_image(img)
    ref = opredict.predict_image(img, wts, cfg)
    assert len(got) == len(ref) and len(got) > 0
    # int(round(coord / scale)) can flip by one pixel when fp32 noise (1e-3 px) meets a .5 boundary: match every
    # detection to an unused reference row of the same label within 1 px and 1e-4 in probability
    free = list(ref)
    exact = 0
    for g in got:
        hit = [r for r in free if r['label'] == g['label'] and abs(r['prob'] - g['prob']) <= 1.01e-4
               and max(abs(a - b) for a, b in zip(g['bbox'], r['bbox'])) <= 1]
        assert hit, 'no reference detection for %r' % (g,)
        best = min(hit, key=lambda r: sum(abs(a - b) for a, b in zip(g['bbox'], r['bbox'])))
        exact += best['bbox'] == g['bbox']
        free.remove(best)
    assert exact >= 0.97 * len(got)
    net.engine.close()


def test_full_size_batch_properties():
    """BASELINE.json's shape (batch 8 x 600x1024, 2000 proposals, 80 classes) is too slow for the CPU oracle, so
    the full-size run is held to size-independent properties: bit-reproducibility, batch-permutation equivariance
    and pipelining neutrality (whole-tile conv schedule), sorted scores, rows inside the image, labels in range."""
    cfg = default_config('fasterrcnn', ['model.base_network.architecture=resnet_v1_50', 'model.network.num_classes=80'])
    wts = synth.make_weights(cfg, seed=0, profile='peaky')
    imgs = synth.make_images(8, 600, 1024, seed=33)
    eng = Engine(cfg, max_batch=8, max_h=600, max_w=1024)
    eng.load_weights(wts).finalize()
    a = eng.predict_raw(imgs)
    for _ in range(5):                                               # eager, graph capture, replays
        for x, y in zip(a, eng.predict_raw(imgs)):
            np.testing.assert_array_equal(x, y)                      # default schedule: run-to-run identical
    boxes, scores, labels, counts = a
    assert counts.min() >= 0 and counts.max() <= eng.max_detections and counts.sum() > 0
    for i in range(8):
        k = int(counts[i])
        assert (np.diff(scores[i, :k]) <= 0).all()
        assert labels[i, :k].min(initial=0) >= 0 and labels[i, :k].max(initial=0) < 80
        bx = boxes[i, :k]
        assert (bx[:, 0] >= 0).all() and (bx[:, 1] >= 0).all() and (bx[:, 2] <= 1023).all() and (bx[:, 3] <= 599).all()
        assert (bx[:, 2] >= bx[:, 0]).all() and (bx[:, 3] >= bx[:, 1]).all()
    eng.set_conv_streamk('off')
    base = eng.predict_raw(imgs)
    perm = np.array([5, 2, 7, 0, 3, 6, 1, 4])
    shuf = eng.predict_raw(imgs[perm])
    for x, y in zip(base, shuf):
        np.testing.assert_array_equal(x[perm], y)                # images are independent units
    eng.set_pipeline(False)
    for x, y in zip(base, eng.predict_raw(imgs)):
        np.testing.assert_array_equal(x, y)                      # two-stream pipeline is bit-neutral
    eng.close()


def test_lumi_eval_on_the_engine_matches_the_oracle_pipeline(tmp_path):
    """SURVEY 8f-3 (`lumi eval`, eval.py:23-224,487-650) end to end: a TFRecord split of PNG images in two sizes, a
    Saver-V2 checkpoint under <job_dir>/<run_name>, the engine's batched forward, COCO-style AP/AR -- compared with the
    same metric code fed by the CPU oracle's detections for the same records.  Ground truth = the oracle's own top
    detections (truncated to integers), so the metrics are far from zero and sensitive to every stage."""
    import io
    from PIL import Image
    from luminoth_b200 import eval as E
    from luminoth_b200 import tf_checkpoint as tfc
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=7)
    run = tmp_path / 'jobs' / 'run1'
    run.mkdir(parents=True)
    tfc.write_bundle(str(run / 'model.ckpt-500'), dict(wts))
    tfc.write_checkpoint_state(str(run), 'model.ckpt-500')
    data = tmp_path / 'data'
    data.mkdir()
    ecfg = E.prepare_eval_config(frcnn_cfg('resnet_v1_50'), 'val', 100)
    images = [synth.make_images(1, 600, 640, seed=50 + i)[0] for i in range(3)] + \
             [synth.make_images(1, 375, 500, seed=60 + i)[0] for i in range(2)]
    payloads, oracle_out = [], {'bboxes': [], 'classes': [], 'scores': [], 'gt_bboxes': [], 'gt_classes': []}
    for i, img in enumerate(images):
        objs, labels, probs, scale = opredict.network_outputs(img, wts, ecfg)        # resized-image coordinates
        top = np.argsort(-probs)[:6]
        gt = [{'label': int(labels[j]), 'xmin': int(objs[j][0] / scale), 'ymin': int(objs[j][1] / scale),
               'xmax': int(objs[j][2] / scale), 'ymax': int(objs[j][3] / scale)} for j in top]
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format='PNG')
        payloads.append(E.make_sequence_example({'width': img.shape[1], 'height': img.shape[0], 'depth': 3,
                                                 'filename': 'img%d.png' % i, 'image_raw': buf.getvalue(), 'gt_boxes': gt}))
        gts = E.scaled_ground_truth(img.shape, np.array([[g['xmin'], g['ymin'], g['xmax'], g['ymax'], g['label']] for g in gt]), ecfg)
        oracle_out['bboxes'].append(objs); oracle_out['classes'].append(labels); oracle_out['scores'].append(probs)
        oracle_out['gt_bboxes'].append(gts[:, :4]); oracle_out['gt_classes'].append(gts[:, 4])
    E.write_tfrecord(str(data / 'val.tfrecords'), payloads)
    cfg2 = frcnn_cfg('resnet_v1_50', ['train.job_dir=' + str(tmp_path / 'jobs'), 'train.run_name=run1',
                                      'dataset.dir=' + str(data)])
    logs = []
    res = E.evaluate(cfg2, 'val', watch=False, max_detections=100, max_batch=2, log=logs.append)
    assert len(res) == 1 and res[0]['global_step'] == 500
    m = res[0]['metrics']
    ap, ar = E.calculate_metrics(oracle_out, 20)
    want = E.summarize_metrics(ap, ar)
    assert m['total_evaluated'] == 5
    # (the mean over 20 classes is diluted by the classes that never appear; the classes that do must score)
    assert np.nanmax(ap[:, 0]) > 0.5, 'the comparison must not be vacuous'
    # per class, like the reference: a class with detections but no ground truth has recall x / 0 = NaN (eval.py:603),
    # so the class means can be NaN on a 5-image split -- on both sides alike
    ap_e = np.array(res[0]['ap_at_50_per_class'])
    np.testing.assert_allclose(ap_e, ap[:, 0], atol=2e-3, equal_nan=True)
    for k in want:
        assert (np.isnan(m[k]) and np.isnan(want[k])) or abs(m[k] - want[k]) <= 2e-3, (k, m[k], want[k])
    assert any('Average Precision (AP) @ [0.50]' in l for l in logs)


def test_nvjpeg_decode_close_to_pil():
    """SURVEY 8f-2: `lumi_decode_jpeg` (nvJPEG, GPU) vs PIL/libjpeg (the reference's decoder, predict.py:72-79) on a
    4:2:0 and a 4:4:4 file: same shape, pixels within a few grey levels (the IDCT / chroma up-sampling differ)."""
    import io
    from PIL import Image
    from luminoth_b200.engine import decode_jpeg
    yy, xx = np.mgrid[0:192, 0:256].astype(np.float64)
    img = np.stack([127 + 120 * np.sin(xx / 37.0) * np.cos(yy / 29.0), 127 + 100 * np.cos(xx / 53.0 + yy / 41.0),
                    40 + 0.7 * xx + 0.1 * yy], -1).clip(0, 255).astype(np.uint8)               # smooth content
    for subsampling in (0, 2):
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format='JPEG', quality=92, subsampling=subsampling)
        got = decode_jpeg(buf.getvalue())
        ref = np.asarray(Image.open(io.BytesIO(buf.getvalue())).convert('RGB'))
        assert got.shape == ref.shape == (192, 256, 3) and got.dtype == np.uint8
        d = np.abs(got.astype(int) - ref.astype(int))
        # 4:4:4 differs only by IDCT rounding; 4:2:0 also by the chroma up-sampling filter (libjpeg's "fancy"
        # triangle filter vs nvJPEG's): a few grey levels on smooth content
        assert d.mean() < (1.0 if subsampling == 0 else 2.5) and np.percentile(d, 99) <= (4 if subsampling == 0 else 12), \
            (subsampling, d.mean(), d.max())
    with pytest.raises(RuntimeError):
        decode_jpeg(b'this is not a jpeg stream at all')
