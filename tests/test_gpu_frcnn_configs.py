"""Faster R-CNN beyond its default head configuration, and the conv kernels those heads launch (`-m gpu`).

The engine reads the anchor grid, the RPN conv (kernel_shape, num_channels, activation_function), the RPN proposal
settings, the RCNN fc stack (layer_sizes, activation_function, use_mean) and the detection limits and variances from
the config.  Each configuration below runs the engine end to end on resnet_v1_50 and is held, stage by stage, to the
float64 oracle with the rules of tests/test_gpu_e2e.py: anchors bit-equal, RPN heads within 1.5 x the fp32 oracle's
noise (floor 1e-5), proposals and detections within 1.5 x its distance (floor 1e-3 px) with identical class assignment,
and the ROI pool and RCNN head against oracle stages fed the engine's own proposals.  The production call (two
half-batches on two streams), the single-stream taps run and a CUDA-graph replay give the same bytes under the
whole-tile conv schedule.

Every configuration draws the same trunk weights (synth draws them first), so the oracle's block3 maps of each image
are computed once per module, and only the head stages per configuration.

The second half runs the stand-alone conv op on non-square and even kernels and on the head and fc shapes these
configurations create, against float64 at sampled pixels (tests/test_gpu_conv_engine_layers.py).
"""
import functools
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import endpoint_oracle as EO
from luminoth_b200 import synth
from luminoth_b200.engine import Engine
from oracle import fasterrcnn as ofr
from oracle import tf_ops as T
from oracle.anchors import fasterrcnn_anchors
from test_gpu_conv_engine_layers import ENGINE, ENGINE_F32, ENGINE_F32_RESERVE, ENGINE_RESERVE, RELU, RELU6, \
    sample_pixels
from test_gpu_conv_numerics import check, conv_io, out_geometry, reference
from test_gpu_e2e import box_dev, float_bound, frcnn_cfg, rel_err, _report

ARCH = 'resnet_v1_50'
SEED = 1
SIZES = {(224, 320): 2, (231, 329): 3}       # image size -> image seed; batch 2 of each
RPN, RCNN = 'fasterrcnn/rpn', 'fasterrcnn/rcnn'

# id -> (config settings as {dotted key: value}, {weight name: factor} applied to the synthetic draw, image size,
#        conv impl).  The pre-activation of each layer whose activation or kernel a case sets has values below 0 and
#        above 6 (a factor puts it there where the draw alone does not), so that relu, relu6 and the identity differ.
CASES = {
    'anchors_9': ({'model.anchors.scales': [0.5, 1, 2], 'model.anchors.ratios': [0.5, 1, 2]}, {}, (224, 320), 'tc'),
    'anchors_1': ({'model.anchors.scales': [1], 'model.anchors.ratios': [1], 'model.anchors.base_size': 100}, {},
                  (224, 320), 'tc'),
    'anchors_15_frac': ({'model.anchors.scales': [0.3, 0.55, 1.1, 1.7, 2.3], 'model.anchors.ratios': [0.3, 1, 3.5],
                         'model.anchors.base_size': 150}, {}, (224, 320), 'tc'),
    'rpn_5x3_relu_256': ({'model.rpn.kernel_shape': [5, 3], 'model.rpn.num_channels': 256,
                          'model.rpn.activation_function': 'relu'}, {}, (231, 329), 'tc'),
    'rpn_5x3_relu_256_simt': ({'model.rpn.kernel_shape': [5, 3], 'model.rpn.num_channels': 256,
                               'model.rpn.activation_function': 'relu'}, {}, (231, 329), 'simt'),
    'rpn_2x2_320': ({'model.rpn.kernel_shape': [2, 2], 'model.rpn.num_channels': 320}, {},
                    (224, 320), 'tc'),
    'rpn_1x1_200_identity': ({'model.rpn.kernel_shape': [1, 1], 'model.rpn.num_channels': 200,
                              'model.rpn.activation_function': None}, {RPN + '/conv/w': 2.0}, (224, 320),
                             'tc'),
    'fc_4096_4096': ({'model.rcnn.layer_sizes': [4096, 4096], 'model.rpn.proposals.post_nms_top_n': 64},
                     {}, (224, 320), 'tc'),
    'fc_100_no_mean_identity': ({'model.rcnn.layer_sizes': [100], 'model.rcnn.use_mean': False,
                                 'model.rcnn.activation_function': None}, {}, (224, 320), 'tc'),
    'det_limits_1class': ({'model.network.num_classes': 1, 'model.rcnn.proposals.class_max_detections': 7,
                           'model.rcnn.proposals.total_max_detections': 5,
                           'model.rcnn.proposals.class_nms_threshold': 0.3,
                           'model.rcnn.target_normalization_variances': [1, 1]}, {}, (224, 320), 'tc'),
    'det_91_var_null': ({'model.network.num_classes': 91, 'model.rcnn.proposals.class_max_detections': 300,
                         'model.rcnn.proposals.total_max_detections': 1000,
                         'model.rcnn.proposals.min_prob_threshold': 0.0,
                         'model.rcnn.target_normalization_variances': None}, {}, (224, 320), 'tc'),
    'det_class_max_20': ({'model.rcnn.proposals.class_max_detections': 3,
                          'model.rcnn.proposals.total_max_detections': 40,
                          'model.rcnn.proposals.min_prob_threshold': 0.0}, {}, (224, 320), 'tc'),
    'rpn_filters': ({'model.rpn.proposals.filter_outside_anchors': True, 'model.rpn.proposals.clip_after_nms': True,
                     'model.rpn.proposals.min_prob_threshold': 0.4, 'model.rpn.proposals.nms_threshold': 0.5}, {},
                    (224, 320), 'tc'),
    # min_prob_threshold only removes proposals while fewer than pre_nms_top_n candidates pass it and fewer than
    # post_nms_top_n survive the NMS, so rpn_filters leaves both counts alone: pre_nms_top_n is cut here, and
    # post_nms_top_n in fc_4096_4096
    'rpn_no_nms': ({'model.rpn.proposals.apply_nms': False, 'model.rpn.proposals.pre_nms_top_n': 300}, {},
                   (224, 320), 'tc'),
    'anchors_9_rpn_only': ({'model.anchors.scales': [0.5, 1, 2], 'model.anchors.ratios': [0.5, 1, 2],
                            'model.network.with_rcnn': False}, {}, (224, 320), 'tc'),
}


def case_config(settings):
    cfg = frcnn_cfg(ARCH)
    for key, value in settings.items():
        node = cfg
        *path, last = key.split('.')
        for k in path:
            node = node[k]
        node[last] = value
    return cfg


def case_weights(cfg, factors):
    """synth's draw, each weight in `factors` scaled, and the RCNN fc biases drawn non-zero (synth draws them as
    zeros): from a generator of their own, so no other draw changes."""
    wts = synth.make_weights(cfg, seed=SEED)
    for name, f in factors.items():
        wts[name] = wts[name] * np.float32(f)
    rng = np.random.default_rng([SEED, 7])
    for i, size in enumerate(cfg['model']['rcnn'].get('layer_sizes') or []):
        wts['%s/fc_%d/b' % (RCNN, i)] = (rng.standard_normal(size) * 0.5).astype(np.float32)
    return wts


@functools.lru_cache(maxsize=None)
def _images(h, w):
    return synth.make_images(2, h, w, seed=SIZES[(h, w)])


@functools.lru_cache(maxsize=None)
def _base_config():
    return frcnn_cfg(ARCH).to_dict()


@functools.lru_cache(maxsize=None)
def _base_weights():
    return synth.make_weights(_base_config(), seed=SEED)


@functools.lru_cache(maxsize=None)
def _trunk(h, w, i, dtype):
    """The oracle's block3 map (1, fh, fw, 1024) of image i of the (h, w) batch, in float32 or float64."""
    return EO.trunk(_images(h, w)[i][None].astype(dtype), _base_weights(), ARCH)


def _assert_same_trunk(wts):
    base = _base_weights()
    trunk = [k for k in base if k.startswith('truncated_base_network/')]
    assert trunk and all(k in wts for k in trunk)
    for k in trunk:
        np.testing.assert_array_equal(wts[k], base[k], err_msg=k)


def _rpn_pre_activation(fmap64, wts):
    return T.conv2d(fmap64, wts[RPN + '/conv/w'], 1, 'SAME', bias=wts[RPN + '/conv/b'])


def _fc_pre_activations(roi64, wts, rcfg):
    """float64 inputs of each RCNN fc layer's activation, on pooled ROIs."""
    feats = roi64.mean(axis=(1, 2)) if rcfg.get('use_mean', True) else roi64
    net = feats.reshape(feats.shape[0], -1)
    act = ofr.activation(rcfg.get('activation_function'))
    out = []
    for i, _ in enumerate(rcfg.get('layer_sizes') or []):
        pre = net @ wts['%s/fc_%d/w' % (RCNN, i)].astype(np.float64) + wts['%s/fc_%d/b' % (RCNN, i)]
        out.append(pre)
        net = act(pre)
    return out


def _straddles(pre):
    return float(pre.min()) < 0 and float(pre.max()) > 6


def _check_not_vacuous(cid, settings, ocfg, wts, tru, fmap64, im_shape):
    """Each case's setting changes the oracle's result."""
    m = ocfg['model']
    if 'model.rpn.activation_function' in settings or 'model.rpn.kernel_shape' in settings:
        pre = _rpn_pre_activation(fmap64, wts)
        assert _straddles(pre), '%s: RPN pre-activation in [%.2f, %.2f]' % (cid, pre.min(), pre.max())
    if m['rcnn'].get('layer_sizes') and m['network']['with_rcnn']:
        for i, pre in enumerate(_fc_pre_activations(tru['roi']['roi_pool'], wts, m['rcnn'])):
            assert _straddles(pre), '%s: fc_%d pre-activation in [%.2f, %.2f]' % (cid, i, pre.min(), pre.max())
            assert np.abs(wts['%s/fc_%d/b' % (RCNN, i)]).min() > 0
    if 'model.anchors.base_size' in settings:
        a = m['anchors']
        exact = [s * np.sqrt(r) * a['base_size'] for r in a['ratios'] for s in a['scales']]
        if cid.endswith('frac'):    # corners (size - 1) / 2 that truncation toward zero changes
            assert any(((e - 1) / 2) % 1 != 0 for e in exact)
    rpn_prefix = 'model.rpn.proposals.'
    for key in settings:            # each RPN proposal setting, alone back at its default, changes the proposals
        if key.startswith(rpn_prefix):
            name = key[len(rpn_prefix):]
            pcfg = dict(m['rpn']['proposals'], **{name: _base_config()['model']['rpn']['proposals'][name]})
            other = ofr.rpn_proposal(tru['rpn']['rpn_cls_prob'], tru['rpn']['rpn_bbox_pred'], tru['all_anchors'],
                                     im_shape, pcfg)['proposals']
            assert _differ(other, tru['rpn_prediction']['proposals']), '%s: %s changes nothing' % (cid, name)
    if 'model.rcnn.proposals.total_max_detections' in settings:
        p = m['rcnn']['proposals']
        props, head = tru['rpn_prediction']['proposals'], tru['rcnn']
        var = m['rcnn'].get('target_normalization_variances')

        def detect(**limits):
            return ofr.rcnn_proposal(props, head['bbox_offsets'], head['cls_prob'], im_shape,
                                     m['network']['num_classes'], dict(p, **limits), variances=var)
        got = tru['classification_prediction']['objects']
        per_class = [len(s) for s in detect(class_max_detections=10 ** 6)['selected_probs']]
        capped = sum(min(c, p['class_max_detections']) for c in per_class)
        assert capped > p['total_max_detections'], '%s: %d candidates' % (cid, capped)    # total_max cuts
        # class_max can only show below total_max (a class never places more than total_max rows) and below the
        # proposal count (no class has more rows than that)
        if p['class_max_detections'] < min(p['total_max_detections'], len(props)):
            assert max(per_class) > p['class_max_detections'], '%s: class_max cuts no class' % cid
            assert _differ(detect(class_max_detections=10 ** 6)['objects'], got), '%s: class_max changes nothing' % cid
        if 'model.rcnn.target_normalization_variances' in settings:
            default = ofr.rcnn_proposal(props, head['bbox_offsets'], head['cls_prob'], im_shape,
                                        m['network']['num_classes'], p, variances=[0.1, 0.2])
            assert _differ(default['objects'], got), '%s: the variances do not change the detections' % cid


def _differ(a, b):
    return a.shape != b.shape or not np.allclose(a, b)


@pytest.mark.parametrize('cid', list(CASES))
def test_head_configuration_stages_and_detections(cid):
    settings, factors, (h, w), impl = CASES[cid]
    cfg = case_config(settings)
    ocfg = cfg.to_dict()
    m = ocfg['model']
    with_rcnn = m['network']['with_rcnn']
    a = m['anchors']
    A = len(a['scales']) * len(a['ratios'])
    post = m['rpn']['proposals']['post_nms_top_n'] if m['rpn']['proposals']['apply_nms'] else \
        m['rpn']['proposals']['pre_nms_top_n']
    wts = case_weights(cfg, factors)
    _assert_same_trunk(wts)
    imgs = _images(h, w)
    eng = Engine(cfg, max_batch=2, max_h=h, max_w=w)
    eng.load_weights(wts).finalize()
    eng.set_conv_impl(impl)
    # whole-tile conv schedule: the pipelined production call, two graph replays and the taps run give the same bytes
    eng.set_conv_streamk('off')
    piped = eng.predict_raw(imgs)
    for _ in range(2):
        for x, y in zip(piped, eng.predict_raw(imgs)):
            np.testing.assert_array_equal(x, y)
    assert eng.last_graph_replays > 0
    eng.set_debug_taps(True)
    for x, y in zip(piped, eng.predict_raw(imgs)):
        np.testing.assert_array_equal(x, y)
    eng.set_conv_streamk('auto')
    boxes, scores, labels, counts = eng.predict_raw(imgs)
    fmap = eng.get_tensor('conv_feature_map')
    anchors = eng.get_tensor('all_anchors').reshape(-1, 4)
    heads = eng.get_tensor('rpn_heads')
    props = eng.get_tensor('proposals')
    pcnt = eng.get_tensor('proposal_counts').astype(int)
    if with_rcnn:
        pooled = eng.get_tensor('roi_pool')
        cls_prob = eng.get_tensor('rcnn_cls_prob')
    eng.close()
    fh, fw = fmap.shape[1:3]
    assert heads.reshape(2, -1).shape[1] == fh * fw * 6 * A
    assert anchors.shape == (fh * fw * A, 4)
    total = 0
    for i in range(2):
        f32, f64 = _trunk(h, w, i, np.float32), _trunk(h, w, i, np.float64)
        ref = EO.fasterrcnn_heads(f32, (h, w), wts, ocfg)
        tru = EO.fasterrcnn_heads(f64, (h, w), wts, ocfg)
        if i == 0:
            _check_not_vacuous(cid, settings, ocfg, wts, tru, f64, (h, w))
        np.testing.assert_array_equal(anchors, tru['all_anchors'])
        np.testing.assert_array_equal(anchors, fasterrcnn_anchors(fh, fw, a['base_size'], a['ratios'], a['scales'],
                                                                  a['stride']))
        e_fm, o_fm = rel_err(fmap[i], f64[0]), rel_err(f32[0], f64[0])
        rh = heads[i].reshape(-1, 6 * A)
        lg = np.concatenate([rh[:, :2 * A].reshape(-1), rh[:, 2 * A:].reshape(-1)])
        lg_t = np.concatenate([tru['rpn']['rpn_cls_score'].reshape(-1), tru['rpn']['rpn_bbox_pred'].reshape(-1)])
        lg_r = np.concatenate([ref['rpn']['rpn_cls_score'].reshape(-1), ref['rpn']['rpn_bbox_pred'].reshape(-1)])
        e_lg, o_lg = rel_err(lg, lg_t), rel_err(lg_r, lg_t)
        tp, rp = tru['rpn_prediction']['proposals'], ref['rpn_prediction']['proposals']
        assert pcnt[i] == tp.shape[0], 'proposal count %d vs %d' % (pcnt[i], tp.shape[0])
        assert 0 < pcnt[i] <= post
        z = np.zeros(pcnt[i], int)
        e_pr, o_pr = box_dev(props[i, :pcnt[i]], z, tp, z), box_dev(rp, z, tp, z)
        assert e_fm <= float_bound(o_fm, 5e-6), 'feature map: engine %.2e vs oracle32 %.2e' % (e_fm, o_fm)
        assert e_lg <= float_bound(o_lg, 1e-5), 'rpn heads: engine %.2e vs oracle32 %.2e' % (e_lg, o_lg)
        assert e_pr <= float_bound(o_pr, 1e-3), 'proposals: engine %.2e px vs oracle32 %.2e px' % (e_pr, o_pr)
        k = int(counts[i])
        total += k
        key = 'frcnn_config/%s/img%d' % (cid, i)
        if not with_rcnn:      # the detections are the proposals
            assert k == pcnt[i]
            np.testing.assert_array_equal(boxes[i, :k], props[i, :k])
            _report(key, rpn_head_rel_engine=e_lg, rpn_head_rel_oracle32=o_lg, proposals_px_engine=e_pr,
                    proposals_px_oracle32=o_pr, detections=k)
            continue
        tc_, rc_ = tru['classification_prediction'], ref['classification_prediction']
        e_det = box_dev(boxes[i, :k], labels[i, :k], tc_['objects'], tc_['labels'])
        o_det = box_dev(rc_['objects'], rc_['labels'], tc_['objects'], tc_['labels'])
        e_p = float(np.abs(np.sort(scores[i, :k]) - np.sort(tc_['probs'])).max()) if k else 0.0
        _report(key, rpn_head_rel_engine=e_lg, rpn_head_rel_oracle32=o_lg, proposals_px_engine=e_pr,
                proposals_px_oracle32=o_pr, detections_px_engine=e_det, detections_px_oracle32=o_det,
                probs_abs_engine=e_p, detections=k)
        assert e_det <= float_bound(o_det, 1e-3), 'detections: engine %.2e px vs oracle32 %.2e px' % (e_det, o_det)
        assert e_p <= 2e-5
        assert (np.diff(scores[i, :k]) <= 0).all()
        roi_ref = ofr.roi_pool(props[i, :pcnt[i]], fmap[i][None], (h, w), 7, 7)['roi_pool']
        assert rel_err(pooled[i * post:i * post + pcnt[i]], roi_ref) < 2e-6, 'roi_pool'
        head_ref = ofr.rcnn_head(roi_ref, wts, m['rcnn'], ARCH)
        np.testing.assert_allclose(cls_prob[i, :pcnt[i]], head_ref['cls_prob'], atol=3e-5)
    assert total > 0, 'the comparison must not be vacuous'


def test_activation_function_null_empty_missing_and_unknown():
    """get_activation_function (utils/vars.py:80-88): null and '' are the identity, a missing key keeps the relu6
    default, and a name other than relu / relu6 is refused when the engine is created."""
    imgs = synth.make_images(1, 96, 128, seed=5)

    def run(rpn_act, rcnn_act):
        cfg = case_config({'model.rcnn.layer_sizes': [64], 'model.rpn.proposals.post_nms_top_n': 50})
        for part, act in (('rpn', rpn_act), ('rcnn', rcnn_act)):
            if act == 'missing':
                del cfg['model'][part]['activation_function']
            else:
                cfg['model'][part]['activation_function'] = act
        eng = Engine(cfg, max_batch=1, max_h=96, max_w=128)
        eng.load_weights(case_weights(cfg, {})).finalize()
        eng.set_debug_taps(True)
        out = tuple(eng.predict_raw(imgs)) + (eng.get_tensor('rpn_heads'), eng.get_tensor('rcnn_fc'))
        eng.close()
        return out

    def same(a, b):
        return all(np.array_equal(x, y) for x, y in zip(a, b))

    relu6 = run('relu6', 'relu6')
    assert same(run('missing', 'missing'), relu6)
    none = run(None, None)
    assert same(run('', ''), none)
    assert not np.array_equal(none[4], relu6[4])                 # the RPN activation matters here
    rpn_only = run(None, 'relu6')
    assert not np.array_equal(rpn_only[5], none[5])              # and so does the fc's
    for part in ('rpn', 'rcnn'):
        cfg = case_config({'model.rcnn.layer_sizes': [64], 'model.%s.activation_function' % part: 'tanh'})
        with pytest.raises(ValueError, match="unsupported activation_function 'tanh'"):
            Engine(cfg, max_batch=1, max_h=96, max_w=128)


# ---------------------------------------------------------------------------------------------- stand-alone conv op
# (name, n, h, w, cin, cout, kh, kw, stride, padding, act, fp32 outputs, signed input)
CONV_ROWS = [
    ('k5x3_s1_same_c1024', 2, 15, 21, 1024, 256, 5, 3, 1, 'SAME', RELU, False, False),
    ('k3x5_s1_same_c1024', 2, 14, 20, 1024, 256, 3, 5, 1, 'SAME', RELU6, False, False),
    ('k3x5_s2_same_c256', 2, 29, 37, 256, 128, 3, 5, 2, 'SAME', RELU, False, True),
    ('k5x3_s2_valid_c256', 2, 29, 37, 256, 96, 5, 3, 2, 'VALID', 0, False, True),
    ('k1x7_s1_valid_c1024', 2, 14, 20, 1024, 128, 1, 7, 1, 'VALID', RELU, False, False),
    ('k7x1_s2_same_c256', 2, 23, 17, 256, 64, 7, 1, 2, 'SAME', 0, False, True),
    ('k7x1_s1_valid_c256', 1, 16, 11, 256, 128, 7, 1, 1, 'VALID', RELU, False, False),
    ('k2x2_s1_same_c1024', 2, 14, 20, 1024, 320, 2, 2, 1, 'SAME', RELU6, False, False),
    ('k2x2_s2_valid_c256', 2, 15, 21, 256, 128, 2, 2, 2, 'VALID', RELU, False, True),
    ('k2x2_s2_same_c1024', 1, 15, 21, 1024, 64, 2, 2, 2, 'SAME', 0, False, False),
    ('k4x4_s1_same_c256', 2, 15, 21, 256, 128, 4, 4, 1, 'SAME', RELU, False, True),
    ('k4x4_s2_same_c1024', 1, 15, 21, 1024, 256, 4, 4, 2, 'SAME', RELU6, False, False),
    ('k4x4_s1_valid_c256', 2, 14, 20, 256, 64, 4, 4, 1, 'VALID', 0, False, True),
    # the heads and fc layers of the configurations above
    ('rpn_heads_a1', 2, 14, 20, 512, 6, 1, 1, 1, 'SAME', 0, True, False),
    ('rpn_heads_a9', 2, 14, 20, 512, 54, 1, 1, 1, 'SAME', 0, True, False),
    ('rpn_heads_a15', 2, 14, 20, 512, 90, 1, 1, 1, 'SAME', 0, True, False),
    ('rpn_heads_c320', 2, 14, 20, 320, 72, 1, 1, 1, 'SAME', 0, True, False),
    ('rpn_heads_c200', 2, 14, 20, 200, 72, 1, 1, 1, 'SAME', 0, True, True),
    ('rpn_conv_1x1_c200', 2, 14, 20, 1024, 200, 1, 1, 1, 'SAME', 0, False, False),
    ('rcnn_heads_c91', 400, 1, 1, 1024, 456, 1, 1, 1, 'SAME', 0, True, False),
    ('fc_1024_4096', 128, 1, 1, 1024, 4096, 1, 1, 1, 'SAME', RELU6, False, False),
    ('fc_4096_4096', 128, 1, 1, 4096, 4096, 1, 1, 1, 'SAME', RELU6, False, False),
    ('fc_50176_100', 128, 1, 1, 50176, 100, 1, 1, 1, 'SAME', 0, False, False),
]
SIMT, SIMT_SPLIT = 0, 13


def _codes(row):
    """The SIMT codes (the op writes split planes for C_out a multiple of 32 only), and the engine's tensor-core
    launches where the tensor-core kernel takes the layer (C_in a multiple of 64, and C_out a multiple of 32 for split
    outputs): elsewhere the engine runs the SIMT kernel."""
    _, _, _, _, cin, cout, _, _, _, _, _, fp32, _ = row
    codes = [SIMT] if fp32 or cout % 32 else [SIMT, SIMT_SPLIT]
    if cin % 64 == 0 and (fp32 or cout % 32 == 0):
        codes += [ENGINE_F32, ENGINE_F32_RESERVE] if fp32 else [ENGINE, ENGINE_RESERVE]
    return codes


@pytest.mark.parametrize('row', CONV_ROWS, ids=[r[0] for r in CONV_ROWS])
def test_conv_kernel_shapes_match_float64(row):
    """Non-square and even kernels (TF SAME puts the odd padding pixel at the bottom / right: pad_top 0 for a 2x2 at
    stride 1, 1 for a 4x4) and the head / fc shapes, per element at sampled pixels."""
    name, n, h, w, cin, cout, kh, kw, stride, padding, act, fp32, signed = row
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    x = rng.standard_normal((n, h, w, cin), dtype=np.float32)
    if not signed:
        np.abs(x, out=x)
    wt = (rng.standard_normal((kh, kw, cin, cout)) * np.sqrt(2.0 / (kh * kw * cin))).astype(np.float32)
    bias = (rng.standard_normal(cout) * 0.05).astype(np.float32)
    ho, wo, pt, pl = out_geometry(h, w, kh, stride, 1, padding, kw=kw)
    if padding == 'SAME':
        assert (pt, pl) == (T.same_pads(h, kh, stride)[1], T.same_pads(w, kw, stride)[1])
    at = sample_pixels(n, ho, wo, zlib.crc32(name.encode()) + 1)
    codes = _codes(row)
    if kh == kw == 1 and cin == 50176:
        # C_out 100: the engine runs this fc on the SIMT kernel, writing split planes, which the op only writes for
        # C_out a multiple of 32; code 0 runs the same K = 50 176 accumulation with fp32 outputs
        assert codes == [SIMT]
    for impl in codes:
        rc, y, _ = conv_io(x, wt, stride, padding, None, bias, None, 1, act, impl)
        assert rc == 0
        assert y.shape == (n, ho, wo, cout)
        ref, bound = reference(x, wt, stride, padding, None, bias, None, 1, act, impl, at=at)
        check('%s/impl%d (%d px)' % (name, impl, len(at[0])), y[at], ref, bound)
