"""SSD beyond its default 300x300 configuration, the float32 input path on SSD, and the conv4_3 L2 norm (`-m gpu`).

The engine takes any fixed_height / fixed_width, num_classes, anchors_per_point, ratios, min_scale and max_scale: the
feature-map grids, the anchors, the multibox head widths 4A + (C + 1)A, the head repack and the length of every class
NMS list follow from them.  Each configuration below is held to the float64 oracle with the rule of
tests/test_gpu_e2e.py: distance <= max(floor, 1.5 x the fp32 oracle's own distance), identical class assignment, and
anchors bit-equal to the oracle's.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import gpu_ops as G
from luminoth_b200.engine import Engine
from luminoth_b200.predicting import PredictorNetwork
from luminoth_b200 import synth
from oracle import predict as opredict
from test_gpu_e2e import match_reference, ssd_parity, _report
from test_gpu_float_input import resized_float_images
from test_ssd_config_host import ssd_cfg

NMS_PATH_UNSTAGED = 2         # lumi_nms_path: the one-phase scan without the shared-memory stage


# (h, w, num_classes, anchors_per_point or None for the default [4,6,6,6,4,4], other anchor keys, min_prob_threshold,
#  conv impl, batch, pinned anchor count).  Batch 3 runs the two-stream pipeline on halves of 2 and 1.
SSD_CONFIGS = [
    (512, 512, 20, None, {}, 0.0, 'tc', 1, 24656),
    (272, 272, 20, None, {}, 0.2, 'tc', 1, 7034),                   # the smallest size: last map 1x1
    (301, 333, 20, None, {}, 0.2, 'tc', 3, 8958),                   # odd sides, fh != fw
    (301, 333, 20, None, {}, 0.2, 'simt', 1, 8958),
    (300, 500, 80, None, {}, 0.2, 'tc', 1, 13716),                  # non-square, heads 340 / 510 wide
    (300, 300, 20, [3, 5, 5, 5, 3, 3], {}, 0.2, 'tc', 1, 6287),     # odd head widths 75 / 125
    (300, 300, 80, [6, 6, 6, 6, 6, 6], {'min_scale': 0.2, 'max_scale': 0.95}, 0.2, 'simt', 1, 10854),
]


def _config_id(c):
    h, w, nc, app, other, mp, impl, n, _ = c
    return '%dx%d-c%d%s%s-p%g-%s-b%d' % (h, w, nc, '-a' + ''.join(map(str, app)) if app else '',
                                        '-scales' if other else '', mp, impl, n)


@pytest.mark.parametrize('case', SSD_CONFIGS, ids=_config_id)
def test_ssd_configurations_stages_and_detections(case):
    """Every tap and the detections against the oracle.  At 512x512 with min_prob_threshold 0 each of the 20 class
    lists holds all 24 656 anchors: beyond the staged scan's shared memory, so the class NMS takes the one-phase
    unstaged scan (lumi_nms_path 2).  The batch-3 case also checks that, under the whole-tile conv schedule, the
    two-stream run gives the same bytes as the single-stream taps run."""
    h, w, nc, app, other, min_prob, impl, n, pinned = case
    cfg = ssd_cfg(h, w, nc, app, **other)
    cfg['model']['proposals']['min_prob_threshold'] = min_prob
    wts = synth.make_weights(cfg, seed=5)
    imgs = synth.make_images(n, h, w, seed=6)
    eng = Engine(cfg, max_batch=n)
    eng.load_weights(wts).finalize()
    eng.set_conv_impl(impl)
    if n > 1:
        eng.set_conv_streamk('off')
        piped = eng.predict_raw(imgs)                  # two half-batches on two streams
        eng.set_debug_taps(True)                       # one stream, taps over the whole batch
        for a, b in zip(piped, eng.predict_raw(imgs)):
            np.testing.assert_array_equal(a, b)
        eng.set_conv_streamk('auto')
    eng.set_debug_taps(True)
    out = eng.predict_raw(imgs)                        # default conv schedule
    total = eng.get_tensor('all_anchors').shape[0]
    print('SSD %dx%d, %d classes, anchors_per_point %s: %d anchors' % (h, w, nc, app or 'default', total))
    assert total == pinned
    if min_prob == 0.0:
        assert G.nms_path(n * nc, total, 0.45) == NMS_PATH_UNSTAGED
    ssd_parity('ssd_config/%s' % _config_id(case), eng, imgs, wts, cfg, out)
    eng.close()


@pytest.mark.parametrize('impl', ['tc', 'simt'])
def test_ssd_float_pixels_stages_and_detections(impl):
    """375x500 images resized to 300x300 on the GPU (float pixels, as PredictorNetwork feeds them): the taps and
    detections of lumi_predict_f32 against the oracle fed the same float array.  On tc this is the only run of the
    float branch of the conv1_1 staging and of the low activation plane of the tensor-core conv1_1."""
    cfg = ssd_cfg(300, 300)
    cfg['model']['proposals']['min_prob_threshold'] = 0.2
    wts = synth.make_weights(cfg, seed=5)
    imgs = resized_float_images(2, 375, 500, 300, 300, seed=9)
    eng = Engine(cfg, max_batch=2)
    eng.load_weights(wts).finalize()
    eng.set_conv_impl(impl)
    eng.set_debug_taps(True)
    out = eng.predict_raw(imgs)
    ssd_parity('ssd_float/%s' % impl, eng, imgs, wts, cfg, out)
    eng.close()


def test_predictor_network_on_ssd():
    """PredictorNetwork.predict_image on SSD against the oracle's predict_image: 375x500 and 480x640 images are
    resized to 300x300 and take the float32 entry point, a 300x300 uint8 image the untouched uint8 one.  Then
    predict_batch with max_batch 2 on a mix of them: in that batch the 300x300 image is resized with the others and
    fed as float, and every entry must still equal the single-image call, in the caller's order."""
    cfg = ssd_cfg(300, 300)
    cfg['model']['proposals']['min_prob_threshold'] = 0.2
    wts = synth.make_weights(cfg, seed=5)
    a = synth.make_images(1, 375, 500, seed=71)[0]
    b = synth.make_images(1, 480, 640, seed=72)[0]
    u = synth.make_images(2, 300, 300, seed=73)
    net = PredictorNetwork(cfg, weights=wts, max_batch=2)
    net.engine.set_conv_streamk('off')                 # batch-size independent bits
    for img in (a, b, u[0]):
        match_reference(net.predict_image(img), opredict.predict_image(img, wts, cfg))
    order = [a, u[0], b, u[1], a]
    got = net.predict_batch(order)
    single = [net.predict_image(im) for im in order]
    assert got == single and all(len(g) > 0 for g in got)
    net.engine.close()


# ---------------------------------------------------------------- conv4_3 L2 norm x gamma
def split_rejoin(x):
    """x as the engine stores it: hi = fp16(x), lo = fp16(x - hi), read back as hi + lo in fp32."""
    x = np.asarray(x, np.float32)
    hi = x.astype(np.float16)
    lo = (x - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float32) + lo.astype(np.float32)


EPS = float(np.float32(1e-12))


def _l2norm_input(c, seed):
    """15 pixels (8 per CTA: the last CTA is partial) of c channels: all zeros (after a ReLU), sum(x^2) < eps (fp16
    subnormals, which the split stores exactly), a one-hot pixel, a negative one-hot pixel below eps, and the rest
    uniform with per-pixel magnitudes from 1e-3 to 6e4."""
    rng = np.random.default_rng(seed)
    scale = np.logspace(-3, np.log10(6e4), 15)
    x = rng.uniform(-1, 1, (15, c)) * scale[:, None]
    x[0] = 0
    x[1] = 0
    x[1, rng.choice(c, 8, replace=False)] = rng.choice([-3, -2, 2, 3], 8) * 2.0 ** -24   # sum(x^2) <= 72 * 2^-48
    x[2] = 0
    x[2, c // 3] = 3.7
    x[3] = 0
    x[3, c - 1] = -2.0 ** -21
    x = split_rejoin(x.reshape(1, 3, 5, c))
    assert (x.astype(np.float64)[0, 0, 1] ** 2).sum() < EPS and (x.astype(np.float64)[0, 0, 3] ** 2).sum() < EPS
    gamma = rng.uniform(-25, 25, c).astype(np.float32)                                  # negative entries too
    return x, gamma


def _l2norm_f64(x, gamma):
    x = x.astype(np.float64)
    ss = (x * x).sum(-1, keepdims=True)
    return x / np.sqrt(np.maximum(ss, EPS)) * gamma.astype(np.float64)


def _l2norm_f32(x, gamma):
    """tf.nn.l2_normalize x gamma restated in float32 (fp32 sum of squares, as TF and the kernel do)."""
    ss = np.sum(x * x, axis=-1, keepdims=True, dtype=np.float32)
    return (x * (np.float32(1) / np.sqrt(np.maximum(ss, np.float32(EPS))))) * gamma


@pytest.mark.parametrize('c', [32, 48, 100, 512, 1000])
def test_l2norm_scale_matches_float64(c):
    """lumi_op_l2norm_scale against float64 x / sqrt(max(sum x^2, eps)) * gamma on the split-rejoined input.

    Tolerance, per element: K ulps of the float64 value (as fp32) plus 2^-25.  The kernel sums the squares in fp32;
    the float32 restatement of the same formula is D ulps from float64 (about 3 here: the sum, the square root, the
    reciprocal and two products each round once).  K = 1.5 D + 2: the suite's 1.5 margin for another fp32
    implementation of the same arithmetic, plus the output's split planes, which keep 22 significant bits (at most
    2 ulps) and, once the low plane is subnormal, an absolute 2^-25.  A pixel with sum(x^2) < eps must come out as
    x * 1e6 * gamma; a kernel that added eps instead of taking the max would be off by 5 % and more there."""
    x, gamma = _l2norm_input(c, seed=c)
    y = G.l2norm_scale(x, gamma, EPS)
    y64 = _l2norm_f64(x, gamma)
    assert np.isfinite(y).all()
    ulp = np.spacing(np.abs(y64).astype(np.float32)).astype(np.float64)
    d32 = float((np.abs(_l2norm_f32(x, gamma) - y64) / ulp).max())
    k = 1.5 * d32 + 2
    err = np.abs(y - y64) - 2.0 ** -25
    worst = float((err / ulp).max())
    _report('l2norm/c%d' % c, ulps_engine_beyond_floor=worst, ulps_oracle32=d32, ulps_bound=k)
    assert worst <= k, 'l2norm: %.2f ulps beyond 2^-25 (bound %.2f; fp32 restatement %.2f)' % (worst, k, d32)
    np.testing.assert_array_equal(y[0, 0, 0], 0)                                         # all-zero pixel stays zero
    small = x[0, 0, 1].astype(np.float64) * 1e6 * gamma
    np.testing.assert_allclose(y[0, 0, 1], small, rtol=1e-6, atol=2.0 ** -25)            # below eps: x * 1e6 * gamma
    np.testing.assert_allclose(y[0, 0, 2, c // 3], gamma[c // 3], rtol=1e-6)              # one-hot: gamma itself
