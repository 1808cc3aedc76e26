"""BGR, NV12 and I420 input (`-m gpu`): the pixel-format readers of the input staging.

* ``lumi_op_pixels_to_rgb`` equals the numpy restatement (tests/pixel_formats_ref.py, held to OpenCV by
  test_pixel_formats_host.py) on the frame holding every (Y, U, V) triple, and the channel flip on BGR.
* Every predict entry point on images in format F gives the bytes of the same call on their RGB conversions made on the
  host: boxes, scores, labels, counts and the ``conv_feature_map`` tap, for the eager, captured and replayed forward of
  each shape, with both pipeline halves in use.
* One engine switching formats never replays a graph of another format.
"""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import pixel_formats_ref as R
from luminoth_b200 import synth
from luminoth_b200.engine import PIXEL_FORMATS, Engine, load_library
from luminoth_b200.predicting import PredictorNetwork
from test_gpu_e2e import frcnn_cfg
from test_gpu_resize_input import assert_same, on_device, sources
from test_ssd_config_host import ssd_cfg


def pixels_to_rgb(image, fmt, h, w):
    """lumi_op_pixels_to_rgb on a device copy of ``image``; ValueError when the op refuses."""
    import torch
    lib = load_library()
    src = torch.from_numpy(np.ascontiguousarray(image)).cuda()
    dst = torch.empty((h, w, 3), dtype=src.dtype, device='cuda')
    rc = lib.lumi_op_pixels_to_rgb(ctypes.c_void_p(src.data_ptr()), PIXEL_FORMATS.get(fmt, fmt),
                                   int(src.dtype == torch.float32), h, w, ctypes.c_void_p(dst.data_ptr()), None)
    if rc != 0:
        raise ValueError(lib.lumi_op_last_error().decode())
    return dst.cpu().numpy()


def frames(fmt, sizes, seed, f32=False):
    """Images of the given pixel sizes in ``fmt`` and their RGB conversions."""
    if fmt in ('nv12', 'i420'):
        imgs = R.random_frames(sizes, seed)[fmt]
    else:
        imgs = sources(sizes, f32, seed)
    return imgs, [R.to_rgb(im, fmt) for im in imgs]


@pytest.mark.parametrize('fmt', ['nv12', 'i420'])
def test_op_yuv_equals_restatement_on_every_triple(fmt):
    frame = R.frame(*R.all_triples_planes(), fmt)
    np.testing.assert_array_equal(pixels_to_rgb(frame, fmt, 4096, 4096), R.to_rgb(frame, fmt))


def test_op_bgr_is_the_channel_flip():
    rng = np.random.default_rng(3)
    u8 = rng.integers(0, 256, (37, 53, 3), dtype=np.uint8)
    np.testing.assert_array_equal(pixels_to_rgb(u8, 'bgr', 37, 53), u8[..., ::-1])
    f32 = (rng.standard_normal((37, 53, 3)) * 400).astype(np.float32)       # non-integer, negative and > 255
    f32[0, 0] = [-0.5, 255.25, 1e6]
    np.testing.assert_array_equal(pixels_to_rgb(f32, 'bgr', 37, 53), f32[..., ::-1])
    np.testing.assert_array_equal(pixels_to_rgb(f32, 'rgb', 37, 53), f32)


def test_op_refuses_bad_yuv():
    for fmt in ('nv12', 'i420'):
        with pytest.raises(ValueError, match='even'):
            pixels_to_rgb(np.zeros((9, 9), np.uint8), fmt, 5, 9)
        with pytest.raises(ValueError, match='even'):
            pixels_to_rgb(np.zeros((9, 9), np.uint8), fmt, 6, 9)
        with pytest.raises(ValueError, match='uint8'):
            pixels_to_rgb(np.zeros((9, 8), np.float32), fmt, 6, 8)
    with pytest.raises(ValueError, match='unknown pixel format'):
        pixels_to_rgb(np.zeros((4, 4, 3), np.uint8), 7, 4, 4)


# ---------------------------------------------------------------- engine calls

FRCNN_HW = (224, 320)
# Sources of mixed sizes (even for YUV), resized to FRCNN_HW; odd counts, so the pipeline halves differ.
EVEN_SOURCES = [(160, 224), (150, 210), (224, 320), (2, 300), (300, 420), (96, 130), (480, 640)]
ODD_SOURCES = [(97, 131), (1, 300), (201, 299)]


@pytest.fixture(scope='module')
def frcnn():
    cfg = frcnn_cfg('resnet_v1_50')
    wts = synth.make_weights(cfg, seed=1)
    eng = Engine(cfg, max_batch=7, max_h=FRCNN_HW[0], max_w=FRCNN_HW[1])
    eng.load_weights(wts).finalize()
    yield eng
    eng.close()


def _same_as_rgb(eng, call, feed, rgb, fmt, tag):
    """call(feed, fmt) three times (eager, capture, replay) equals call(rgb, 'rgb'), with the conv_feature_map tap."""
    want = call(rgb, 'rgb')
    assert int(want[3].sum()) > 0, tag + ': the comparison must not be vacuous'
    tap = eng.get_tensor('conv_feature_map')
    for k in range(3):
        got = call(feed, fmt)
        assert_same(want, got, '%s call %d' % (tag, k))
        np.testing.assert_array_equal(eng.get_tensor('conv_feature_map'), tap, err_msg='%s call %d tap' % (tag, k))
    return want


@pytest.mark.parametrize('fmt', ['bgr', 'nv12', 'i420'])
def test_predict_dense_batch(frcnn, fmt):
    imgs, rgb = frames(fmt, [FRCNN_HW] * 3, seed=11)
    call = lambda batch, f: frcnn.predict_raw(batch, pixel_format=f)        # noqa: E731
    _same_as_rgb(frcnn, call, np.stack(imgs), np.stack(rgb), fmt, fmt + ' host')
    _same_as_rgb(frcnn, lambda b, f: frcnn.predict_raw(on_device([b])[0], pixel_format=f), np.stack(imgs),
                 np.stack(rgb), fmt, fmt + ' device')


def test_predict_f32_bgr(frcnn):
    imgs, rgb = frames('bgr', [FRCNN_HW] * 2, seed=12, f32=True)
    call = lambda batch, f: frcnn.predict_raw(batch, pixel_format=f)        # noqa: E731
    _same_as_rgb(frcnn, call, np.stack(imgs), np.stack(rgb), 'bgr', 'bgr f32 host')
    _same_as_rgb(frcnn, lambda b, f: frcnn.predict_raw(on_device([b])[0], pixel_format=f), np.stack(imgs),
                 np.stack(rgb), 'bgr', 'bgr f32 device')


@pytest.mark.parametrize('fmt', ['bgr', 'nv12', 'i420'])
def test_predict_resize_mixed_sizes(frcnn, fmt):
    sizes = EVEN_SOURCES if fmt != 'bgr' else EVEN_SOURCES[:4] + ODD_SOURCES
    imgs, rgb = frames(fmt, sizes, seed=13)
    call = lambda srcs, f: frcnn.predict_resize(srcs, *FRCNN_HW, pixel_format=f)     # noqa: E731
    _same_as_rgb(frcnn, call, imgs, rgb, fmt, fmt + ' resize host')
    _same_as_rgb(frcnn, lambda s, f: call(on_device(s), f), imgs, rgb, fmt, fmt + ' resize device')
    if fmt == 'bgr':
        imgs, rgb = frames(fmt, sizes, seed=14, f32=True)
        _same_as_rgb(frcnn, call, imgs, rgb, fmt, 'bgr f32 resize host')


@pytest.mark.parametrize('fmt', ['bgr', 'nv12', 'i420'])
def test_predict_sizes_packed_canvas(frcnn, fmt):
    imgs, rgb = frames(fmt, [(160, 224), (300, 420), (96, 130), (480, 640)], seed=15)
    targets = [(224, 320), (201, 299), (160, 224), (222, 222)]
    call = lambda srcs, f: frcnn.predict_sizes(srcs, targets, pixel_format=f)        # noqa: E731
    _same_as_rgb(frcnn, call, imgs, rgb, fmt, fmt + ' sizes host')
    _same_as_rgb(frcnn, lambda s, f: call(on_device(s), f), imgs, rgb, fmt, fmt + ' sizes device')


@pytest.mark.parametrize('fmt', ['nv12', 'i420'])
def test_predict_windows_at_odd_origins(frcnn, fmt):
    """Windows of a 1080 x 1920 frame starting at odd and even rows and columns: each reads the chroma of its
    source-frame position, so the windows' detections, the merge and the conv_feature_map tap (of the call's last
    forward) equal those of the RGB frame."""
    imgs, rgb = frames(fmt, [(1080, 1920)], seed=16)
    wins = [(0, 1, 1, 301, 421), (0, 101, 333, 300, 420), (0, 778, 1498, 302, 421), (0, 779, 1499, 301, 421),
            (0, 0, 0, 1080, 1920), (0, 0, 3, 224, 320), (0, 333, 0, 225, 321)]
    windows = [w + FRCNN_HW for w in wins]
    scales = [(224.0 / w[3], 320.0 / w[4]) for w in wins]
    for where, feed in (('host', imgs), ('device', on_device(imgs))):
        want = frcnn.predict_windows(rgb, windows, scales, 0.5)
        want_win = frcnn.last_window_detections()[:4]
        assert int(want_win[3].sum()) > 0, 'the comparison must not be vacuous'
        tap = frcnn.get_tensor('conv_feature_map')
        for k in range(3):
            got = frcnn.predict_windows(feed, windows, scales, 0.5, pixel_format=fmt)
            assert_same(want, got, '%s windows %s call %d' % (fmt, where, k))
            np.testing.assert_array_equal(frcnn.get_tensor('conv_feature_map'), tap,
                                          err_msg='%s windows %s call %d tap' % (fmt, where, k))
            assert_same(want_win, frcnn.last_window_detections()[:4], '%s windows %s call %d per window'
                        % (fmt, where, k))


def test_engine_refuses_bad_inputs(frcnn):
    want = frcnn.predict_raw(np.zeros((2,) + FRCNN_HW + (3,), np.uint8))
    with pytest.raises(ValueError, match='even'):
        frcnn.predict_resize([np.zeros((10, 8), np.uint8)], *FRCNN_HW, pixel_format='nv12')
    with pytest.raises(ValueError, match='uint8'):
        frcnn.predict_raw(np.zeros((2, 336, 320), np.float32), pixel_format='i420')
    with pytest.raises(ValueError, match='pixel_format'):
        frcnn.predict_raw(np.zeros((2,) + FRCNN_HW + (3,), np.uint8), pixel_format='yuyv')
    lib = load_library()
    assert lib.lumi_set_pixel_format(frcnn._h, 4) != 0
    assert 'unknown pixel format' in lib.lumi_last_error(frcnn._h).decode()
    # the C entry points check the format against the image on their own: float32 NV12, odd NV12 sizes
    assert lib.lumi_set_pixel_format(frcnn._h, 2) == 0
    frcnn._pixel_format = 2
    x = np.zeros((2, 336, 320), np.float32)
    out = [np.empty((2, frcnn.max_detections * 4), np.float32) for _ in range(4)]
    args = [ctypes.c_void_p(a.ctypes.data) for a in out]
    assert lib.lumi_predict_f32(frcnn._h, ctypes.c_void_p(x.ctypes.data), 0, 2, 224, 320, *args, 0) != 0
    assert 'uint8' in lib.lumi_last_error(frcnn._h).decode()
    y = np.zeros((2, 336, 321), np.uint8)
    assert lib.lumi_predict(frcnn._h, ctypes.c_void_p(y.ctypes.data), 0, 2, 224, 321, *args, 0) != 0
    assert 'even' in lib.lumi_last_error(frcnn._h).decode()
    assert_same(want, frcnn.predict_raw(np.zeros((2,) + FRCNN_HW + (3,), np.uint8)), 'after the refused calls')


def test_switching_formats_never_replays_another_formats_graph(frcnn):
    """RGB, NV12, BGR, RGB on one engine, each shape captured and replayed: every format gives its own RGB
    conversion's result, and the last RGB calls reproduce the first bit for bit."""
    rgb0 = np.stack(frames('bgr', [FRCNN_HW] * 2, seed=17)[0])
    nv12, nv12_rgb = frames('nv12', [FRCNN_HW] * 2, seed=18)
    bgr, bgr_rgb = frames('bgr', [FRCNN_HW] * 2, seed=19)
    want_nv12, want_bgr = frcnn.predict_raw(np.stack(nv12_rgb)), frcnn.predict_raw(np.stack(bgr_rgb))
    first = frcnn.predict_raw(rgb0)
    for k in range(2):
        assert_same(first, frcnn.predict_raw(rgb0), 'rgb call %d' % k)
    for k in range(3):
        assert_same(want_nv12, frcnn.predict_raw(np.stack(nv12), pixel_format='nv12'), 'nv12 call %d' % k)
    for k in range(3):
        assert_same(want_bgr, frcnn.predict_raw(np.stack(bgr), pixel_format='bgr'), 'bgr call %d' % k)
    assert_same(first, frcnn.predict_raw(rgb0), 'rgb again')
    assert frcnn.last_graph_replays > 0


@pytest.mark.parametrize('fmt', ['bgr', 'nv12'])
def test_ssd_from_camera_frames(fmt):
    cfg = ssd_cfg(300, 300)
    cfg['model']['proposals']['min_prob_threshold'] = 0.2
    eng = Engine(cfg, max_batch=3)
    eng.load_weights(synth.make_weights(cfg, seed=5)).finalize()
    imgs, rgb = frames(fmt, [(480, 640)] * 3, seed=20)
    call = lambda srcs, f: eng.predict_resize(srcs, 300, 300, pixel_format=f)       # noqa: E731
    want = call(rgb, 'rgb')
    assert int(want[3].sum()) > 0, 'the comparison must not be vacuous'
    for where, feed in (('host', imgs), ('device', on_device(imgs))):
        for k in range(3):
            assert_same(want, call(feed, fmt), 'ssd %s %s call %d' % (fmt, where, k))
    eng.close()


@pytest.mark.parametrize('fmt', ['bgr', 'nv12'])
def test_predictor_batch_and_tiled(fmt):
    """PredictorNetwork.predict_batch (the dense fast path and the resize path) and predict_tiled on frames in
    ``fmt`` return the predictions of the RGB conversions."""
    from luminoth_b200 import default_config
    cfg = default_config('fasterrcnn', ['model.base_network.architecture=resnet_v1_50', 'model.network.num_classes=20',
                                        'model.rpn.proposals.post_nms_top_n=100',
                                        'model.rcnn.proposals.min_prob_threshold=0.05',
                                        'dataset.image_preprocessing.min_size=160',
                                        'dataset.image_preprocessing.max_size=224'])
    net = PredictorNetwork(cfg, weights=synth.make_weights(cfg, seed=0), max_batch=4)
    imgs, rgb = frames(fmt, [(160, 224), (160, 224), (480, 640), (300, 200)], seed=21)
    want = net.predict_batch(rgb)
    assert sum(len(p) for p in want) > 0, 'the comparison must not be vacuous'
    assert net.predict_batch(imgs, pixel_format=fmt) == want
    big, big_rgb = frames(fmt, [(700, 1100), (500, 300)], seed=22)
    want = net.predict_tiled(big_rgb, 400)
    assert sum(len(p) for p in want) > 0, 'the comparison must not be vacuous'
    assert net.predict_tiled(big, 400, pixel_format=fmt) == want
    net.engine.close()
