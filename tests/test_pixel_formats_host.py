"""Pixel formats without a device: the numpy YUV restatement against OpenCV, and the Python shape and dtype rules.

The restatement (tests/pixel_formats_ref.py) is the oracle of tests/test_gpu_pixel_formats.py, so it is held to
``cv2.cvtColor`` here on a frame that holds every (Y, U, V) triple, for NV12 and for I420.
"""
import numpy as np
import pytest

import pixel_formats_ref as R
from luminoth_b200 import engine as E
from luminoth_b200 import predicting as P


def test_all_triples_frame_holds_every_triple():
    Y, U, V = R.all_triples_planes()
    up = lambda c: np.repeat(np.repeat(c, 2, axis=0), 2, axis=1)     # noqa: E731
    code = (Y.astype(np.int64) << 16) | (up(U).astype(np.int64) << 8) | up(V)
    assert np.unique(code).size == 256 ** 3


@pytest.mark.parametrize('fmt', ['nv12', 'i420'])
def test_restatement_equals_opencv(fmt):
    cv2 = pytest.importorskip('cv2', reason='OpenCV is not installed: the YUV restatement is not checked against it')
    frame = R.frame(*R.all_triples_planes(), fmt)
    code = {'nv12': cv2.COLOR_YUV2RGB_NV12, 'i420': cv2.COLOR_YUV2RGB_I420}[fmt]
    np.testing.assert_array_equal(R.to_rgb(frame, fmt), cv2.cvtColor(frame, code))


def test_frame_layouts_round_trip():
    fr = R.random_frames([(6, 10)], seed=0)
    for fmt in ('nv12', 'i420'):
        f = fr[fmt][0]
        assert f.shape == (9, 10) and f.dtype == np.uint8
        Y, U, V = R.planes(f, fmt)
        np.testing.assert_array_equal(R.frame(Y, U, V, fmt), f)
    Yn, Un, Vn = R.planes(fr['nv12'][0], 'nv12')
    Yi, Ui, Vi = R.planes(fr['i420'][0], 'i420')
    for a, b in ((Yn, Yi), (Un, Ui), (Vn, Vi)):
        np.testing.assert_array_equal(a, b)


def test_pixel_size_of_each_format():
    assert E.pixel_size((1080, 1920, 3), 'rgb') == (1080, 1920)
    assert E.pixel_size((1080, 1920, 3), 'bgr', uint8=False) == (1080, 1920)
    assert E.pixel_size((1620, 1920), 'nv12') == (1080, 1920)
    assert E.pixel_size((3, 2), 'i420') == (2, 2)
    assert [E.pixel_format_code(f) for f in ('rgb', 'bgr', 'nv12', 'i420')] == [0, 1, 2, 3]


@pytest.mark.parametrize('fmt', ['nv12', 'i420'])
def test_bad_yuv_images_are_refused(fmt):
    with pytest.raises(ValueError, match='even height'):
        E.pixel_size((1621, 1920), fmt)          # h = 1080.67: not a frame of an even height
    with pytest.raises(ValueError, match='even height'):
        E.pixel_size((7, 8), fmt)                # an odd height (5 rows of Y would take 7.5 rows)
    with pytest.raises(ValueError, match='even height'):
        E.pixel_size((6, 9), fmt)                # an odd width
    with pytest.raises(ValueError, match='even height'):
        E.pixel_size((6, 8, 3), fmt)             # an RGB-shaped array
    with pytest.raises(ValueError, match='uint8'):
        E.pixel_size((6, 8), fmt, uint8=False)


def test_bad_formats_and_rgb_shapes_are_refused():
    with pytest.raises(ValueError, match='pixel_format'):
        E.pixel_format_code('yuyv')
    with pytest.raises(ValueError, match='BGR'):
        E.pixel_size((6, 8), 'bgr')
    # the RGB messages the predictor gave before pixel formats existed
    with pytest.raises(ValueError, match=r'expected an \(H, W, 3\) RGB image'):
        P._pixel_sizes([np.zeros((6, 8), np.uint8)], 'rgb')
    assert P._pixel_sizes([np.zeros((9, 8), np.uint8)], 'nv12') == [(6, 8)]
    with pytest.raises(ValueError, match='uint8'):
        P._pixel_sizes([np.zeros((9, 8), np.float32)], 'i420')


def test_predictor_passes_the_pixel_size_and_format():
    """predict_batch_raw: targets from the pixel size, the uint8 fast path on NV12 frames of the target size, and the
    keyword reaches the engine only for formats other than RGB."""
    calls = []

    class FakeEngine(object):
        max_batch = 4

        def predict_raw(self, batch, **kw):
            calls.append(('raw', batch.shape, kw))
            n = len(batch)
            return np.zeros((n, 1, 4), np.float32), np.ones((n, 1), np.float32), np.zeros((n, 1), np.int32), \
                np.ones(n, np.int32)

        def predict_resize(self, srcs, h, w, **kw):
            calls.append(('resize', (h, w), kw))
            return self.predict_raw(np.zeros((len(srcs), 1, 1, 3)), **kw)

    net = P.PredictorNetwork.__new__(P.PredictorNetwork)
    net.config = {'dataset': {'image_preprocessing': {'min_size': 600, 'max_size': 1024}}}
    net.engine, net.class_labels, net.pack_sizes = FakeEngine(), None, False
    frames = [np.zeros((900, 800), np.uint8)] * 2                # 600 x 800: its own target size
    net.predict_batch_raw(frames, pixel_format='nv12')
    assert calls == [('raw', (2, 900, 800), {'pixel_format': 'nv12'})]
    del calls[:]
    out = net.predict_batch_raw([np.zeros((450, 600), np.uint8)], pixel_format='i420')     # 300 x 600 -> 600 x 1200
    assert calls[0] == ('resize', (600, 1200), {'pixel_format': 'i420'})
    assert out[0][3] == 2.0
    del calls[:]
    net.predict_batch_raw([np.zeros((600, 800, 3), np.uint8)])
    assert calls == [('raw', (1, 600, 800, 3), {})]
