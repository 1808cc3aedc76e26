"""Numpy restatement of the engine's pixel-format conversion (LUMI_PIXELS_*), the oracle of the pixel-format tests.

``yuv_to_rgb`` is OpenCV's BT.601 limited-range fixed-point formula (``cv2.cvtColor`` with COLOR_YUV2RGB_NV12 /
COLOR_YUV2RGB_I420); test_pixel_formats_host.py checks it against OpenCV on a frame holding every (Y, U, V) triple.
"""
import numpy as np


def yuv_to_rgb(Y, U, V):
    """(..., 3) uint8 RGB of equally shaped Y, U, V arrays: integer arithmetic only."""
    Y, U, V = (np.asarray(a, np.int64) for a in (Y, U, V))
    uu, vv = U - 128, V - 128
    yy = np.maximum(0, Y - 16) * 1220542 + (1 << 19)
    r = (yy + 1673527 * vv) >> 20
    g = (yy - 852492 * vv - 409993 * uu) >> 20
    b = (yy + 2116026 * uu) >> 20
    return np.clip(np.stack([r, g, b], axis=-1), 0, 255).astype(np.uint8)


def planes(frame, fmt):
    """The Y [h][w], U and V [h/2][w/2] planes of a (3h/2, w) NV12 or I420 frame."""
    frame = np.asarray(frame)
    h, w = frame.shape[0] * 2 // 3, frame.shape[1]
    flat = frame.reshape(-1)
    Y = flat[:h * w].reshape(h, w)
    q = (h // 2) * (w // 2)
    if fmt == 'nv12':
        uv = flat[h * w:].reshape(h // 2, w // 2, 2)
        return Y, uv[..., 0], uv[..., 1]
    return Y, flat[h * w:h * w + q].reshape(h // 2, w // 2), flat[h * w + q:].reshape(h // 2, w // 2)


def frame(Y, U, V, fmt):
    """The (3h/2, w) uint8 NV12 or I420 frame of the planes Y [h][w], U and V [h/2][w/2]."""
    h, w = Y.shape
    if fmt == 'nv12':
        chroma = np.stack([U, V], axis=-1).reshape(h // 2, w)
    else:
        chroma = np.concatenate([U.reshape(-1), V.reshape(-1)]).reshape(h // 2, w)
    return np.ascontiguousarray(np.concatenate([Y, chroma], axis=0), dtype=np.uint8)


def to_rgb(image, fmt):
    """The RGB image the engine sees for ``image`` in pixel format ``fmt`` ('rgb', 'bgr', 'nv12', 'i420')."""
    if fmt == 'rgb':
        return image
    if fmt == 'bgr':
        return np.ascontiguousarray(image[..., ::-1])
    Y, U, V = planes(image, fmt)
    up = lambda c: np.repeat(np.repeat(c, 2, axis=0), 2, axis=1)     # noqa: E731 -- chroma of each 2 x 2 block
    return yuv_to_rgb(Y, up(U), up(V))


def random_frames(sizes, seed):
    """Seeded (h, w) YUV planes, as {'nv12': [frames], 'i420': [frames]} of the same pixels."""
    rng = np.random.default_rng(seed)
    out = {'nv12': [], 'i420': []}
    for h, w in sizes:
        Y = rng.integers(0, 256, (h, w), dtype=np.uint8)
        U = rng.integers(0, 256, (h // 2, w // 2), dtype=np.uint8)
        V = rng.integers(0, 256, (h // 2, w // 2), dtype=np.uint8)
        for fmt in out:
            out[fmt].append(frame(Y, U, V, fmt))
    return out


def all_triples_planes():
    """Y [4096][4096], U and V [2048][2048] holding every (Y, U, V) triple: each 2 x 2 luma block shares one chroma
    sample, so chroma sample b (row-major) carries the pair (b // 64 // 256, b // 64 % 256) and its block the luma
    values 4 (b % 64) .. 4 (b % 64) + 3; the 64 blocks of a pair cover all 256 luma values."""
    b = np.arange(2048 * 2048, dtype=np.int64)
    pair, k = b // 64, b % 64
    U = (pair // 256).astype(np.uint8).reshape(2048, 2048)
    V = (pair % 256).astype(np.uint8).reshape(2048, 2048)
    base = (4 * k).reshape(2048, 2048)
    Y = np.empty((4096, 4096), np.uint8)
    for dy in range(2):
        for dx in range(2):
            Y[dy::2, dx::2] = base + 2 * dy + dx
    return Y, U, V
