"""Sliced prediction without a GPU: the window grid, the argument checks of ``predict_tiled`` and ``lumi predict
--tile`` that come before any device call, and the numpy restatement of the cross-window merge."""
import itertools

import numpy as np
import pytest

from luminoth_b200 import default_config, predict
from luminoth_b200.predicting import PredictorNetwork, tile_grid
from tile_merge_ref import map_boxes, merge_windows


def _cover(h, w, wins):
    c = np.zeros((h, w), np.int32)
    for y0, x0, wh, ww in wins:
        c[y0:y0 + wh, x0:x0 + ww] += 1
    return c


@pytest.mark.parametrize('h,w,th,tw,ov', [
    (4000, 6000, 600, 600, 0.2), (1000, 1000, 600, 600, 0.2), (700, 1100, 400, 400, 0.2), (1300, 500, 400, 400, 0.0),
    (601, 1199, 600, 600, 0.5), (37, 53, 10, 7, 0.3), (1, 1000, 300, 300, 0.2), (1000, 1, 300, 300, 0.2),
    (1, 1, 5, 5, 0.2), (10, 10, 1, 1, 0.0), (10, 10, 3, 3, 0.9)])
def test_tile_grid_covers_unique_inside(h, w, th, tw, ov):
    wins = tile_grid(h, w, th, tw, ov)
    assert len(set(wins)) == len(wins)
    for y0, x0, wh, ww in wins:
        assert 0 <= y0 and 0 <= x0 and y0 + wh <= h and x0 + ww <= w
        assert (wh, ww) == (min(th, h), min(tw, w))
    assert (_cover(h, w, wins) >= 1).all()
    # every border is touched by a window flush with it
    assert min(y for y, _, _, _ in wins) == 0 and min(x for _, x, _, _ in wins) == 0
    assert max(y + wh for y, _, wh, _ in wins) == h and max(x + ww for _, x, _, ww in wins) == w


def test_tile_grid_steps_and_overlap():
    wins = tile_grid(4000, 6000, 600, 600, 0.2)
    ys = sorted(set(y for y, _, _, _ in wins))
    xs = sorted(set(x for _, x, _, _ in wins))
    assert ys == list(range(0, 3400, 480)) + [3400]
    assert xs == list(range(0, 5400, 480)) + [5400]
    assert len(wins) == len(ys) * len(xs) == 9 * 13
    # neighbours overlap by tile - step = 120 px, the last pair by more
    assert all(b - a == 480 for a, b in zip(xs[:-2], xs[1:-1]))
    assert 0 < xs[-1] - xs[-2] <= 480
    assert tile_grid(1000, 1000, 600, 600, 0.99)[:2] == [(0, 0, 600, 600), (0, 6, 600, 600)]   # step at least 1


def test_tile_grid_small_images_are_one_window():
    assert tile_grid(500, 400, 600, 600, 0.2) == [(0, 0, 500, 400)]
    assert tile_grid(600, 600, 600, 600, 0.2) == [(0, 0, 600, 600)]
    assert tile_grid(1, 1, 600, 600, 0.2) == [(0, 0, 1, 1)]
    assert tile_grid(1, 2000, 600, 600, 0.2) == [(0, x, 1, 600) for x in [0, 480, 960, 1400]]


@pytest.mark.parametrize('args', [(0, 10, 5, 5, 0.2), (10, 0, 5, 5, 0.2), (10, 10, 0, 5, 0.2), (10, 10, 5, -1, 0.2),
                                  (10, 10, 5, 5, 1.0), (10, 10, 5, 5, -0.1)])
def test_tile_grid_rejects(args):
    with pytest.raises(ValueError):
        tile_grid(*args)


class _Stub(PredictorNetwork):
    """A PredictorNetwork without an engine: only the host-side steps run."""

    def __init__(self, config):
        self.config = config
        self.class_labels = None

        class _E:
            def predict_windows(self, *a, **k):
                raise AssertionError('no device call expected')
        self.engine = _E()


def test_tile_windows_targets_and_full_image():
    cfg = default_config('fasterrcnn', [])
    net = _Stub(cfg)
    wins, scales = net.tile_windows((4000, 6000, 3), 600, 0.2, True)
    assert len(wins) == 9 * 13 + 1
    assert wins[0] == (0, 0, 600, 600, 600, 600) and scales[0] == (1.0, 1.0)
    assert wins[-1][:4] == (0, 0, 4000, 6000) and wins[-1][4:] == (682, 1024)
    assert scales[-1][0] == scales[-1][1] == np.float32(1024) / np.float32(6000)
    wins, _ = net.tile_windows((4000, 6000, 3), 600, 0.2, False)
    assert len(wins) == 9 * 13
    wins, _ = net.tile_windows((500, 400, 3), 600, 0.2, True)
    assert [w_[:4] for w_ in wins] == [(0, 0, 500, 400)]                  # no duplicate of the whole image
    ssd = _Stub(default_config('ssd', []))
    wins, scales = ssd.tile_windows((900, 900, 3), 600, 0.2, False)
    assert all(w_[4:] == (300, 300) for w_ in wins)
    assert scales[0] == (np.float32(300) / np.float32(600),) * 2


def test_merge_threshold_defaults():
    assert _Stub(default_config('fasterrcnn', [])).merge_iou_threshold() == 0.5
    assert _Stub(default_config('fasterrcnn', ['model.network.with_rcnn=false'])).merge_iou_threshold() == 0.7
    assert _Stub(default_config('ssd', [])).merge_iou_threshold() == pytest.approx(0.45)


@pytest.mark.parametrize('images,kw', [
    ([np.zeros((10, 10), np.uint8)], {'tile': 5}),
    ([np.zeros((10, 10, 4), np.uint8)], {'tile': 5}),
    ([np.zeros((10, 10, 3), np.uint8)], {'tile': 0}),
    ([np.zeros((10, 10, 3), np.uint8)], {'tile': 5, 'overlap': 1.0}),
    ([np.zeros((10, 10, 3), np.uint8)], {'tile': (5, -2)}),
])
def test_predict_tiled_rejects_before_the_device(images, kw):
    with pytest.raises(ValueError):
        _Stub(default_config('fasterrcnn', [])).predict_tiled(images, **kw)


def test_predict_tiled_empty_list():
    assert _Stub(default_config('fasterrcnn', [])).predict_tiled([], 600) == []


@pytest.mark.parametrize('argv,msg', [(['--tile', '0'], '--tile must be'), (['--tile', '600', '--tile-overlap', '1'],
                                                                            '--tile-overlap'),
                                      (['--tile', '600', '--tile-overlap', '-0.5'], '--tile-overlap')])
def test_cli_tile_rejects(argv, msg, tmp_path):
    with pytest.raises(SystemExit) as ei:
        predict.main([str(tmp_path / 'x.jpg')] + argv)
    assert msg in str(ei.value)


def test_cli_tile_rejects_video(tmp_path):
    v = tmp_path / 'clip.mp4'
    v.write_bytes(b'')
    with pytest.raises(SystemExit) as ei:
        predict.main([str(v), '--tile', '600', '-c', 'unused.yml'])
    assert 'video' in str(ei.value)


# ---- the numpy merge restatement on hand-built window detections
def _dets(rows, k=4):
    """rows: per window a list of (x1, y1, x2, y2, score, label) -> padded arrays as the engine returns them."""
    n = len(rows)
    b = np.zeros((n, k, 4), np.float32)
    s = np.zeros((n, k), np.float32)
    lab = np.full((n, k), -1, np.int32)
    c = np.zeros((n,), np.int32)
    for i, r in enumerate(rows):
        for j, (x1, y1, x2, y2, sc, lb) in enumerate(r):
            b[i, j] = (x1, y1, x2, y2); s[i, j] = sc; lab[i, j] = lb
        c[i] = len(r)
    return b, s, lab, c


def test_map_boxes_is_float32_division_then_offset():
    b = np.array([[1.0, 2.0, 3.0, 4.0]], np.float32)
    m = map_boxes(b, (100, 200, np.float32(0.3), np.float32(0.7)))
    assert m.dtype == np.float32
    assert m[0, 0] == np.float32(np.float32(1.0) / np.float32(0.7)) + np.float32(200)
    assert m[0, 3] == np.float32(np.float32(4.0) / np.float32(0.3)) + np.float32(100)


def test_merge_identical_boxes_from_two_windows():
    # the same object seen by two windows whose origins differ: identical in source pixels, the first window wins a tie
    b, s, lab, c = _dets([[(10, 10, 20, 20, 0.9, 0)], [(0, 10, 10, 20, 0.9, 0)]])
    wmap = [(0, 0, 1, 1), (0, 10, 1, 1)]
    (ob, os_, ol), = merge_windows(b, s, lab, c, [0, 0], wmap, 1, 2, 10, 10, 0.5)
    assert ob.tolist() == [[10, 10, 20, 20]] and os_.tolist() == [np.float32(0.9)] and ol.tolist() == [0]


def test_merge_score_ties_across_windows_and_labels():
    b, s, lab, c = _dets([[(0, 0, 10, 10, 0.5, 1), (50, 50, 60, 60, 0.5, 0)],
                          [(100, 0, 110, 10, 0.5, 0), (0, 100, 10, 110, 0.5, 1)]])
    (ob, os_, ol), = merge_windows(b, s, lab, c, [0, 0], [(0, 0, 1, 1)] * 2, 1, 2, 10, 10, 0.5)
    # label-major on ties, then window order within a label
    assert ol.tolist() == [0, 0, 1, 1]
    assert ob[:, 0].tolist() == [50, 100, 0, 0] and ob[:, 1].tolist() == [50, 0, 0, 100]


def test_merge_iou_exactly_at_threshold_is_kept():
    # boxes of area 100 overlapping by 50: IoU = 50 / 150 = 1/3 in float32; suppression needs IoU > thr
    b, s, lab, c = _dets([[(0, 0, 10, 10, 0.9, 0)], [(5, 0, 15, 10, 0.8, 0)]])
    iou = np.float32(50) / np.float32(150)
    kw = dict(win_src=[0, 0], wmap=[(0, 0, 1, 1)] * 2, nsrc=1, nc=1, class_max=10, total_max=10)
    assert len(merge_windows(b, s, lab, c, thr=float(iou), **kw)[0][0]) == 2
    assert len(merge_windows(b, s, lab, c, thr=float(np.nextafter(iou, np.float32(0))), **kw)[0][0]) == 1


def test_merge_caps():
    rows = [[(i * 20, 0, i * 20 + 10, 10, 0.9 - 0.01 * i, i % 2) for i in range(4)] for _ in range(1)]
    rows.append([(200 + i * 20, 0, 210 + i * 20, 10, 0.5 - 0.01 * i, i % 2) for i in range(4)])
    b, s, lab, c = _dets(rows)
    kw = dict(win_src=[0, 0], wmap=[(0, 0, 1, 1)] * 2, nsrc=1, nc=2, thr=0.5)
    (ob, os_, ol), = merge_windows(b, s, lab, c, class_max=3, total_max=10, **kw)
    assert ol.tolist().count(0) == 3 and ol.tolist().count(1) == 3          # class_max per label
    (ob, os_, ol), = merge_windows(b, s, lab, c, class_max=10, total_max=5, **kw)
    assert len(ob) == 5 and (np.diff(os_) <= 0).all()                        # total_max, by score
    assert os_.tolist() == sorted(s[:, :4].ravel().tolist(), reverse=True)[:5]


def test_merge_empty_windows_and_sources():
    b, s, lab, c = _dets([[], [(0, 0, 10, 10, 0.7, 2)], []])
    out = merge_windows(b, s, lab, c, [0, 0, 2], [(0, 0, 1, 1)] * 3, 3, 3, 5, 5, 0.5)
    assert [len(o[0]) for o in out] == [1, 0, 0]
    assert out[0][2].tolist() == [2]


def test_merge_maps_to_source_pixels_per_window():
    b, s, lab, c = _dets([[(0, 0, 60, 30, 0.9, 0)], [(0, 0, 60, 30, 0.8, 0)]])
    sc = np.float32(0.5)
    (ob, _, _), = merge_windows(b, s, lab, c, [0, 0], [(0, 0, sc, sc), (300, 400, sc, sc)], 1, 1, 5, 5, 0.5)
    assert ob.tolist() == [[0, 0, 120, 60], [400, 300, 520, 360]]


def test_merge_greedy_order_within_label():
    # a suppressed box does not suppress others: A (0.9) suppresses B (0.8), B would have suppressed C (0.7)
    b, s, lab, c = _dets([[(0, 0, 10, 10, 0.9, 0), (4, 0, 14, 10, 0.8, 0), (8, 0, 18, 10, 0.7, 0)]])
    (ob, os_, _), = merge_windows(b, s, lab, c, [0], [(0, 0, 1, 1)], 1, 1, 5, 5, 0.3)
    assert os_.tolist() == [np.float32(0.9), np.float32(0.7)]


def test_merge_many_random_lists_are_sorted_and_capped():
    rng = np.random.RandomState(0)
    nwin, k, nc = 6, 20, 4
    b = np.sort(rng.uniform(0, 100, (nwin, k, 4)).astype(np.float32).reshape(nwin, k, 2, 2), axis=2).reshape(nwin, k, 4)
    b = b[:, :, [0, 2, 1, 3]]
    s = rng.choice(np.float32([0.25, 0.5, 0.75]), (nwin, k)).astype(np.float32)
    lab = rng.randint(0, nc, (nwin, k)).astype(np.int32)
    c = rng.randint(0, k + 1, nwin).astype(np.int32)
    out = merge_windows(b, s, lab, c, [0, 1, 0, 1, 0, 1], [(0, 0, 1, 1)] * nwin, 2, nc, 7, 12, 0.4)
    for ob, os_, ol in out:
        assert len(ob) <= 12 and (np.diff(os_) <= 0).all()
        for lb in range(nc):
            assert (ol == lb).sum() <= 7
        for (i, j) in itertools.combinations(range(len(ob)), 2):
            assert not (ol[i] == ol[j] and (ob[i] == ob[j]).all())
