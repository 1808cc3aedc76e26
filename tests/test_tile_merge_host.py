"""CPU-only: the list grouping of the cross-window merge (tests/tile_merge_ref.plan_groups, the restatement of
plan_window_merge that tests/test_gpu_tile_merge.py checks the merge statistics against) on hand-worked plans, and
the NMS path boundaries those GPU cases rely on, from the staged scan's shared-memory formula and from the library."""
import numpy as np
import pytest

from test_nms_path_host import _paths, _staged_max
from tile_merge_ref import list_lengths, nms_path, nms_words, plan_groups, staged_fits

INF = float('inf')


@pytest.mark.parametrize('lengths,groups', [
    ([], []),
    ([0, 0, 0], []),
    ([7], [(1, 7)]),
    # T = 10: the 5-list takes 10 // 5 = 2 lists (5 and 3, padded to 5), the 2-list is alone
    ([0, 5, 3, 0, 2], [(2, 5), (1, 2)]),
    # equal lengths: one group, in list order
    ([3, 3, 3], [(3, 3)]),
    # one long list next to many short ones: T // 100 = 1, then all 50 short ones in one group
    ([100] + [1] * 50, [(1, 100), (50, 1)]),
    # three lists of 4 096 are one group only when T >= 3 x 4 096
    ([4096, 4096, 4096], [(3, 4096)]),
    ([4096, 4095, 4096], [(2, 4096), (1, 4095)]),
    ([6000, 6000, 6000], [(3, 6000)]),
    # 5 000, 4 500 and 4 200 with 30 lists of 50: T = 15 200, 15 200 // 5 000 = 3, then the 30 short lists
    ([5000, 4500, 4200] + [50] * 30, [(3, 5000), (30, 50)]),
    ([6000] + [60] + [10] * 39, [(1, 6000), (40, 60)]),
    ([20000], [(1, 20000)]),
    # longest first, stable on the list index among equal lengths
    ([1, 4, 2, 4, 1, 1], [(3, 4), (3, 1)]),
])
def test_plan_groups_hand_worked(lengths, groups):
    assert plan_groups(lengths) == groups
    # every list with candidates lands in exactly one group, and no group holds more than T slots
    assert sum(p for p, _ in groups) == sum(1 for v in lengths if v)
    assert all(p * cap <= max(sum(lengths), 1) for p, cap in groups)


def test_list_lengths_counts_only_counted_rows():
    labels = np.array([[0, 2, 2, 1], [1, 1, -1, 5], [2, 0, 0, 0]], np.int32)
    counts = np.array([3, 2, 1], np.int32)
    # window 2 (source 1) counts one row; the rows past each count are never read
    assert list_lengths(labels, counts, [0, 0, 1], 2, 3).tolist() == [1, 2, 2, 0, 0, 1]


def test_nms_words_and_staged_limit():
    assert [nms_words(n) for n in (1, 64, 65, 128, 129, 4096, 12672, 12673)] == [2, 2, 2, 2, 4, 64, 198, 200]
    assert staged_fits(12672) and not staged_fits(12673)
    assert _staged_max() == 12672


def test_path_boundaries_of_the_gpu_cases():
    """The restatement's path for every (lists, cap, thr) the GPU merge cases take, equal to lumi_nms_path."""
    table = [((1, 4095, 0.5), 0), ((1, 4096, 0.5), 0), ((1, 12672, 0.5), 0), ((1, 12673, 0.5), 2),
             ((1, 20000, 0.5), 2), ((3, 4096, 0.5), 1), ((3, 6000, 0.5), 1), ((3, 5000, 0.5), 1),
             ((2, 4096, 0.5), 0), ((3, 4095, 0.5), 0), ((40, 60, 0.5), 0), ((30, 50, 0.5), 0),
             ((3, 4096, 0.0), 0), ((3, 4096, 1.0), 1), ((3, 4096, INF), 0), ((3, 12672, 0.7), 1),
             ((3, 12673, 0.7), 2), ((1, 12673, 0.0), 2), ((1, 12673, INF), 2)]
    for (p, n, t), want in table:
        assert nms_path(p, n, t) == want, (p, n, t)
    assert _paths([q for q, _ in table], None) == [w for _, w in table]
