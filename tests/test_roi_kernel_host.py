"""CPU-only: which ROI kernel instance the launcher starts (lumi_roi_kernel, the function launch_roi_pool dispatches
on) at the edges of its table, and the engine's check of the pooled size.

Codes: 0-2 the row-walk kernel at 6 / 5 / 4 resident CTAs per SM, 3-4 the column-walk kernel at 4 / 8 channels per
lane, 5-8 the cell kernel <8,4,4>, <8,4,8>, <8,1,8>, <4,1,8>, -1 no instance.  The crop is 2*pw rows x 2*ph columns
(quirk Q4).  Each table runs in a fresh interpreter because the library reads the LUMI_ROI_* variables once per
process."""
import json
import os
import subprocess
import sys

import pytest

from luminoth_b200 import config as C, engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS6, ROWS5, ROWS4, COLS4, COLS8, CELLS844, CELLS848, CELLS818, CELLS418 = range(9)
ENV_KEYS = ('LUMI_ROI_KERNEL', 'LUMI_ROI_MINB', 'LUMI_ROI_COLS_CPL', 'LUMI_ROI_CPL', 'LUMI_ROI_RB', 'LUMI_ROI_NW')


def _kernels(queries, env_over):
    import __graft_entry__ as g
    g.build()
    env = dict(os.environ)
    for k in ENV_KEYS:
        env.pop(k, None)
    env.update(env_over)
    code = ('import json, sys; sys.path.insert(0, %r)\n'
            'from luminoth_b200 import engine\n'
            'lib = engine.load_library()\n'
            'print(json.dumps([lib.lumi_roi_kernel(c, ph, pw) for c, ph, pw in json.loads(sys.argv[1])]))' % ROOT)
    out = subprocess.run([sys.executable, '-c', code, json.dumps(queries)], env=env, cwd=ROOT, capture_output=True,
                         text=True, check=True).stdout
    return json.loads(out.strip().splitlines()[-1])


def _check(table, env_over):
    got = _kernels([q for q, _ in table], env_over)
    bad = [(q, want, g) for (q, want), g in zip(table, got) if g != want]
    assert not bad, '%s: (c, ph, pw), wanted, got: %s' % (env_over, bad)


# (c, ph, pw): crop_h = 2 pw, crop_w = 2 ph
EDGES = {
    'square_7': (1024, 7, 7),      # crop 14 x 14: the row-walk kernel's home
    'crop_h_16': (256, 8, 8),      # crop_h 16, sum 32: the largest the row-walk kernel takes
    'crop_h_18': (256, 7, 9),      # crop_h 18, sum 32: too tall for the row walk, fits the 4-warp cell kernel
    'sum_34': (256, 9, 8),         # crop_h 16, sum 34: too many samples for one warp's lanes
    'wide_9x5': (1024, 5, 9),      # pooled_width 9, pooled_height 5: crop_h 18, sum 28
    'sum_64': (1024, 16, 16),      # the largest crop the cell kernels take
    'flat_64': (8, 31, 1),         # crop_h 2, sum 64
    'tall_64': (8, 1, 31),         # crop_h 62, sum 64
    'two': (8, 2, 2),
}
INVALID = [(256, 17, 16), (256, 16, 17), (1024, 0, 7), (1024, 7, 0), (1024, -1, 7), (12, 7, 7), (1028, 7, 7)]


def _table(expect):
    return [(EDGES[k], v) for k, v in expect.items()] + [(q, -1) for q in INVALID]


@pytest.mark.parametrize('env', [{}, {'LUMI_ROI_KERNEL': 'rows'}, {'LUMI_ROI_KERNEL': 'junk'},
                                 {'LUMI_ROI_MINB': '6'}, {'LUMI_ROI_MINB': '7'}])
def test_default_table(env):
    """The row-walk kernel wherever crop_h <= 16 and crop_h + crop_w <= 32, else the <8,4,4> cell kernel up to a
    sum of 32 and the <8,4,8> one up to 64."""
    _check(_table({'square_7': ROWS6, 'crop_h_16': ROWS6, 'crop_h_18': CELLS844, 'sum_34': CELLS848,
                   'wide_9x5': CELLS844, 'sum_64': CELLS848, 'flat_64': CELLS848, 'tall_64': CELLS848,
                   'two': ROWS6}), env)


@pytest.mark.parametrize('minb,code', [('5', ROWS5), ('4', ROWS4)])
def test_row_walk_occupancy(minb, code):
    _check(_table({'square_7': code, 'crop_h_16': code, 'crop_h_18': CELLS844, 'sum_34': CELLS848, 'two': code}),
           {'LUMI_ROI_MINB': minb})


@pytest.mark.parametrize('cpl,code', [(None, COLS4), ('4', COLS4), ('8', COLS8)])
def test_column_walk(cpl, code):
    """LUMI_ROI_KERNEL=cols: the column walk up to a sample sum of 32 whatever crop_h is, the cell kernels above."""
    env = {'LUMI_ROI_KERNEL': 'cols'}
    if cpl is not None:
        env['LUMI_ROI_COLS_CPL'] = cpl
    _check(_table({'square_7': code, 'crop_h_16': code, 'crop_h_18': code, 'sum_34': CELLS848, 'wide_9x5': code,
                   'sum_64': CELLS848, 'two': code}), env)


@pytest.mark.parametrize('extra,small,large', [
    ({}, CELLS844, CELLS848),
    ({'LUMI_ROI_NW': '8'}, CELLS848, CELLS848),
    ({'LUMI_ROI_RB': '1'}, CELLS818, CELLS818),
    ({'LUMI_ROI_RB': '1', 'LUMI_ROI_NW': '8'}, CELLS818, CELLS818),
    ({'LUMI_ROI_CPL': '4'}, CELLS418, CELLS418),
    ({'LUMI_ROI_CPL': '4', 'LUMI_ROI_RB': '1'}, CELLS418, CELLS418),
])
def test_cell_kernel(extra, small, large):
    """LUMI_ROI_KERNEL=cells: <8,4,4> while 4 rois x the samples fit its 128 threads (sum <= 32), else <8,4,8>;
    LUMI_ROI_RB=1 one roi per CTA, LUMI_ROI_CPL=4 four channels per lane."""
    env = {'LUMI_ROI_KERNEL': 'cells'}
    env.update(extra)
    _check(_table({'square_7': small, 'crop_h_16': small, 'crop_h_18': small, 'sum_34': large, 'wide_9x5': small,
                   'sum_64': large, 'flat_64': large, 'tall_64': large, 'two': small}), env)


def test_cells_setting_leaves_other_settings_out():
    """With the cell kernel forced, the row-walk and column-walk settings pick nothing."""
    _check(_table({'square_7': CELLS844, 'sum_34': CELLS848}),
           {'LUMI_ROI_KERNEL': 'cells', 'LUMI_ROI_MINB': '4', 'LUMI_ROI_COLS_CPL': '8'})


def _cfg(pw, ph):
    return C.default_config('fasterrcnn', ['model.base_network.architecture=resnet_v1_50',
                                           'model.rcnn.roi.pooled_width=%d' % pw,
                                           'model.rcnn.roi.pooled_height=%d' % ph])


@pytest.mark.parametrize('pw,ph', [(0, 7), (7, 0), (-1, 7), (17, 16), (16, 17), (32, 1)])
def test_engine_rejects_pooled_sizes_no_kernel_takes(pw, ph):
    """A ValueError from the config check, before any device is touched."""
    with pytest.raises(ValueError, match='pooled_width and pooled_height'):
        engine.Engine(_cfg(pw, ph))


@pytest.mark.parametrize('pw,ph', [(7, 7), (9, 5), (16, 16), (31, 1), (1, 1)])
def test_engine_accepts_pooled_sizes(pw, ph):
    """Without a GPU the engine then stops at the device, not at the config."""
    try:
        eng = engine.Engine(_cfg(pw, ph))
    except RuntimeError as e:
        assert 'pooled' not in str(e)
    else:
        eng.close()
