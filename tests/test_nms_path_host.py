"""CPU-only: the NMS path decision (lumi_nms_path, the function run_nms dispatches on) at the edges of its table.

0: one-phase staged scan, 1: two-phase NMS, 2: one-phase unstaged scan.  Each table runs in a fresh interpreter
because the library reads LUMI_NMS_LAZY once per process."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INF = float('inf')

STAGED, TWO_PHASE, UNSTAGED = 0, 1, 2


def _staged_max():
    """The longest list the staged scan takes: its shared memory (removed words + two chunks of 64 mask rows, the
    row length rounded up to an even number of u64 words) must fit in 200 KiB."""
    def fits(n):
        words = (-(-n // 64) + 1) & ~1
        return (words + 2 * 64 * words) * 8 <= 200 * 1024
    n = 64
    while fits(n + 64):
        n += 64
    while fits(n + 1):
        n += 1
    return n


def _paths(queries, lazy_env):
    import __graft_entry__ as g
    g.build()
    env = dict(os.environ)
    env.pop('LUMI_NMS_LAZY', None)
    if lazy_env is not None:
        env['LUMI_NMS_LAZY'] = lazy_env
    code = ('import json, sys; sys.path.insert(0, %r)\n'
            'from luminoth_b200 import engine\n'
            'lib = engine.load_library()\n'
            'print(json.dumps([lib.lumi_nms_path(p, n, t) for p, n, t in json.loads(sys.argv[1])]))' % ROOT)
    out = subprocess.run([sys.executable, '-c', code, json.dumps(queries)], env=env, cwd=ROOT, capture_output=True,
                         text=True, check=True).stdout
    return json.loads(out.strip().splitlines()[-1])


def _check(table, lazy_env):
    got = _paths([q for q, _ in table], lazy_env)
    bad = [(q, want, g) for (q, want), g in zip(table, got) if g != want]
    assert not bad, 'LUMI_NMS_LAZY=%s: (problems, ncap, thr), wanted, got: %s' % (lazy_env, bad)


@pytest.mark.parametrize('lazy_env', [None, '', 'junk'])
def test_default_table(lazy_env):
    """LUMI_NMS_LAZY unset: two-phase from 3 lists on.  Set to anything atoi reads as 0: never two-phase."""
    hi = _staged_max()                       # 12 672: pre_nms_top_n 12 000 stays staged, 20 000 does not
    auto = TWO_PHASE if lazy_env is None else STAGED
    table = [
        ((3, 4095, 0.7), STAGED), ((3, 4096, 0.7), auto), ((3, hi, 0.7), auto), ((3, hi + 1, 0.7), UNSTAGED),
        ((2, 4096, 0.7), STAGED), ((2, hi, 0.7), STAGED), ((2, hi + 1, 0.7), UNSTAGED),
        ((1, 12000, 0.7), STAGED), ((1, 20000, 0.7), UNSTAGED), ((1, 1, 0.7), STAGED),
        ((8, 12000, 0.7), auto), ((160, 8096, 0.45), auto), ((640, 2000, 0.5), STAGED),
        ((3, 4096, 0.0), STAGED), ((3, 4096, 1.0), auto), ((3, 4096, INF), STAGED), ((3, 4096, -0.5), STAGED),
        ((3, 4096, float('nan')), STAGED), ((3, 4096, 1e-30), auto),
        ((3, hi + 1, 0.0), UNSTAGED), ((3, hi + 1, INF), UNSTAGED), ((8, 20000, 0.7), UNSTAGED),
    ]
    _check(table, lazy_env)


def test_forced_on_and_off():
    hi = _staged_max()
    on = [((1, 4096, 0.7), TWO_PHASE), ((2, hi, 0.5), TWO_PHASE), ((1, 4095, 0.7), STAGED),
          ((1, hi + 1, 0.7), UNSTAGED), ((1, 4096, 0.0), STAGED), ((1, 4096, INF), STAGED), ((3, 4096, 1.0), TWO_PHASE)]
    _check(on, '1')
    off = [((3, 4096, 0.7), STAGED), ((8, 12000, 0.7), STAGED), ((3, hi + 1, 0.7), UNSTAGED)]
    _check(off, '0')
