"""The conv schedule at every SM budget (`-m gpu`, except the host checks).

Many launch decisions read the SM count: the persistent grid G = min(tiles, SMs - reserve), the stream-K partition of
the U = tiles x K-slices units into G ranges U b / G .. U (b + 1) / G (which CTA publishes a partial, which holds a
tile's head and how many partials the head adds), whether stream-K runs at all (last wave under 92 % full, at least 12
K slices and 12 units per CTA; forced: 3 units per CTA), the 128 x 256 tile rule (wide tiles >= 50 % of the budget),
the 2-CTA cluster pairs (sms / 2 units) and the NMS mask grid.  An H100 SXM reports 132 SMs, the PCIe card 114, MIG
slices 16 to 64, and a pipelined half-batch on a 16-SM slice gets 8.  `lumi_op_conv2d_sched` and
`Engine.set_sm_limit` run a smaller budget on any H100 (never a larger one: every CTA of a stream-K grid must be
resident, since the head CTA waits on flags of later CTAs).

* Host: a restatement of TcSched, the head CTA's fix-up walk and the launch decision.  Every stream-K tile is covered
  once, in CTA order, by its head and exactly the units the walk adds, and no CTA publishes two partials.  The GPU
  sweep's (shape, G) cases reach every partition pattern listed in SCHEDULE_PATTERNS, and budgets 114 and 16 change
  the kernel choice of some layer of the R50 and SSD plans (run with -s for the table).
* GPU sweep: ten launches (the RPN conv, block3 conv2, a 1x1 K = 1024 layer on four warpgroups, a wide-tile layer,
  SSD's conv8_1, which the engine runs on the wide tile only at budgets up to 66, resnet_v2 conv3 writing x and p or p
  only, the RCNN fp32 head, the 2-CTA pair kernel and a ragged few-tile layer) at G in G_VALUES below the device's
  count.  Whole-tile codes give the full-device bytes at every G; stream-K and engine
  codes meet the float64 bound of test_gpu_conv_numerics at sampled pixels and give the same bytes over three
  back-to-back launches on one workspace as over one.  Forced stream-K gives the whole-tile bytes where every range
  ends on a tile boundary; the engine's launch gives the bytes of the explicit code (tile width, stream-K or not) the
  restatement names at that budget.  Pair kernels below a budget of 2 return LUMI_EINVAL.
* GPU engines: R50 Faster R-CNN (bench's weights, 80 classes, four 600x800 photos, pipeline and graphs on) and SSD
  300x300 at batch 8 at budgets 114, 66, 16 and 8: with stream-K off the bytes of the full-device engine, eager and on
  replay; with the default stream-K one image of each pipeline half meets the fp32 and float64 oracle at 114 and 16,
  replays equal eager launches, and budget changes on one engine give a fresh engine's bytes at that budget.
"""
import collections
import ctypes
import zlib

import numpy as np
import pytest

import gpu_ops as G
from luminoth_b200.engine import LUMI_EINVAL
from test_gpu_baseline_configs import _assert_parity, _det_compare, _report
from test_gpu_conv_engine_layers import (LAYERS, PAD, Launch, _gather, _inputs, _row, check, out_geometry,
                                         preact_reference, reference, sample_pixels)
from test_gpu_conv_numerics import pick_tile


H100_SXM_SMS = 132
PIPELINE_RESERVE = 8                 # CONV_PIPELINE_SM_RESERVE
G_VALUES = [1, 2, 3, 5, 8, 13, 16, 31, 32, 60, 64, 66, 97, 114, 124, 131]
ENGINE_BUDGETS = [114, 66, 16, 8]
PLAN_BUDGETS = [132, 124, 114, 66, 16, 8]

# lumi_op_conv2d codes (include/luminoth_b200.h)
WHOLE_CODES = (1, 3, 4, 6, 12, 14)
STREAMK_CODES = {2: 1, 5: 4, 7: 6, 15: 14}          # forced stream-K code -> the same kernel on whole tiles
ENGINE_CODES = (16, 17, 18, 19)
PAIR_CODES = (6, 7)
RESERVED_CODES = (17, 19)
F32_CODES = (1, 2, 18, 19)


def cdiv(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------- the restatement
def sm_budget(limit, reserve=0, device=H100_SXM_SMS):
    """conv.cu sm_budget: min(limit, device) (limit 0: the device), less the reserve when it leaves an SM."""
    n = min(limit, device) if limit > 0 else device
    return n - reserve if 0 < reserve < n else n


def cout_pad(cout):
    p = cdiv(cout, 64) * 64
    return cdiv(cout, 128) * 128 if p > 64 and p % 128 else p


Plan = collections.namedtuple('Plan', 'bn pair m_tiles total n_iters units_max grid streamk eff upc')


def launch_plan(row, code, sms):
    """What launch_conv_tc / launch_tc_cfg launch for lumi_op_conv2d code `code` (16-19: the engine's own launch) of
    the row at an SM budget of `sms` (after any reserve).  Pairs: the budget below the device's cluster limit."""
    ho, wo, _, _ = out_geometry(row.h, row.w, row.k, row.stride, row.rate, row.padding)
    nb, th, tw = pick_tile(row.n, ho, wo)
    m_tiles = cdiv(row.n, nb) * cdiv(ho, th) * cdiv(wo, tw)
    n_iters = row.k * row.k * row.cin // 64
    cp = cout_pad(row.cout)
    f32_out = code in F32_CODES
    if code in ENGINE_CODES:
        wide_min, wide_pct = 16, 50
    else:
        wide_min, wide_pct = (1, 0) if code in (14, 15) else (0, 50)
    wide = (wide_min > 0 and cp % 256 == 0 and n_iters >= wide_min and not f32_out and not row.pre and
            m_tiles * (cp // 256) * 100 >= sms * wide_pct)
    bn = 256 if wide else 128 if cp % 128 == 0 else 64
    pair = code in PAIR_CODES and bn == 128 and not f32_out
    total = (cdiv(m_tiles, 2) if pair else m_tiles) * (cp // bn)
    units_max = sms // 2 if pair else sms
    mode = 2 if code in STREAMK_CODES else 1 if code in ENGINE_CODES else 0
    eff, upc, sk = 1.0, 0, False
    if mode and units_max:
        waves = total / units_max
        eff = waves / np.ceil(waves)
        upc = total * n_iters // units_max
        sk = (mode >= 2 and upc >= 3) or (eff < 0.92 and n_iters >= 12 and upc >= 12)
    grid = units_max if sk else min(total, units_max)
    return Plan(bn, pair, m_tiles, total, n_iters, units_max, grid, sk, eff, upc)


def cta_items(total, n_iters, g, b):
    """TcSched(mode 1).next: the (tile, k0, k1) items of scheduling unit b of g."""
    u, u_end = total * n_iters * b // g, total * n_iters * (b + 1) // g
    while u < u_end:
        tile = u // n_iters
        k0 = u - tile * n_iters
        k1 = min(n_iters, k0 + (u_end - u))
        yield tile, k0, k1
        u += k1 - k0


def range_end(unit, total, n_iters, g):
    return total * n_iters * (unit + 1) // g


def fixup_walk(total, n_iters, g, b, tile):
    """The units whose partials the head CTA b of `tile` adds, in order (conv_tc_kernel's stream-K fix-up)."""
    tile_end, out = (tile + 1) * n_iters, []
    for unit in range(b + 1, g):
        out.append(unit)
        if range_end(unit, total, n_iters, g) >= tile_end:
            break
    return out


def schedule(total, n_iters, g):
    """Every unit's items, checked: each tile's K slices are covered once in unit order by its head (k0 = 0) and the
    units the head's walk adds, and no unit publishes more than one partial (one slot per CTA).  U >= g: a unit with
    an empty range never publishes, and a head walking over it would wait forever (launch_tc_cfg runs stream-K only
    with at least 3 units per CTA)."""
    assert total * n_iters >= g, (total, n_iters, g)
    items = [list(cta_items(total, n_iters, g, b)) for b in range(g)]
    per_tile = collections.defaultdict(list)
    for b, its in enumerate(items):
        assert sum(1 for _, k0, _ in its if k0) <= 1 and all(k0 == 0 for _, k0, _ in its[1:]), (total, n_iters, g, b)
        for t, k0, k1 in its:
            per_tile[t].append((b, k0, k1))
    assert sorted(per_tile) == list(range(total))
    for t, parts in per_tile.items():
        assert parts[0][1] == 0 and parts[-1][2] == n_iters and all(
            a[2] == c[1] for a, c in zip(parts, parts[1:])), (total, n_iters, g, t, parts)
        if len(parts) > 1:
            assert fixup_walk(total, n_iters, g, parts[0][0], t) == [b for b, _, _ in parts[1:]], (total, n_iters, g, t)
    return items, per_tile


def explicit_code(code, plan):
    """The lumi_op_conv2d code that launches what engine code `code` launches under `plan`: the same kernel (fp32 or
    split outputs, 128 x 256 or narrower tiles, four warpgroups allowed) on whole tiles or forced stream-K."""
    if code in F32_CODES:
        return 2 if plan.streamk else 1
    if plan.bn == 256:
        return 15 if plan.streamk else 14
    return 5 if plan.streamk else 4


def whole_ranges(plan):
    """Stream-K on and every range ends on a tile boundary: no CTA writes a partial."""
    u = plan.total * plan.n_iters
    return plan.streamk and all(u * b // plan.grid % plan.n_iters == 0 for b in range(plan.grid + 1))


# ---------------------------------------------------------------------------------------------- the GPU sweep's cases
_BY = {r.name: r for r in LAYERS}
# name, row, codes: the whole-tile code first, then its stream-K code, then the engine's codes
SWEEP = [
    ('rpn_conv_3x3_1024', _BY['r50/rpn/conv'], (3, 5, 16, 17)),
    ('block3_conv2_3x3_256', _BY['r50/block3/unit_1/conv2'], (3, 5, 16, 17)),
    ('1x1_k1024_four_warpgroups', _BY['r50/block3/unit_2/conv1'], (4, 5, 16, 17)),
    ('wide_1x1_128_512_residual', _BY['r50/block2/unit_4/conv3'], (14, 15, 16)),
    ('ssd_conv8_1_wide_below_66', _BY['ssd/conv8_1'], (4, 5, 16, 17)),
    ('v2_conv3_x_and_p', _BY['r50_v2/block3/unit_1/conv3'], (3, 4, 5, 16, 17)),
    ('v2_conv3_p_only', _BY['r50_v2/block2/unit_4/conv3'], (3, 5, 16, 17)),
    ('rcnn_heads_fp32', _BY['r50/rcnn/heads'], (1, 2, 18, 19)),
    ('pair_3x3_ragged', _row('pair', 3, 37, 61, 256, 256, 3, act=1), (6, 7)),
    ('ragged_few_tiles_3x37x61', _row('ragged', 3, 37, 61, 128, 128, 3, act=1), (3, 5, 16, 17)),
]
SWEEP_IDS = [c[0] for c in SWEEP]


def sweep_cases(device=H100_SXM_SMS):
    """(shape name, row, code, G, plan) of every launch the GPU sweep makes at a budget below the device's."""
    for name, row, codes in SWEEP:
        for code in codes:
            for g in [v for v in G_VALUES if v < device] + [device]:
                sms = sm_budget(g, PIPELINE_RESERVE if code in RESERVED_CODES else 0, device)
                if code in PAIR_CODES and sms < 2:
                    continue
                yield name, row, code, g, launch_plan(row, code, sms)


def schedule_patterns(cases):
    found = collections.defaultdict(list)
    for name, row, code, g, plan in cases:
        key = '%s/code%d/G%d' % (name, code, g)
        if plan.total < plan.units_max:
            found['fewer tiles than CTAs'].append(key)
        if plan.pair and plan.m_tiles % 2:
            found['pairs on an odd number of M tiles'].append(key)
        if code in ENGINE_CODES and plan.bn == 256 and launch_plan(row, code, H100_SXM_SMS).bn != 256:
            found['wide tile only at the smaller budget'].append(key)
        if code in ENGINE_CODES and plan.n_iters >= 12 and plan.upc >= 12:
            if 0.88 <= plan.eff < 0.92:
                found['last wave just under 92 %'].append(key)
            if 0.92 <= plan.eff < 0.96:
                found['last wave just over 92 %'].append(key)
        if not plan.streamk:
            continue
        items, per_tile = schedule(plan.total, plan.n_iters, plan.grid)
        if plan.grid == 1:
            found['G = 1 with stream-K'].append(key)
        if code in STREAMK_CODES and plan.upc == 3:
            found['3 units per CTA (forced)'].append(key)
        if code in ENGINE_CODES and plan.upc == 12:
            found['12 units per CTA (auto)'].append(key)
        if whole_ranges(plan):
            found['every range on a tile boundary'].append(key)
        if any(len(p) >= 3 and any(k0 and k1 != plan.n_iters for _, k0, k1 in p) for p in per_tile.values()):
            found['a tile over 3 or more CTAs'].append(key)
        if any(len(its) >= 3 and its[0][1] != 0 and its[-1][2] != plan.n_iters for its in items):
            found['3 or more tiles in one range, partial at both ends'].append(key)
    return found


SCHEDULE_PATTERNS = ['a tile over 3 or more CTAs', '3 or more tiles in one range, partial at both ends',
                     'every range on a tile boundary', 'G = 1 with stream-K', '3 units per CTA (forced)',
                     '12 units per CTA (auto)', 'last wave just under 92 %', 'last wave just over 92 %',
                     'fewer tiles than CTAs', 'wide tile only at the smaller budget',
                     'pairs on an odd number of M tiles']


# ---------------------------------------------------------------------------------------------- host checks
def test_budget_rule():
    """The limit only lowers the count; the reserve applies to the limited count while it leaves an SM."""
    assert sm_budget(0) == 132 and sm_budget(0, 8) == 124 and sm_budget(500) == 132 and sm_budget(500, 8) == 124
    assert sm_budget(114) == 114 and sm_budget(114, 8) == 106 and sm_budget(16, 8) == 8 and sm_budget(8, 8) == 8
    assert sm_budget(1) == 1 and sm_budget(1, 8) == 1


def test_schedule_restatement_on_small_partitions():
    """Every partition of up to 9 tiles x 7 K slices over up to 20 CTAs with at least one unit each covers each tile
    once, in CTA order, by its head and the units of its fix-up walk."""
    for total in range(1, 10):
        for n_iters in range(1, 8):
            for g in range(1, min(20, total * n_iters) + 1):
                schedule(total, n_iters, g)


def test_sweep_reaches_every_schedule_pattern():
    """The GPU sweep's (shape, G) cases at 132 SMs produce every partition and decision pattern at least once."""
    found = schedule_patterns(list(sweep_cases()))
    for p in SCHEDULE_PATTERNS:
        print('%-52s %3d cases, e.g. %s' % (p, len(found[p]), found[p][:2]))
    missing = [p for p in SCHEDULE_PATTERNS if not found[p]]
    assert not missing, 'patterns no sweep case reaches: %s' % missing


def _plan_rows(prefix):
    return [r for r in LAYERS if r.name.startswith(prefix)]


@pytest.mark.parametrize('prefix', ['r50/', 'ssd/'])
def test_engine_plan_changes_with_the_budget(prefix):
    """Per layer of the R50 600x1024 and SSD 300x300 plans, which layers run stream-K (S) and which the 128 x 256 tile
    (W) at budgets 132 ... 8 (the SMs a launch may use); budgets 114 and 16 each change at least one layer's choice."""
    rows = _plan_rows(prefix)
    assert rows
    choice = {}
    print('\n%-40s %s' % ('layer', ' '.join('%5d' % b for b in PLAN_BUDGETS)))
    for r in rows:
        code = 18 if r.f32 else 16
        marks = []
        for b in PLAN_BUDGETS:
            p = launch_plan(r, code, b)
            choice[r.name, b] = (p.streamk, p.bn == 256)
            marks.append(('S' if p.streamk else '.') + ('W' if p.bn == 256 else '.'))
        print('%-40s %s' % (r.name, ' '.join('%5s' % m for m in marks)))
    for b in (114, 16):
        changed = [r.name for r in rows if choice[r.name, b] != choice[r.name, 132]]
        assert changed, '%s: budget %d changes no layer' % (prefix, b)


# ---------------------------------------------------------------------------------------------- GPU: the sweep
def device_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


class SchedLaunch(Launch):
    def run_sched(self, impl, sm_limit, launches=1):
        """lumi_op_conv2d_sched -> (rc, x output, pre-activation output); rc != 0 returns no outputs."""
        import torch
        r = self.row
        rh, rw, rs = (r.res[0], r.res[1], r.res[2]) if r.res else (0, 0, 1)
        xd, wd, sd, bd, rd = self.d
        args = [G._p(xd), r.n, r.h, r.w, r.cin, G._p(wd), r.k, r.k, r.cout, r.stride, r.rate, PAD[r.padding],
                G._p(sd), G._p(bd), G._p(rd), rh, rw, rs, r.act, impl, G._p(self.dpre[0]), G._p(self.dpre[1]),
                sm_limit, launches]
        ho, wo = ctypes.c_int(), ctypes.c_int()
        lib = G._lib()
        G._check(lib.lumi_op_conv2d_sched(*args, None, None, ctypes.byref(ho), ctypes.byref(wo), None))
        shape = (r.n, ho.value, wo.value, r.cout)
        y = None if r.pre == 'p_only' else torch.empty(shape, dtype=torch.float32, device='cuda')
        p = torch.empty(shape, dtype=torch.float32, device='cuda') if r.pre else None
        rc = lib.lumi_op_conv2d_sched(*args, G._p(y), G._p(p), ctypes.byref(ho), ctypes.byref(wo), None)
        torch.cuda.synchronize()
        return (rc, None, None) if rc else (rc, y, p)


def _same(a, b):
    import torch
    return all((u is None and v is None) or u.view(torch.int32).equal(v.view(torch.int32)) for u, v in zip(a, b))


@pytest.mark.gpu
@pytest.mark.parametrize('case', SWEEP, ids=SWEEP_IDS)
def test_schedule_sweep(case):
    name, row, codes = case
    dev = device_sms()
    budgets = [g for g in G_VALUES if g < dev] + [0]
    inputs = _inputs(row)
    x, w, scale, bias, res, pre = inputs
    launch = SchedLaunch(row, inputs)
    ho, wo, _, _ = out_geometry(row.h, row.w, row.k, row.stride, row.rate, row.padding)
    at = sample_pixels(row.n, ho, wo, zlib.crc32(name.encode()))
    rs = row.res[2] if row.res else 1
    ref, bound = reference(x, w, row.stride, row.padding, scale, bias, res, rs, row.act, codes[0], rate=row.rate, at=at)
    pref, pbound = preact_reference(ref, bound, *pre) if pre else (None, None)

    def within(tag, out):
        worst = 0.0
        for t, r_, b_, what in ((out[1], ref, bound, ''), (out[2], pref, pbound, '/p')):
            if t is not None:
                worst = max(worst, check(tag + what, _gather(t, at), r_, b_))
        return worst

    worst, full, runs = 0.0, {}, {}
    for code in codes:
        rc, y, p = launch.run_sched(code, 0)
        assert rc == 0, G._lib().lumi_op_last_error().decode()
        full[code] = (y, p)
        worst = max(worst, within('%s/code%d/device' % (name, code), (rc, y, p)))
    n_whole = 0
    for code in codes:
        reserve = PIPELINE_RESERVE if code in RESERVED_CODES else 0
        for g in budgets:
            tag = '%s/code%d/G%d' % (name, code, g)
            plan = launch_plan(row, code, sm_budget(g, reserve, dev))
            out = runs[code, g] = launch.run_sched(code, g)
            if code in PAIR_CODES and sm_budget(g, reserve, dev) < 2:
                assert out[0] == LUMI_EINVAL, '%s: a pair grid at budget %d was launched' % (tag, g)
                assert 'budget' in G._lib().lumi_op_last_error().decode()
                continue
            assert out[0] == 0, '%s: %s' % (tag, G._lib().lumi_op_last_error().decode())
            if code in WHOLE_CODES:
                assert _same(out[1:], full[code]), '%s: whole tiles differ from the full-device bytes' % tag
                continue
            worst = max(worst, within(tag, out))
            again = launch.run_sched(code, g, launches=3)
            assert again[0] == 0 and _same(out[1:], again[1:]), '%s: three launches differ from one' % tag
            if code in ENGINE_CODES:
                # the engine's choice is the explicit code the restatement names, at the same budget: same kernel,
                # same partition, same bytes
                named = explicit_code(code, plan)
                limit = sm_budget(g, reserve, dev)
                if (named, limit) not in runs:
                    runs[named, limit] = launch.run_sched(named, limit)
                assert _same(out[1:], runs[named, limit][1:]), '%s: differs from code %d at %d SMs' % (tag, named, limit)
            elif whole_ranges(plan):
                whole = STREAMK_CODES[code]
                if whole == 4 and plan.n_iters > 16:          # four warpgroups only up to 16 K slices: code 3's kernel
                    whole = 4 if 4 in full else 3
                if whole in full:
                    n_whole += 1
                    assert _same(out[1:], full[whole]), '%s: whole-tile ranges differ from code %d' % (tag, whole)
    print('%s: max err/bound %.3f over %d budgets, %d whole-range stream-K launches equal to whole tiles'
          % (name, worst, len(budgets), n_whole))
    _report('sm_budget/sweep/' + name, err_over_bound=worst, whole_range_launches=n_whole)


# ---------------------------------------------------------------------------------------------- GPU: engines
def _model(model):
    """(config, bench's weights, the predict call, batch, images compared: one per pipeline half, oracle pair)."""
    from luminoth_b200 import default_config, synth
    from luminoth_b200.engine import Engine
    if model == 'r50':
        from test_gpu_photo_sizes import _production, oracle_pair, target
        from test_gpu_resize_input import sources
        cfg, wts = _production('resnet_v1_50')
        hw = target((480, 640))
        srcs = sources([(480, 640)] * 4, False, seed=41)

        def make():
            eng = Engine(cfg, max_batch=4, max_h=hw[0], max_w=hw[1])
            return eng.load_weights(wts).finalize()

        return make, lambda e: e.predict_resize(srcs, *hw), (0, 3), lambda i: oracle_pair(cfg, wts, srcs[i], hw)
    from oracle import ssd as ossd
    cfg = default_config('ssd', [])
    wts = synth.make_weights(cfg, seed=0, profile='peaky')
    imgs = synth.make_images(8, 300, 300, seed=42)

    def make():
        return Engine(cfg, max_batch=8).load_weights(wts).finalize()

    return make, lambda e: e.predict_raw(imgs), (1, 6), lambda i: (ossd.forward(imgs[i], wts, cfg),
                                                                  ossd.forward(imgs[i], wts, cfg, dtype=np.float64))


def _three(eng, call, what):
    """Eager, captured and replayed forwards of one shape give the same bytes; returns the first."""
    outs = [call(eng) for _ in range(3)]
    assert eng.last_graph_replays > 0, what
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            np.testing.assert_array_equal(a, b, err_msg=what + ': a replay differs from the eager forward')
    return outs[0]


def _equal(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


@pytest.mark.gpu
@pytest.mark.parametrize('model', ['r50', 'ssd'])
def test_engine_whole_tiles_at_every_budget(model):
    """Stream-K off: the full-device bytes at every budget, eager and on replay, on one engine."""
    make, call, _, _ = _model(model)
    eng = make()
    eng.set_conv_streamk('off')
    base = _three(eng, call, '%s full device' % model)
    assert int(base[3].sum()) > 0, 'the comparison must not be vacuous'
    for b in ENGINE_BUDGETS:
        eng.set_sm_limit(b)
        assert _equal(_three(eng, call, '%s budget %d' % (model, b)), base), '%s: budget %d changed bytes' % (model, b)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize('model', ['r50', 'ssd'])
def test_engine_default_streamk_at_reduced_budgets(model):
    """Default stream-K at budgets 114 and 16 on fresh engines: replays equal eager forwards and one image of each
    pipeline half meets the fp32 and float64 oracle.  One engine switched between budgets (its graphs captured at
    the full budget first) gives the fresh engines' bytes at each, and the full-budget bytes again at the end."""
    make, call, picks, oracle = _model(model)
    eng = make()
    base = _three(eng, call, '%s full device' % model)
    fresh, results, oracles = {}, [], {}
    for b in (114, 16):
        e2 = make()
        e2.set_sm_limit(b)
        fresh[b] = out = _three(e2, call, '%s fresh engine at budget %d' % (model, b))
        e2.close()
        for i in picks:
            if i not in oracles:
                oracles[i] = oracle(i)
            ref, tru = (o['classification_prediction'] for o in oracles[i])
            boxes, scores, labels, counts = out
            r = _det_compare('sm_budget/%s/budget%d/img%d' % (model, b, i), boxes[i], scores[i], labels[i],
                             int(counts[i]), ref, tru, dict(image_index=i, sm_limit=b))
            print('%s budget %d image %d: boxes %.2e px from float64 (fp32 oracle %.2e px)'
                  % (model, b, i, r.get('boxes_px_engine_vs_oracle64', np.nan),
                     r.get('boxes_px_oracle32_vs_oracle64', np.nan)))
            results.append(('%s budget %d image %d' % (model, b, i), r))
    assert any(not _equal(fresh[b], base) for b in fresh), \
        '%s: no budget changed a bit, so the graph key of the budget is not exercised' % model
    for b in (114, 16, 0):
        eng.set_sm_limit(b)
        want = fresh.get(b, base)
        for call_no in range(3):
            assert _equal(call(eng), want), '%s: call %d at budget %d differs from a fresh engine' % (model, call_no, b)
    eng.close()
    for what, r in results:
        _assert_parity(r, what)
        assert r['detections_engine'] > 0, '%s: the comparison must not be vacuous' % what


@pytest.mark.gpu
def test_negative_sm_limit_is_rejected():
    from luminoth_b200 import default_config
    from luminoth_b200.engine import Engine
    eng = Engine(default_config('ssd', []), max_batch=1)
    with pytest.raises(ValueError, match='SM limit'):
        eng.set_sm_limit(-1)
    eng.close()
