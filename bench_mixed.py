"""Mixed-size benchmark: PredictorNetwork.predict_batch_raw on a batch of photos of different sizes, packing off vs on.

bench.py times full batches of one size.  The callers that matter most (`lumi predict` on a folder, the web server's
micro-batcher, `lumi eval`) see mixed sizes: without packing a batch runs as one engine call per size bucket.  This
script times both groupings end to end, alternated, `--runs` runs each, on one engine (Faster R-CNN ResNet-50 as
bench.py's frcnn_r50, max_batch 8, host uint8 images):

  photos     480x640, 640x480, 427x640, 640x427, 375x500, 500x375, 612x612, 480x640 (six target sizes)
  landscape  480x640 x3, 427x640 x3, 612x612 x2 -> three target sizes, all landscape or square
  uniform    8 x 480x640: one target size, the same engine call both ways (the control)

Per workload it prints one JSON line: images/s (median, min, max over the runs) of each grouping, engine calls and
kernel launches per predict_batch_raw call, the band clear's share of the packed forward's device time (a separate
profiled call), and how far the packed results are from the unpacked ones (identical counts and labels asserted; the
box and score differences come from stream-K split points that depend on the batch).  Writes nothing.

    python bench_mixed.py [--runs 5] [--iters 10] [--workloads photos,landscape,uniform]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

WORKLOADS = {
    'photos': [(480, 640), (640, 480), (427, 640), (640, 427), (375, 500), (500, 375), (612, 612), (480, 640)],
    'landscape': [(480, 640)] * 3 + [(427, 640)] * 3 + [(612, 612)] * 2,
    'uniform': [(480, 640)] * 8,
}


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader',
                            '-i', '0'], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'unknown'
    return name, q or 'unknown'


class Counting(object):
    """The engine, counting the predict calls and kernel launches a predict_batch_raw makes."""

    def __init__(self, eng):
        self.eng, self.calls, self.launches = eng, 0, 0

    def __getattr__(self, name):
        attr = getattr(self.eng, name)
        if not name.startswith('predict'):
            return attr

        def call(*a, **k):
            r = attr(*a, **k)
            self.calls += 1
            self.launches += self.eng.last_launch_count
            return r
        return call


def network(cfg, eng, pack):
    from luminoth_b200.predicting import PredictorNetwork
    net = PredictorNetwork.__new__(PredictorNetwork)        # the engine is shared by both groupings
    net.config, net.engine, net.class_labels, net.pack_sizes = cfg, Counting(eng), None, pack
    return net


def run(name, shapes, runs, iters):
    import bench
    from luminoth_b200 import synth
    from luminoth_b200.engine import Engine
    cfg = bench.build_config(bench.WORKLOADS['frcnn_r50'])
    eng = Engine(cfg, device=0, max_batch=8)
    eng.load_weights(synth.make_weights(cfg, seed=0, profile='peaky')).finalize()
    rng = np.random.default_rng(7)
    sets = [[rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8) for h, w in shapes] for _ in range(2)]
    nets = {'off': network(cfg, eng, False), 'on': network(cfg, eng, True)}
    box_d = score_d = 0.0
    for images in sets:
        want = nets['off'].predict_batch_raw(images)
        for _ in range(3):                        # eager, graph capture, replay
            got = nets['on'].predict_batch_raw(images)
        for (b0, l0, s0, _), (b1, l1, s1, _) in zip(want, got):
            assert b0.shape == b1.shape and np.array_equal(l0, l1), 'packing changed the counts or classes'
            if len(b0):
                box_d = max(box_d, float(np.abs(b0 - b1).max()))
                score_d = max(score_d, float(np.abs(s0 - s1).max()))
        nets['off'].predict_batch_raw(images)
    per_call = {}
    for k, net in nets.items():
        net.engine.calls = net.engine.launches = 0
        net.predict_batch_raw(sets[0])
        per_call[k] = (net.engine.calls, net.engine.launches)
    rates = {k: [] for k in nets}
    for _ in range(runs):
        for k, net in nets.items():
            t0 = time.perf_counter()
            for i in range(iters):
                net.predict_batch_raw(sets[i % 2])     # host outputs: each call ends synchronised
            rates[k].append(iters * len(shapes) / (time.perf_counter() - t0))
    eng.profile(True)                                  # device time per category of one packed batch, graphs off
    nets['on'].predict_batch_raw(sets[0])
    cats = eng.profile_read()
    band = sum(ms for layer, _, ms, _ in eng.profile_read_layers() if layer == 'band_clear')
    eng.profile(False)
    eng.close()
    out = {'workload': name, 'model': 'frcnn_r50', 'images': ['%dx%d' % s for s in shapes], 'runs': runs,
           'calls_per_run': iters, 'max_box_diff_px': box_d, 'max_score_diff': score_d}
    for k, r in rates.items():
        out['pack_%s_images_per_s' % k] = {'median': round(statistics.median(r), 1), 'min': round(min(r), 1),
                                           'max': round(max(r), 1)}
        out['pack_%s_engine_calls' % k], out['pack_%s_launches' % k] = per_call[k]
    out['speedup_median'] = round(statistics.median(rates['on']) / statistics.median(rates['off']), 3)
    total = sum(ms for _, ms, _ in cats.values())
    out['band_clear_share_of_forward'] = round(band / total, 4) if total else None
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--runs', type=int, default=5)
    ap.add_argument('--iters', type=int, default=10, help='predict_batch_raw calls per timed run')
    ap.add_argument('--workloads', default='photos,landscape,uniform')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_mixed.py measures on a CUDA device; none is visible')
    name, query = card()
    for wl in args.workloads.split(','):
        res = run(wl, WORKLOADS[wl], args.runs, args.iters)
        res['gpu'] = name
        res['power_limit,sm_clock,max_sm_clock'] = query
        print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
