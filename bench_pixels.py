"""Pixel-format benchmark: video frames fed as they arrive (BGR, NV12) against converting them to RGB first.

Faster R-CNN ResNet-50 (bench.py's frcnn_r50 config and weights, max_batch 8), seeded 1080 x 1920 frames resized to
576 x 1024 in the engine's input staging (Engine.predict_resize), 8 calls of 8 frames per run.  Three pairs:

  (a) bgr_flip   host BGR frames flipped on the host with predict_video's expression, then RGB
      bgr        the same host BGR frames as they are (pixel_format='bgr')
  (b) rgb_host   host RGB frames
      nv12_host  the same pixels as host NV12 frames (1.5 bytes per pixel instead of 3)
  (c) rgb_dev    the RGB frames as CUDA tensors
      nv12_dev   the NV12 frames as CUDA tensors

The two sides of each pair alternate, `--runs` times each; it prints one JSON line with the median, min and max frames
per second of each, the card's name and power limit read in the same run, and whether the two sides of each pair gave
identical detections (boxes, scores, labels and counts of every call, byte for byte).  Writes nothing.

    python bench_pixels.py [--runs 5]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import numpy as np  # noqa: E402

from bench_mixed import card  # noqa: E402

SRC, TARGET, BATCH, CALLS, DISTINCT = (1080, 1920), (576, 1024), 8, 8, 16


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=5)
    args = ap.parse_args()
    import torch
    import bench
    import pixel_formats_ref as R
    from luminoth_b200 import synth
    from luminoth_b200.engine import Engine
    cfg = bench.build_config(bench.WORKLOADS['frcnn_r50'])
    eng = Engine(cfg, max_batch=BATCH, max_h=TARGET[0], max_w=TARGET[1])
    eng.load_weights(synth.make_weights(cfg, seed=0, profile='peaky')).finalize()
    nv12 = R.random_frames([SRC] * DISTINCT, seed=0)['nv12']
    rgb = [R.to_rgb(f, 'nv12') for f in nv12]
    bgr = [np.ascontiguousarray(f[:, :, ::-1]) for f in rgb]
    rgb_dev = [torch.from_numpy(f).cuda() for f in rgb]
    nv12_dev = [torch.from_numpy(f).cuda() for f in nv12]

    def run(frames, fmt, flip=False):
        outs = []
        for c in range(CALLS):
            batch = [frames[(c * BATCH + j) % DISTINCT] for j in range(BATCH)]
            if flip:                                   # predict.py:predict_video's per-frame conversion
                batch = [np.ascontiguousarray(f[:, :, ::-1]) for f in batch]
            outs.append(eng.predict_resize(batch, *TARGET, pixel_format=fmt))
        return outs

    sides = {'bgr_flip': lambda: run(bgr, 'rgb', flip=True), 'bgr': lambda: run(bgr, 'bgr'),
             'rgb_host': lambda: run(rgb, 'rgb'), 'nv12_host': lambda: run(nv12, 'nv12'),
             'rgb_dev': lambda: run(rgb_dev, 'rgb'), 'nv12_dev': lambda: run(nv12_dev, 'nv12')}
    pairs = (('bgr_flip', 'bgr'), ('rgb_host', 'nv12_host'), ('rgb_dev', 'nv12_dev'))
    first = {name: fn() for name, fn in sides.items()}                 # warm-up: every shape, format and graph
    same = {}
    for a, b in pairs:
        same[a + '=' + b] = all(all(np.array_equal(x, y) for x, y in zip(oa, ob))
                                for oa, ob in zip(first[a], first[b]))
    times = {name: [] for name in sides}
    for _ in range(args.runs):
        for a, b in pairs:
            for name in (a, b):
                t0 = time.perf_counter()
                sides[name]()
                times[name].append(BATCH * CALLS / (time.perf_counter() - t0))
    name, power = card()
    eng.close()
    out = {'workload': 'frcnn_r50 1080x1920 frames -> 576x1024, max_batch 8, %d frames per run' % (BATCH * CALLS),
           'runs': args.runs, 'card': name, 'power_limit_clocks': power,
           'detections_per_run': int(sum(int(o[3].sum()) for o in first['rgb_host'])), 'identical': same}
    for k, v in times.items():
        out[k + '_fps'] = {'median': statistics.median(v), 'min': min(v), 'max': max(v)}
    for a, b in pairs:
        out['gain_' + b] = statistics.median(times[b]) / statistics.median(times[a])
    print(json.dumps(out))
    assert all(same.values()), 'a format gave other detections than its RGB conversion: %s' % same


if __name__ == '__main__':
    main()
