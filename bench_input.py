"""Input-path benchmark: detection on images at their original sizes, resize included.

Every real image needs a resize before the network sees it; bench.py feeds images that already have the network's
size, so it never times that step.  This script times two ways of doing it on one engine, alternated, `--runs` runs
each:

  old    per image: pageable upload, lumi_op_resize_bilinear into a float32 device batch, synchronise; then
         predict_raw on that batch (lumi_predict_f32) -- what PredictorNetwork did before lumi_predict_resize
  fused  one predict_resize call (lumi_predict_resize): the sources packed through a pinned buffer, the resize done by
         the kernels that stage the first conv's input, inside the CUDA graph and the two-stream pipeline

on three workloads a user runs:

  video  8 video frames 1080x1920 -> 576x1024, Faster R-CNN ResNet-50 as bench.py's frcnn_r50
  photo  8 photos 480x640 -> 600x800, the same model
  ssd    32 photos 375x500 -> 300x300, SSD VGG-16 as bench.py's ssd

Both paths must give identical bytes (asserted).  Prints one JSON line per workload with images/s (median, min, max
over the runs) and the card's name and power limit.  Writes nothing.

    python bench_input.py [--runs 5] [--iters 20] [--workloads video,photo,ssd]
"""
import argparse
import ctypes
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
    'video': dict(bench='frcnn_r50', n=8, h0=1080, w0=1920),
    'photo': dict(bench='frcnn_r50', n=8, h0=480, w0=640),
    'ssd': dict(bench='ssd', n=32, h0=375, w0=500),
}


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = 'unknown'
    return name, power or 'unknown'


def old_path(eng, images, h, w):
    """Per-image upload and resize into a float32 device batch, then the float32 entry point."""
    import torch
    dev = torch.device('cuda', eng.device)
    batch = torch.empty((len(images), h, w, 3), dtype=torch.float32, device=dev)
    for i, im in enumerate(images):
        src = torch.from_numpy(im).to(dev)
        rc = eng._lib.lumi_op_resize_bilinear(ctypes.c_void_p(src.data_ptr()), 0, im.shape[0], im.shape[1],
                                              ctypes.c_void_p(batch[i].data_ptr()), h, w, None)
        if rc != 0:
            raise RuntimeError(eng._lib.lumi_op_last_error().decode())
    torch.cuda.synchronize(dev)
    return eng.predict_raw(batch)


def fused_path(eng, images, h, w):
    return eng.predict_resize(images, h, w)


def run(name, wl, runs, iters):
    import bench
    from luminoth_b200 import synth
    from luminoth_b200.engine import Engine
    from luminoth_b200.predicting import target_size
    cfg = bench.build_config(bench.WORKLOADS[wl['bench']])
    n = wl['n']
    h, w, _ = target_size((wl['h0'], wl['w0']), cfg)
    eng = Engine(cfg, device=0, max_batch=n, max_h=h, max_w=w)
    eng.load_weights(synth.make_weights(cfg, seed=0, profile='peaky')).finalize()
    # two rotating sets of decoded uint8 sources, as a stream of frames would give them
    sets = [list(synth.make_images(n, wl['h0'], wl['w0'], seed=100 + s)) for s in range(2)]
    paths = {'old': old_path, 'fused': fused_path}
    for images in sets:
        want = old_path(eng, images, h, w)
        assert int(want[3].sum()) > 0, 'no detections: the comparison would be vacuous'
        for _ in range(3):                     # eager, graph capture, replay
            got = fused_path(eng, images, h, w)
            for a, b in zip(want, got):
                assert np.array_equal(a, b), 'the fused resize changed the results'
        old_path(eng, images, h, w)
    rates = {k: [] for k in paths}
    for _ in range(runs):
        for k, fn in paths.items():
            t0 = time.perf_counter()
            for i in range(iters):
                fn(eng, sets[i % 2], h, w)        # returns host outputs: each call ends synchronised
            rates[k].append(iters * n / (time.perf_counter() - t0))
    eng.close()
    out = {'workload': name, 'model': bench.WORKLOADS[wl['bench']]['name'].split(',')[0],
           'images': '%d x %dx%d -> %dx%d' % (n, wl['h0'], wl['w0'], h, w), 'runs': runs, 'calls_per_run': iters,
           'identical_bytes': True}
    for k, r in rates.items():
        out[k + '_images_per_s'] = {'median': round(statistics.median(r), 1), 'min': round(min(r), 1),
                                    'max': round(max(r), 1)}
    out['speedup_median'] = round(statistics.median(rates['fused']) / statistics.median(rates['old']), 3)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--runs', type=int, default=5)
    ap.add_argument('--iters', type=int, default=20, help='calls per timed run')
    ap.add_argument('--workloads', default='video,photo,ssd')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_input.py measures on a CUDA device; none is visible')
    name, power = card()
    for wl in args.workloads.split(','):
        res = run(wl, WORKLOADS[wl], args.runs, args.iters)
        res['gpu'] = name
        res['power_limit'] = power
        print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
