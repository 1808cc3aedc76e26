"""Sliced-prediction benchmark: one large photo through PredictorNetwork.predict_tiled against the by-hand way.

A seeded synthetic 4000 x 6000 uint8 photo, Faster R-CNN ResNet-50 (bench.py's frcnn_r50 config and weights, 80
classes, max_batch 8), 600 px tiles at overlap 0.2 plus the whole image (118 windows):

  tiled   PredictorNetwork.predict_tiled: the photo is uploaded once, the windows are cut and resized in the engine's
          input staging, and their detections are merged on the GPU (lumi_predict_windows)
  host    the same windows cropped on the host, PredictorNetwork.predict_batch_raw on the crops (one engine call per
          target size and max_batch chunk), then the numpy merge of tests/tile_merge_ref.py

The two ways alternate, `--runs` times each; it prints one JSON line with the median, min and max seconds per photo
of each, the card's name and power limit read in the same run, and whether the two give the same detections
(counts, labels, boxes and scores compared; both run the same per-window forwards, but predict_batch_raw sizes its
chunks differently, so stream-K split points may differ in the last bits).  Writes nothing.

    python bench_tiles.py [--runs 5]
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

TILE, OVERLAP, SHAPE = 600, 0.2, (4000, 6000)


def host_way(net, photo):
    wins, scales = net.tile_windows(photo.shape, TILE, OVERLAP, True)
    crops = [photo[y0:y0 + h, x0:x0 + w] for y0, x0, h, w, _, _ in wins]
    raw = net.predict_batch_raw(crops)
    from tile_merge_ref import merge_windows
    k = net.engine.max_detections
    n = len(wins)
    b = np.zeros((n, k, 4), np.float32)
    s = np.zeros((n, k), np.float32)
    lab = np.full((n, k), -1, np.int32)
    c = np.zeros((n,), np.int32)
    for j, (objs, labels, probs, _) in enumerate(raw):
        m = len(probs)
        b[j, :m] = objs; s[j, :m] = probs; lab[j, :m] = labels; c[j] = m
    p = net.config.model.rcnn.proposals
    wmap = [(w[0], w[1], sc[0], sc[1]) for w, sc in zip(wins, scales)]
    return merge_windows(b, s, lab, c, [0] * n, wmap, 1, net.config.model.network.num_classes,
                         p.class_max_detections, k, net.merge_iou_threshold())[0]


def tiled_way(net, photo):
    wins, scales = net.tile_windows(photo.shape, TILE, OVERLAP, True)
    boxes, scores, labels, counts = net.engine.predict_windows([photo], [(0,) + w for w in wins], scales,
                                                               net.merge_iou_threshold())
    k = int(counts[0])
    return boxes[0, :k], scores[0, :k], labels[0, :k]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=5)
    args = ap.parse_args()
    import bench
    from luminoth_b200 import synth
    from luminoth_b200.predicting import PredictorNetwork
    cfg = bench.build_config(bench.WORKLOADS["frcnn_r50"])
    wts = synth.make_weights(cfg, seed=0, profile='peaky')
    net = PredictorNetwork(cfg, weights=wts, max_batch=8)
    photo = np.random.default_rng(0).integers(0, 256, size=SHAPE + (3,), dtype=np.uint8)
    tiled, host = tiled_way(net, photo), host_way(net, photo)        # warm-up: every shape and graph
    same_counts = len(tiled[1]) == len(host[1]) and (np.sort(tiled[2]) == np.sort(host[2])).all()
    box_diff = float(np.abs(tiled[0] - host[0]).max()) if same_counts and len(host[1]) else None
    times = {'tiled': [], 'host': []}
    for _ in range(args.runs):
        for name, fn in (('tiled', tiled_way), ('host', host_way)):
            t0 = time.perf_counter()
            fn(net, photo)
            times[name].append(time.perf_counter() - t0)
    name, power = card()
    net.engine.close()
    out = {'workload': 'frcnn_r50 4000x6000 photo, 600 px tiles, overlap 0.2, full image',
           'windows': len(net.tile_windows(photo.shape, TILE, OVERLAP, True)[0]), 'runs': args.runs,
           'card': name, 'power_limit_clocks': power, 'detections': len(tiled[1]),
           'same_counts_and_labels': bool(same_counts), 'max_box_diff_px': box_diff}
    for k, v in times.items():
        out[k + '_s'] = {'median': statistics.median(v), 'min': min(v), 'max': max(v)}
    out['speedup'] = statistics.median(times['host']) / statistics.median(times['tiled'])
    print(json.dumps(out))


if __name__ == '__main__':
    main()
