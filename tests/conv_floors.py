"""Per-layer floors of the Faster R-CNN ResNet-50 conv stack (bench.py's headline workload, batch 8 x 600x1024).

    python tests/conv_floors.py RUN.json [RUN.json ...]

RUN.json: the JSON line of `bench.py --layers`.  Prints one markdown row per conv layer: measured time (median over
the runs), algorithmic TFLOP/s, and the layer's floor -- the larger of its HBM byte time and its tensor time -- with
the bound named.

* Bytes: every activation element crosses HBM once at 4 B (the fp16 hi + lo planes; fp32 for fp32 outputs): input,
  output, residual, plus the fp16 hi + lo weights.  L2 reuse of overlapping 3x3 windows is assumed perfect.
* Tensor time: 3 fp16 MMAs per MAC the kernel runs (the hi/lo split, DESIGN section 3) at the dense-FP16 rate scaled
  to the SM clock the run reported (989 TFLOP/s at 1830 MHz on the H100 SXM data sheet).  The stem runs as four
  K = 64 taps (space-to-depth), so its tensor work is that of K = 256, not 7 x 7 x 3.
* HBM: 3.35 TB/s (data sheet).  Neither rate is measured, so the floors are lower bounds.

Not a test: nothing runs on import.
"""
import json
import statistics
import sys

B, H, W = 8, 600, 1024
HBM = 3.35e12
FP16_AT_1830 = 989e12
PREFIX = 'truncated_base_network/resnet_v1_50/'


def layers():
    """(name, m_in, cin, m_out, cout, kdim, residual, out_bytes) of every conv of the workload."""
    out = []

    def conv(name, hw_in, cin, hw_out, cout, kdim, res=False, ob=4):
        out.append((name, B * hw_in[0] * hw_in[1], cin, B * hw_out[0] * hw_out[1], cout, kdim, res, ob))

    # stem: the 7x7/2 conv of the 3-channel image runs as 4 taps of K = 64 over a 16-channel space-to-depth staging
    conv(PREFIX + 'conv1#s2d', (303, 515), 16, (300, 512), 64, 256)
    hw = (150, 256)                                       # after the 3x3/2 max pool
    cin = 64
    for blk, (units, depth) in enumerate([(3, 64), (4, 128), (6, 256)], start=1):
        for u in range(1, units + 1):
            # slim resnet_v1: stride 2 in the 3x3 conv of the last unit of block1 and block2 (block3 is truncated)
            stride = 2 if (u == units and blk < 3) else 1
            hw2 = ((hw[0] + 1) // 2, (hw[1] + 1) // 2) if stride == 2 else hw
            base = PREFIX + 'block%d/unit_%d/bottleneck_v1/' % (blk, u)
            if u == 1:
                conv(base + 'shortcut', hw, cin, hw, depth * 4, cin)
            conv(base + 'conv1', hw, cin, hw, depth, cin)
            conv(base + 'conv2', hw, depth, hw2, depth, 9 * depth)
            conv(base + 'conv3', hw2, depth, hw2, depth * 4, depth, res=True)
            hw, cin = hw2, depth * 4
    conv('fasterrcnn/rpn/conv', hw, 1024, hw, 512, 9 * 1024)
    conv('fasterrcnn/rpn/heads', hw, 512, hw, 54, 512)
    # box head: pooled, spatially averaged 1024-channel rows of 2000 proposals per image -> 81 scores + 320 deltas
    out.append(('fasterrcnn/rcnn/heads', 2000 * B, 1024, 2000 * B, 401, 1024, False, 4))
    return out


def floor(m_in, cin, m_out, cout, kdim, res, ob, sm_mhz):
    nbytes = 4.0 * m_in * cin + ob * m_out * cout + (4.0 * m_out * cout if res else 0.0) + 4.0 * kdim * cout
    t_hbm = nbytes / HBM
    t_tc = 3 * 2.0 * m_out * kdim * cout / (FP16_AT_1830 * sm_mhz / 1830.0)
    return (t_hbm, 'HBM') if t_hbm >= t_tc else (t_tc, 'tensor')


def main(paths):
    runs = [json.loads(open(p).read().strip().splitlines()[-1]) for p in paths]
    sm = statistics.median(r['clocks']['sm_mhz'] for r in runs if r.get('clocks') and r['clocks'].get('sm_mhz'))
    meas = {}
    for r in runs:
        for row in r['conv_layers']:
            meas.setdefault(row['layer'], []).append((row['us'], row['gflop']))
    print('SM clock (median of the runs): %.0f MHz; tensor floor at %.0f TFLOP/s fp16 = %.0f algorithmic' %
          (sm, FP16_AT_1830 * sm / 1830 / 1e12, FP16_AT_1830 * sm / 1830 / 3e12))
    print('| layer | us | TFLOP/s | floor us | bound |')
    print('|---|---|---|---|---|')
    tot = {'us': 0.0, 'floor': 0.0}
    by_bound = {'HBM': [0.0, 0.0], 'tensor': [0.0, 0.0]}
    for name, m_in, cin, m_out, cout, kdim, res, ob in layers():
        if name not in meas:
            continue
        us = statistics.median(t for t, _ in meas[name])
        gf = meas[name][0][1]
        f, bound = floor(m_in, cin, m_out, cout, kdim, res, ob, sm)
        tot['us'] += us
        tot['floor'] += f * 1e6
        by_bound[bound][0] += us
        by_bound[bound][1] += f * 1e6
        print('| %s | %.0f | %.0f | %.0f | %s |' % (name.replace(PREFIX, ''), us, gf / us * 1e3, f * 1e6, bound))
    print('| **all** | %.0f | | %.0f | |' % (tot['us'], tot['floor']))
    for b, (us, fl) in by_bound.items():
        print('| %s-bound layers | %.0f | | %.0f | |' % (b, us, fl))


if __name__ == '__main__':
    main(sys.argv[1:])
