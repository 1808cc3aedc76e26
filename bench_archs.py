"""bench.py's measurement for the Faster R-CNN base networks bench.py does not list: resnet_v1_152 and the
pre-activation resnet_v2_{50,101,152}, in bench.py's flagship setting (batch 8 x 600x1024, 80 classes).

Registers one workload per network in bench.WORKLOADS and runs bench.py's own main, so the arguments and the JSON
line are bench.py's, e.g.  python bench_archs.py --workload frcnn_v2_r50 --gpus 1 --steps 50 --warmup 5 --layers
"""
import bench

ARCHS = {'frcnn_r152': 'resnet_v1_152', 'frcnn_v2_r50': 'resnet_v2_50', 'frcnn_v2_r101': 'resnet_v2_101',
         'frcnn_v2_r152': 'resnet_v2_152'}

for key, arch in ARCHS.items():
    bench.WORKLOADS[key] = dict(
        model='fasterrcnn', batch=8, h=600, w=1024,
        overrides=['model.base_network.architecture=' + arch, 'model.network.num_classes=80'],
        name='Faster R-CNN %s (reference COCO config: 80 classes, post_nms_top_n 2000), batch 8 x 600x1024x3 '
             'synthetic uint8' % arch)

if __name__ == '__main__':
    bench.main()
