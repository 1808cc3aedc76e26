"""bench.py's measurement for the Faster R-CNN base networks bench.py does not list: resnet_v1_152 and the
pre-activation resnet_v2_{50,101,152}, in bench.py's flagship setting (batch 8 x 600x1024, 80 classes), ResNet-50
at output_stride 8 and 4, and ResNet-50 from the block4 and block2 endpoints.

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

# ResNet-50 at output_stride 8 and 4 with anchors of the same stride: 115 200 and 460 800 anchors per image, 9.6 and
# 38.4 per kept RPN candidate (pre_nms_top_n 12 000), against bench.py's frcnn_r50 at 2.4 -- workloads on both sides
# of the RPN's top-k cut
for stride in (8, 4):
    bench.WORKLOADS['frcnn_r50_os%d' % stride] = dict(
        model='fasterrcnn', batch=8, h=600, w=1024,
        overrides=['model.base_network.architecture=resnet_v1_50', 'model.network.num_classes=80',
                   'model.base_network.output_stride=%d' % stride, 'model.anchors.stride=%d' % stride],
        name='Faster R-CNN ResNet-50 at output_stride %d, anchor stride %d (reference COCO config: 80 classes, '
             'post_nms_top_n 2000), batch 8 x 600x1024x3 synthetic uint8' % (stride, stride))

# ResNet-50 from the block4 endpoint (the 2048-channel C5 map, block4 atrous at rate 2 in the trunk) and from block2
# (512 channels), both at output_stride 16 like bench.py's frcnn_r50: the RPN conv and the RCNN head read 2048 and 512
# channels instead of 1024
for endpoint in ('block4', 'block2'):
    bench.WORKLOADS['frcnn_r50_' + endpoint] = dict(
        model='fasterrcnn', batch=8, h=600, w=1024,
        overrides=['model.base_network.architecture=resnet_v1_50', 'model.network.num_classes=80',
                   'model.base_network.endpoint=' + endpoint],
        name='Faster R-CNN ResNet-50 from endpoint %s (reference COCO config: 80 classes, post_nms_top_n 2000), '
             'batch 8 x 600x1024x3 synthetic uint8' % endpoint)

if __name__ == '__main__':
    bench.main()
