"""The engine's weight list on the GPU (`-m gpu`): the ordered (name, shape) list lumi_create derives from the config
(`Engine.weight_specs()`, read by checkpoint loading and by parallel.pack_weights, whose packing follows its order),
checked against tests/golden/weight_specs.json over the ResNet architectures, endpoints, output strides and head
options, and the SSD default.  The fixture keeps each list's length and SHA-256; regenerate it with a GPU by

    python tests/test_gpu_weight_specs.py
"""
import hashlib
import json
import os
import sys

import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, 'golden', 'weight_specs.json')

ARCHS = ['resnet_v1_50', 'resnet_v1_101', 'resnet_v1_152', 'resnet_v2_50', 'resnet_v2_101', 'resnet_v2_152']


def _cases():
    # id -> (model type, override params, list-valued settings)
    cases = {'ssd': ('ssd', [], {})}
    for arch in ARCHS:
        for rcnn in ('true', 'false'):
            cases['%s-rcnn_%s' % (arch, rcnn)] = ('fasterrcnn', ['model.base_network.architecture=' + arch,
                                                                 'model.network.with_rcnn=' + rcnn], {})
    cases['resnet_v1_101-no_tail'] = ('fasterrcnn', ['model.base_network.architecture=resnet_v1_101',
                                                     'model.base_network.use_tail=false'], {})
    for v, arch in ((1, 'resnet_v1_50'), (2, 'resnet_v2_50')):
        unit = 'block2/unit_1/bottleneck_v%d/' % v
        for ep in ['conv1', 'block1', 'block2', 'block4'] + [unit + p for p in ('conv1', 'conv2', 'conv3', 'shortcut')]:
            cases['%s-%s' % (arch, ep.replace('/', '.'))] = (
                'fasterrcnn', ['model.base_network.architecture=' + arch, 'model.base_network.endpoint=' + ep], {})
        for os_ in (8, 32):
            cases['%s-os%d' % (arch, os_)] = ('fasterrcnn', ['model.base_network.architecture=' + arch,
                                                             'model.base_network.output_stride=%d' % os_], {})
    cases['resnet_v1_50-no_mean'] = ('fasterrcnn', ['model.base_network.architecture=resnet_v1_50',
                                                    'model.rcnn.use_mean=false'], {})
    cases['resnet_v1_101-no_mean'] = ('fasterrcnn', ['model.base_network.architecture=resnet_v1_101',
                                                     'model.rcnn.use_mean=false'], {})
    cases['resnet_v1_50-rpn_5x3-fc_64_32'] = ('fasterrcnn', ['model.base_network.architecture=resnet_v1_50'],
                                              {'rpn.kernel_shape': [5, 3], 'rcnn.layer_sizes': [64, 32]})
    return cases


CASES = _cases()


def weight_list_digest(case):
    from luminoth_b200 import default_config
    from luminoth_b200.engine import Engine
    mtype, params, lists = case
    cfg = default_config(mtype, params)
    for key, value in lists.items():
        scope, name = key.rsplit('.', 1)
        node = cfg.model
        for k in scope.split('.'):
            node = node[k]
        node[name] = value
    eng = Engine(cfg)
    specs = [[name, list(shape)] for name, shape in eng.weight_specs()]
    eng.close()
    return {'count': len(specs), 'sha256': hashlib.sha256(json.dumps(specs).encode()).hexdigest()}


def _fixture():
    with open(FIXTURE) as f:
        return json.load(f)


def test_fixture_covers_the_cases():
    assert sorted(_fixture()) == sorted(CASES)


@pytest.mark.parametrize('case', sorted(CASES))
def test_weight_list_matches_fixture(case):
    want = _fixture()[case]
    assert want['params'] == CASES[case][1] and want['lists'] == CASES[case][2], 'fixture made for another config'
    got = weight_list_digest(CASES[case])
    assert got == {'count': want['count'], 'sha256': want['sha256']}, (case, got, want)


if __name__ == '__main__':
    sys.path.insert(0, os.path.dirname(HERE))
    out = {}
    for case_id, case in sorted(CASES.items()):
        out[case_id] = dict(weight_list_digest(case), params=case[1], lists=case[2])
    with open(FIXTURE, 'w') as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write('\n')
    print('wrote %d cases to %s' % (len(out), FIXTURE))
