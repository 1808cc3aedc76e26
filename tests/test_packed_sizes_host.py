"""CPU-only checks of packing images of different sizes into one engine call (``lumi_predict_sizes``): the grouping
rule of ``PredictorNetwork(pack_sizes=True)``, today's grouping when it is off, the ``--pack-sizes`` flags and the
exported entry point."""
import argparse
import os
import re

import numpy as np
import pytest

from luminoth_b200 import predicting as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def fill(targets, group):
    hc = max(targets[i][0] for i in group)
    wc = max(targets[i][1] for i in group)
    return sum(targets[i][0] * targets[i][1] for i in group) / float(len(group) * hc * wc)


def test_pack_groups_rule():
    rng = np.random.default_rng(0)
    for trial in range(200):
        n = int(rng.integers(1, 30))
        targets = [(int(rng.integers(100, 1000)), int(rng.integers(100, 1000))) for _ in range(n)]
        max_batch = int(rng.integers(1, 9))
        groups = P.pack_groups(targets, max_batch)
        assert sorted(i for g in groups for i in g) == list(range(n))           # every image once
        order = [i for g in groups for i in g]
        keys = [(targets[i][0] > targets[i][1], targets[i][0], targets[i][1]) for i in order]
        assert keys == sorted(keys)                                              # orientation, then size
        for k, g in enumerate(groups):
            assert 1 <= len(g) <= max_batch
            assert len(g) == 1 or fill(targets, g) >= P.PACK_FILL
            if k + 1 < len(groups) and len(g) < max_batch:                       # a cut only where the next image
                assert fill(targets, g + [groups[k + 1][0]]) < P.PACK_FILL      # would drop the fill


def test_pack_groups_examples():
    photos = [(600, 800), (800, 600), (600, 899), (600, 600), (600, 800)]
    groups = P.pack_groups(photos, 8)
    assert [[photos[i] for i in g] for g in groups] == [[(600, 600), (600, 800), (600, 800), (600, 899)],
                                                        [(800, 600)]]
    assert P.pack_groups(photos, 2) == [[3, 0], [4, 2], [1]]
    assert P.pack_groups([(600, 800)] * 3, 8, fill=1.0) == [[0, 1, 2]]
    assert P.pack_groups([(600, 800), (300, 400)], 8, fill=0.7) == [[1], [0]]


def test_size_groups_are_todays_buckets():
    targets = [(600, 800), (800, 600), (600, 800), (600, 800), (600, 899), (800, 600)]
    assert P.size_groups(targets, 2) == [[0, 2], [3], [1, 5], [4]]
    assert P.size_groups(targets, 8) == [[0, 2, 3], [1, 5], [4]]


class FakeEngine(object):
    max_batch = 3

    def __init__(self):
        self.calls = []

    def _out(self, n, h, w):
        boxes = np.zeros((n, 2, 4), np.float32)
        boxes[:, 0] = [0, 0, w - 1, h - 1]
        return boxes, np.ones((n, 2), np.float32), np.zeros((n, 2), np.int32), np.ones(n, np.int32)

    def predict_raw(self, batch):
        self.calls.append(('raw', [im.shape[:2] for im in batch]))
        return self._out(len(batch), *batch.shape[1:3])

    def predict_resize(self, srcs, h, w):
        self.calls.append(('resize', [(h, w)] * len(srcs)))
        return self._out(len(srcs), h, w)

    def predict_sizes(self, srcs, targets):
        self.calls.append(('sizes', [tuple(t) for t in targets]))
        out = self._out(len(srcs), 1, 1)
        for j, (h, w) in enumerate(targets):
            out[0][j, 0] = [0, 0, w - 1, h - 1]
        return out


def fake_network(pack):
    net = P.PredictorNetwork.__new__(P.PredictorNetwork)
    net.config = {'dataset': {'image_preprocessing': {'min_size': 600, 'max_size': 1024}}}
    net.engine, net.class_labels, net.pack_sizes = FakeEngine(), None, pack
    return net


def test_predictor_groups_and_caller_order():
    shapes = [(480, 640), (640, 480), (600, 800), (375, 500), (612, 612), (480, 640), (600, 800)]
    images = [np.zeros(s + (3,), np.uint8) for s in shapes]
    targets = [P.target_size(s, fake_network(False).config)[:2] for s in shapes]
    for pack in (False, True):
        net = fake_network(pack)
        out = net.predict_batch_raw(images)
        for (boxes, _, _, _), (h, w) in zip(out, targets):           # each result is its own image's, in order
            np.testing.assert_array_equal(boxes[0], [0, 0, w - 1, h - 1])
        calls = net.engine.calls
        if not pack:                                                  # today's calls: one per size-bucket chunk
            want = P.size_groups(targets, 3)
            assert [c[1] for c in calls] == [[targets[i] for i in g] for g in want]
            assert [c[0] for c in calls] == ['resize', 'resize', 'resize', 'raw']   # 612x612 keeps its size
        else:
            assert [c[1] for c in calls] == [[targets[i] for i in g] for g in P.pack_groups(targets, 3)]
            assert all(c[0] == ('sizes' if len(set(c[1])) > 1 else 'resize') or c[0] == 'raw' for c in calls)


class Parsed(Exception):
    pass


@pytest.mark.parametrize('module,argv', [
    ('predict', ['img.jpg']),
    ('server', ['-c', 'cfg.yml']),
    ('eval', ['-c', 'cfg.yml']),
])
def test_cli_pack_sizes_flag(monkeypatch, module, argv):
    import importlib
    mod = importlib.import_module('luminoth_b200.' + module)
    parse = argparse.ArgumentParser.parse_args

    def capture(self, args=None, namespace=None):
        raise Parsed(parse(self, args, namespace))
    monkeypatch.setattr(argparse.ArgumentParser, 'parse_args', capture)
    for extra, want in (([], False), (['--pack-sizes'], True)):
        with pytest.raises(Parsed) as ex:
            mod.main(argv + extra)
        assert ex.value.args[0].pack_sizes is want


def test_predict_sizes_is_declared_and_bound():
    from luminoth_b200 import engine
    hdr = open(os.path.join(ROOT, 'include', 'luminoth_b200.h')).read()
    assert re.search(r'\bint lumi_predict_sizes\s*\(', hdr)
    assert 'lumi_predict_sizes' in engine.SIGNATURES
    import __graft_entry__ as g
    g.build()
    assert hasattr(engine.load_library(), 'lumi_predict_sizes')
