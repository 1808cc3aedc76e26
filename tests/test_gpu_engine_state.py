"""Engine-handle isolation (`-m gpu`): no process-global launch state.  The reference's web server keeps one
network and calls it from request threads next to a loader thread (``tools/server/web.py:53-62``); here several
engines may live in one process, on one or several devices, each driven by its own thread."""
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from luminoth_b200 import default_config, synth, parallel as P
from luminoth_b200.engine import Engine, load_library


def _cfg(extra=()):
    return default_config('fasterrcnn', ['model.base_network.architecture=resnet_v1_50', 'model.network.num_classes=20',
                                         'model.rpn.proposals.post_nms_top_n=200',
                                         'model.rcnn.proposals.min_prob_threshold=0.05'] + list(extra))


def test_two_engines_two_threads_bit_identical():
    """Two engines with DIFFERENT switch settings (stream-K off / always, pipeline on / off, batch 2 / 1) run
    concurrently from two threads; each must reproduce, bit for bit, what it gives when it runs alone.  With the
    round-1 process globals (conv SM reserve, stream-K mode) the two raced."""
    cfg = _cfg()
    wts = synth.make_weights(cfg, seed=1)
    ndev = load_library().lumi_device_count()
    imgs_a = synth.make_images(2, 224, 320, seed=2)
    imgs_b = synth.make_images(1, 192, 256, seed=3)
    ea = Engine(cfg, device=0, max_batch=2, max_h=224, max_w=320)
    ea.load_weights(wts).finalize()
    ea.set_conv_streamk('always')
    eb = Engine(cfg, device=1 if ndev > 1 else 0, max_batch=1, max_h=192, max_w=256)
    eb.load_weights(wts).finalize()
    eb.set_conv_streamk('off')
    eb.set_pipeline(False)
    alone_a = ea.predict_raw(imgs_a)
    alone_b = eb.predict_raw(imgs_b)
    errors = []

    def work(eng, imgs, want):
        try:
            for _ in range(8):
                got = eng.predict_raw(imgs)
                for x, y in zip(got, want):
                    np.testing.assert_array_equal(x, y)
        except Exception as ex:          # noqa: BLE001
            errors.append(ex)

    ta = threading.Thread(target=work, args=(ea, imgs_a, alone_a))
    tb = threading.Thread(target=work, args=(eb, imgs_b, alone_b))
    ta.start(); tb.start(); ta.join(); tb.join()
    ea.close(); eb.close()
    assert not errors, errors[0]
    assert int(alone_a[3].sum()) > 0 and int(alone_b[3].sum()) > 0


def test_second_device_engine_matches_first():
    """cudaFuncSetAttribute / SM count are per device: an engine on device 1 needs its own opt-in for the large
    dynamic shared memory of the conv kernel.  Skipped on a single-GPU box."""
    if load_library().lumi_device_count() < 2:
        pytest.skip('needs two visible GPUs')
    cfg = _cfg()
    wts = synth.make_weights(cfg, seed=1)
    imgs = synth.make_images(2, 224, 320, seed=2)
    outs = []
    for dev in (0, 1):
        e = Engine(cfg, device=dev, max_batch=2, max_h=224, max_w=320)
        e.load_weights(wts).finalize()
        outs.append(e.predict_raw(imgs))
        e.close()
    for x, y in zip(*outs):
        np.testing.assert_array_equal(x, y)


@pytest.mark.parametrize('with_rcnn', [True, False])
def test_record_output_equals_packed_outputs(with_rcnn):
    """lumi_set_record_output: the detection kernel writes the all-gather record {count, boxes, scores, labels} itself;
    it must equal parallel.pack_detections of the ordinary outputs (both pipeline halves, RPN-only mode too)."""
    import torch
    cfg = _cfg([] if with_rcnn else ['model.network.with_rcnn=False'])
    wts = synth.make_weights(cfg, seed=1)
    imgs = torch.from_numpy(synth.make_images(3, 160, 224, seed=5)).cuda()
    eng = Engine(cfg, max_batch=3, max_h=160, max_w=224)
    eng.load_weights(wts).finalize()
    K = eng.max_detections
    rec = torch.full((3, P.record_width(K)), -7.0, device='cuda')
    eng.set_record_output(rec)
    boxes = torch.empty((3, K, 4), device='cuda'); scores = torch.empty((3, K), device='cuda')
    labels = torch.empty((3, K), dtype=torch.int32, device='cuda'); counts = torch.empty((3,), dtype=torch.int32, device='cuda')
    eng.predict_device(imgs, boxes, scores, labels, counts)
    eng.synchronize()
    torch.cuda.synchronize()
    want = P.pack_detections(boxes, scores, labels, counts)
    assert torch.equal(rec, want)
    assert int(counts.sum()) > 0
    eng.set_record_output(None)
    rec.fill_(-7.0)
    eng.predict_device(imgs, boxes, scores, labels, counts)
    eng.synchronize()
    torch.cuda.synchronize()
    assert bool((rec == -7.0).all())
    del rec, boxes, scores, labels, counts, imgs
    eng.close()


@pytest.mark.parametrize('model', ['fasterrcnn', 'ssd'])
def test_cuda_graph_replay_is_bit_identical(model):
    """lumi_set_graphs(1): the forward of a shape runs eagerly the first time, is captured the second time and
    replayed afterwards.  Every call must give the eager result bit for bit -- both pipeline halves, the
    stream-K schedule (its flags are cleared by the consumer, so a replay with the captured epoch starts clean),
    after switching to another shape and back, and through the host (H2D staged) and device entry points."""
    import torch
    if model == 'fasterrcnn':
        cfg = _cfg()
        shapes = [(3, 224, 320), (1, 160, 224)]
    else:
        cfg = default_config('ssd', ['model.proposals.min_prob_threshold=0.2'])
        shapes = [(3, 300, 300), (1, 300, 300)]
    wts = synth.make_weights(cfg, seed=1)
    eng = Engine(cfg, max_batch=3, max_h=shapes[0][1], max_w=shapes[0][2])
    eng.load_weights(wts).finalize()
    eng.set_conv_streamk('always')
    batches = [synth.make_images(n, h, w, seed=10 + i) for i, (n, h, w) in enumerate(shapes)]
    eng.set_graphs(False)
    want = [eng.predict_raw(b) for b in batches]
    eng.set_graphs(True)
    for rnd in range(4):
        for b, w_ in zip(batches, want):
            got = eng.predict_raw(b)
            for x, y in zip(got, w_):
                np.testing.assert_array_equal(x, y)
            if rnd >= 2:
                assert eng.last_graph_replays >= 1, 'the forward must be served by a graph replay by now'
    # device entry point: inputs are staged into the engine's buffer, so one graph serves any caller pointer
    K = eng.max_detections
    n = shapes[0][0]
    outs = [torch.empty((n, K, 4), device='cuda'), torch.empty((n, K), device='cuda'),
            torch.empty((n, K), dtype=torch.int32, device='cuda'), torch.empty((n,), dtype=torch.int32, device='cuda')]
    for _ in range(2):
        dimg = torch.from_numpy(batches[0]).cuda()
        eng.predict_device(dimg, *outs)
        eng.synchronize()
        for x, y in zip(outs, want[0]):
            np.testing.assert_array_equal(x.cpu().numpy(), y)
    assert eng.last_graph_replays >= 1
    assert int(want[0][3].sum()) > 0
    del outs, dimg
    eng.close()
