"""``lumi eval`` on the H100 engine (SURVEY.md section 8f-3).

Mirrors ``luminoth/eval.py``: the caller-side config mutations (:61-76), the walk over the checkpoints of
``<job_dir>/<run_name>`` (:222-275 ``get_checkpoints``), one pass over ``<dataset.dir>/<split>.tfrecords`` with the
inference preprocessing (``datasets/object_detection_dataset.py:71-139``: decode, resize, ground-truth boxes scaled
with the image, ``utils/image.py:6-35``) and the COCO-style metrics of ``calculate_metrics`` (:487-650): AP@0.50,
AP@0.75, AP@[0.50:0.95], AR@[0.50:0.95].  What is NOT here: the validation *losses* (:122-134) -- they need the
training targets, which are outside the predict path -- and the TensorBoard image summaries.

The record format is TensorFlow's (TFRecord framing + ``tf.train.SequenceExample``), read here without
TensorFlow; ``write_tfrecord`` / ``make_sequence_example`` produce the same bytes as
``tools/dataset/writers/object_detection_writer.py:123-177`` and exist for tests and for building small splits.
The forward pass is the engine's batched call: images are bucketed by preprocessed size (``PredictorNetwork.
predict_batch_raw``), so a split of equally sized images runs ``max_batch`` images per ``lumi_predict``.
"""
import io
import json
import os
import struct
import time

import numpy as np

from .tf_checkpoint import (CheckpointError, _field, _get_varint, _parse_proto, _put_varint, _signed64, crc32c,
                            get_checkpoint_state, mask_crc)


# ---------------------------------------------------------------------------------------------- TFRecord framing
def read_tfrecord(path, verify=True):
    """Yields the payload of every record of a TFRecord file (uint64 length, masked crc32c of the length, payload,
    masked crc32c of the payload -- all little endian)."""
    with open(path, 'rb') as f:
        while True:
            head = f.read(12)
            if not head:
                return
            if len(head) != 12:
                raise CheckpointError('%s: truncated record header' % path)
            length, lcrc = struct.unpack('<QI', head)
            if verify and mask_crc(crc32c(head[:8])) != lcrc:
                raise CheckpointError('%s: corrupted record length' % path)
            data = f.read(length)
            tail = f.read(4)
            if len(data) != length or len(tail) != 4:
                raise CheckpointError('%s: truncated record' % path)
            if verify and mask_crc(crc32c(data)) != struct.unpack('<I', tail)[0]:
                raise CheckpointError('%s: corrupted record payload' % path)
            yield data


def write_tfrecord(path, payloads):
    with open(path, 'wb') as f:
        for data in payloads:
            head = struct.pack('<Q', len(data))
            f.write(head + struct.pack('<I', mask_crc(crc32c(head))) + data + struct.pack('<I', mask_crc(crc32c(data))))


# ---------------------------------------------------------------------------------------------- SequenceExample
def _parse_feature(buf):
    """tf.train.Feature -> list (bytes | float | int)."""
    f = _parse_proto(buf)
    if 1 in f:                                           # BytesList
        return list(_parse_proto(f[1][0]).get(1, []))
    if 3 in f:                                           # Int64List, packed or not
        out = []
        for v in _parse_proto(f[3][0]).get(1, []) if f[3][0] else []:
            if isinstance(v, bytes):
                pos = 0
                while pos < len(v):
                    x, pos = _get_varint(v, pos)
                    out.append(_signed64(x))
            else:
                out.append(_signed64(v))
        return out
    if 2 in f:                                           # FloatList
        out = []
        for v in _parse_proto(f[2][0]).get(1, []) if f[2][0] else []:
            if isinstance(v, bytes):
                out.extend(struct.unpack('<%df' % (len(v) // 4), v))
            else:
                out.append(struct.unpack('<f', struct.pack('<I', v))[0])
        return out
    return []


def parse_sequence_example(buf):
    """-> (context {name: list}, feature_lists {name: [list per step]})  (``tf.parse_single_sequence_example``)."""
    top = _parse_proto(buf)
    context, lists = {}, {}
    for features in top.get(1, []):
        for entry in _parse_proto(features).get(1, []):
            kv = _parse_proto(entry)
            context[kv[1][0].decode()] = _parse_feature(kv.get(2, [b''])[0])
    for fl in top.get(2, []):
        for entry in _parse_proto(fl).get(1, []):
            kv = _parse_proto(entry)
            steps = _parse_proto(kv.get(2, [b''])[0]).get(1, [])
            lists[kv[1][0].decode()] = [_parse_feature(s) for s in steps]
    return context, lists


def _ld(num, payload):
    return _field(num, 2, _put_varint(len(payload)) + payload)


def _int64_feature(values):
    packed = b''.join(_put_varint(int(v)) for v in values)
    return _ld(3, _ld(1, packed))


def _bytes_feature(value):
    return _ld(1, _ld(1, value))


def make_sequence_example(record):
    """The bytes ``ObjectDetectionWriter._record_to_tf`` serialises for ``record`` = {width, height, depth, filename,
    image_raw (encoded image bytes), gt_boxes: [{label, xmin, ymin, xmax, ymax}]}."""
    ctx = b''
    for key in ('width', 'height', 'depth'):
        ctx += _ld(1, _ld(1, key.encode()) + _ld(2, _int64_feature([record[key]])))
    fname = record['filename']
    ctx += _ld(1, _ld(1, b'filename') + _ld(2, _bytes_feature(fname.encode() if isinstance(fname, str) else fname)))
    ctx += _ld(1, _ld(1, b'image_raw') + _ld(2, _bytes_feature(record['image_raw'])))
    fls = b''
    for key in ('label', 'xmin', 'ymin', 'xmax', 'ymax'):
        steps = b''.join(_ld(1, _int64_feature([b[key]])) for b in record['gt_boxes'])
        fls += _ld(1, _ld(1, key.encode()) + _ld(2, steps))
    return _ld(1, ctx) + _ld(2, fls)


# ---------------------------------------------------------------------------------------------- dataset
def decode_image(raw):
    """``tf.image.decode_image(..., channels=3)``: any PIL-readable encoding -> (H, W, 3) uint8 RGB."""
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(raw)).convert('RGB'))


def read_split(dataset_dir, split):
    """Yields (image uint8 HWC, bboxes (n,5) int32 [xmin,ymin,xmax,ymax,label], filename) --
    ``ObjectDetectionDataset.read_record`` (:85-139) without preprocessing."""
    path = os.path.join(dataset_dir, '{}.tfrecords'.format(split))
    if not os.path.exists(path):
        raise ValueError('"{}" does not exist.'.format(path))          # base_dataset.py:37-40
    for payload in read_tfrecord(path):
        ctx, fl = parse_sequence_example(payload)
        image = decode_image(ctx['image_raw'][0])
        h, w = int(ctx['height'][0]), int(ctx['width'][0])
        if image.shape[:2] != (h, w):
            raise ValueError('record %r: image is %s, header says %dx%d' % (ctx['filename'][0], image.shape[:2], h, w))
        cols = [[int(s[0]) for s in fl.get(k, [])] for k in ('xmin', 'ymin', 'xmax', 'ymax', 'label')]
        bboxes = np.array(cols, np.int32).T.reshape(-1, 5)
        yield image, bboxes, ctx['filename'][0].decode()


def adjust_bboxes(bboxes, old_height, old_width, new_height, new_width):
    """``utils/image.py:6-35`` in float32: normalise by the old size, scale by the new FLOAT size, truncate."""
    f32 = np.float32
    b = np.asarray(bboxes).astype(f32)
    out = np.empty(b.shape, np.int32)
    out[:, 0] = np.trunc((b[:, 0] / f32(old_width)) * f32(new_width))
    out[:, 1] = np.trunc((b[:, 1] / f32(old_height)) * f32(new_height))
    out[:, 2] = np.trunc((b[:, 2] / f32(old_width)) * f32(new_width))
    out[:, 3] = np.trunc((b[:, 3] / f32(old_height)) * f32(new_height))
    out[:, 4] = b[:, 4]
    return out


def scaled_ground_truth(shape, bboxes, config):
    """Ground-truth boxes in the coordinates of the preprocessed image (what the model's ``objects`` live in)."""
    f32 = np.float32
    h, w = f32(shape[0]), f32(shape[1])
    ip = config['dataset']['image_preprocessing']
    if ip.get('fixed_height') and ip.get('fixed_width'):
        return adjust_bboxes(bboxes, h, w, f32(ip['fixed_height']), f32(ip['fixed_width']))
    mn, mx = ip.get('min_size'), ip.get('max_size')
    up = max(f32(mn) / min(h, w), f32(1.)) if mn is not None else f32(1.)
    down = min(f32(mx) / max(h, w), f32(1.)) if mx is not None else f32(1.)
    scale = f32(up * down)
    return adjust_bboxes(bboxes, h, w, h * scale, w * scale)            # new size NOT truncated here (image.py:88-103)


# ---------------------------------------------------------------------------------------------- metrics
def bbox_overlap(bboxes1, bboxes2):
    """``utils/bbox_overlap.py:52-94`` (+1 pixel convention, 0 where the boxes do not intersect)."""
    b1 = np.asarray(bboxes1, np.float64).reshape(-1, 4)
    b2 = np.asarray(bboxes2, np.float64).reshape(-1, 4)
    xI1 = np.maximum(b1[:, [0]], b2[:, [0]].T)
    yI1 = np.maximum(b1[:, [1]], b2[:, [1]].T)
    xI2 = np.minimum(b1[:, [2]], b2[:, [2]].T)
    yI2 = np.minimum(b1[:, [3]], b2[:, [3]].T)
    inter = np.maximum(xI2 - xI1 + 1, 0.) * np.maximum(yI2 - yI1 + 1, 0.)
    a1 = (b1[:, [2]] - b1[:, [0]] + 1) * (b1[:, [3]] - b1[:, [1]] + 1)
    a2 = (b2[:, [2]] - b2[:, [0]] + 1) * (b2[:, [3]] - b2[:, [1]] + 1)
    union = (a1 + a2.T) - inter
    iou = np.zeros((b1.shape[0], b2.shape[0]))
    np.divide(inter, union, out=iou, where=inter > 0.)
    return iou


def calculate_metrics(output_per_batch, num_classes):
    """``eval.py:487-650``: per class, greedy highest-score-first matching of detections to ground truth at the IoU
    thresholds 0.50:0.05:0.95, interpolated precision integrated at 101 recall levels.  Returns
    (ap_per_class, ar_per_class), both (num_classes, 10)."""
    iou_thresholds = np.linspace(0.50, 0.95, int(np.round((0.95 - 0.50) / 0.05)) + 1)
    rec_thresholds = np.linspace(0.00, 1.00, int(np.round((1.00 - 0.00) / 0.01)) + 1)
    tp_fp_labels_by_class = [[] for _ in range(num_classes)]
    num_examples_per_class = [0 for _ in range(num_classes)]
    for idx in range(len(output_per_batch['bboxes'])):
        classes = np.asarray(output_per_batch['classes'][idx])
        bboxes = np.asarray(output_per_batch['bboxes'][idx]).reshape(-1, 4)
        scores = np.asarray(output_per_batch['scores'][idx])
        gt_classes = np.asarray(output_per_batch['gt_classes'][idx])
        gt_bboxes = np.asarray(output_per_batch['gt_bboxes'][idx]).reshape(-1, 4)
        for cls in range(num_classes):
            cls_bboxes = bboxes[classes == cls, :]
            cls_scores = scores[classes == cls]
            cls_gt_bboxes = gt_bboxes[gt_classes == cls, :]
            num_gt = cls_gt_bboxes.shape[0]
            num_examples_per_class[cls] += num_gt
            sorted_indices = np.argsort(-cls_scores)
            is_detected = np.zeros((num_gt, len(iou_thresholds)))
            tp_fp_labels = np.zeros((len(sorted_indices), len(iou_thresholds)))
            if num_gt == 0:
                tp_fp_labels_by_class[cls].append((tp_fp_labels, cls_scores[sorted_indices]))
                continue
            ious = bbox_overlap(cls_bboxes, cls_gt_bboxes)
            for bbox_idx in sorted_indices:
                gt_match = np.argmax(ious[bbox_idx, :])
                for iou_idx, iou_threshold in enumerate(iou_thresholds):
                    if ious[bbox_idx, gt_match] >= iou_threshold:
                        if not is_detected[gt_match, iou_idx]:
                            tp_fp_labels[bbox_idx, iou_idx] = True
                            is_detected[gt_match, iou_idx] = True
            tp_fp_labels_by_class[cls].append((tp_fp_labels, cls_scores[sorted_indices]))
    ap_per_class = np.zeros((num_classes, len(iou_thresholds)))
    ar_per_class = np.zeros((num_classes, len(iou_thresholds)))
    for cls in range(num_classes):
        if not tp_fp_labels_by_class[cls]:
            continue
        labels, scores = zip(*tp_fp_labels_by_class[cls])
        labels = np.concatenate(labels)
        scores = np.concatenate(scores)
        num_examples = num_examples_per_class[cls]
        sorted_indices = np.argsort(-scores)
        true_positives = labels[sorted_indices, :]
        false_positives = 1 - true_positives
        cum_tp = np.cumsum(true_positives, axis=0)
        cum_fp = np.cumsum(false_positives, axis=0)
        with np.errstate(divide='ignore', invalid='ignore'):
            recall = cum_tp.astype(float) / num_examples
            precision = np.divide(cum_tp.astype(float), cum_tp + cum_fp)
        for iou_idx in range(len(iou_thresholds)):
            p = precision[:, iou_idx]
            r = recall[:, iou_idx]
            for i in range(len(p) - 1, 0, -1):
                if p[i] > p[i - 1]:
                    p[i - 1] = p[i]
            ap = 0
            for pidx in np.searchsorted(r, rec_thresholds):
                if pidx >= len(r):
                    break
                ap += p[pidx] / len(rec_thresholds)
            ap_per_class[cls, iou_idx] = ap
            ar_per_class[cls, iou_idx] = r[-1] if len(r) else 0
    return ap_per_class, ar_per_class


def summarize_metrics(ap_per_class, ar_per_class):
    """The four scalars ``evaluate_once`` logs (:403-406)."""
    return {'AP@0.50': float(np.mean(ap_per_class[:, 0])), 'AP@0.75': float(np.mean(ap_per_class[:, 5])),
            'AP@[0.50:0.95]': float(np.mean(ap_per_class)), 'AR@[0.50:0.95]': float(np.mean(ar_per_class))}


# ---------------------------------------------------------------------------------------------- checkpoints
def get_checkpoints(run_dir, from_global_step=None, last_only=False):
    """``eval.py:222-275``: [{'global_step', 'file'}] sorted by step; ValueError when there are none."""
    state = get_checkpoint_state(run_dir)
    if not state or not state[1]:
        raise ValueError('Could not find checkpoint in {}.'.format(run_dir))
    checkpoints = sorted([{'global_step': int(path.split('-')[-1]), 'file': path} for path in state[1]],
                         key=lambda c: c['global_step'])
    if last_only:
        checkpoints = checkpoints[-1:]
    elif from_global_step is not None:
        checkpoints = [c for c in checkpoints if c['global_step'] > from_global_step]
    return checkpoints


# ---------------------------------------------------------------------------------------------- evaluation
def prepare_eval_config(config, dataset_split='val', max_detections=100):
    """The config mutations of ``eval.py:50-76``."""
    config.dataset.split = dataset_split
    config.dataset.data_augmentation = []
    if config.model.type == 'fasterrcnn':
        if config.model.network.with_rcnn:
            config.model.rcnn.proposals.total_max_detections = max_detections
        else:
            config.model.rpn.proposals.post_nms_top_n = max_detections
        config.model.rcnn.proposals.min_prob_threshold = 0.0
    elif config.model.type == 'ssd':
        config.model.proposals.total_max_detections = max_detections
        config.model.proposals.min_prob_threshold = 0.0
    else:
        raise ValueError("Model type '{}' not supported".format(config.model.type))
    return config


def evaluate_dataset(network, config, dataset_split='val', batch_size=None, log=None):
    """One pass over the split with an already built ``PredictorNetwork`` -> (metrics dict, ap, ar, n images).
    Detections and ground truth are compared in the preprocessed image's coordinates, like ``evaluate_once``."""
    out = {'bboxes': [], 'classes': [], 'scores': [], 'gt_bboxes': [], 'gt_classes': []}
    num_classes = config.model.network.num_classes
    if config.model.type == 'fasterrcnn' and not config.model.network.with_rcnn:
        num_classes = 1                                                   # eval.py:111-112
    bs = batch_size or network.engine.max_batch
    start = time.time()
    pending_imgs, pending_gt = [], []

    def flush():
        for (boxes, labels, probs, _), gt in zip(network.predict_batch_raw(pending_imgs), pending_gt):
            out['bboxes'].append(boxes); out['classes'].append(labels); out['scores'].append(probs)
            out['gt_bboxes'].append(gt[:, :4]); out['gt_classes'].append(gt[:, 4])
        del pending_imgs[:], pending_gt[:]

    total = 0
    for image, bboxes, _filename in read_split(config.dataset.dir, dataset_split):
        pending_imgs.append(image)
        pending_gt.append(scaled_ground_truth(image.shape, bboxes, config))
        total += 1
        if len(pending_imgs) >= 4 * bs:          # several chunks at once so that size buckets fill whole batches
            flush()
            if log:
                log('{} processed in {:.2f}s ({:.2f} images/s)'.format(total, time.time() - start,
                                                                       total / (time.time() - start)))
    if pending_imgs:
        flush()
    ap, ar = calculate_metrics(out, num_classes)
    metrics = summarize_metrics(ap, ar)
    metrics['total_evaluated'] = total
    metrics['evaluation_time'] = time.time() - start
    return metrics, ap, ar, total


def evaluate(config, dataset_split='val', watch=False, from_global_step=None, max_detections=100, device=0,
             max_batch=8, log=print, poll_seconds=5.0):
    """``lumi eval``: every (or, without ``watch``, the last) checkpoint of ``<job_dir>/<run_name>`` evaluated on the
    split; returns [{'global_step', 'metrics'}].  ``watch=True`` keeps polling for new checkpoints like the reference
    (:168-219)."""
    from .predicting import PredictorNetwork, load_checkpoint_weights
    if not config.train.job_dir:
        raise KeyError('`job_dir` should be set.')
    if not config.train.run_name:
        raise KeyError('`run_name` should be set.')
    run_dir = os.path.join(config.train.job_dir, config.train.run_name)
    config = prepare_eval_config(config, dataset_split, max_detections)
    results = []
    last_global_step = from_global_step
    while True:
        try:
            checkpoints = get_checkpoints(run_dir, last_global_step, last_only=not watch)
        except ValueError:
            if not watch:
                raise
            time.sleep(poll_seconds)
            continue
        for checkpoint in checkpoints:
            log("Evaluating global_step {} using checkpoint '{}'".format(checkpoint['global_step'], checkpoint['file']))
            start = time.time()
            network = PredictorNetwork(config, device=device, max_batch=max_batch,
                                       weights=lambda eng, f=checkpoint['file']: load_checkpoint_weights(eng, None, prefix=f))
            metrics, ap, _ar, total = evaluate_dataset(network, config, dataset_split, log=log)
            network.engine.close()
            last_global_step = checkpoint['global_step']
            log('Finished evaluation at step {}.'.format(checkpoint['global_step']))
            log('Evaluated {} images.'.format(total))
            for key in ('AP@0.50', 'AP@0.75', 'AP@[0.50:0.95]', 'AR@[0.50:0.95]'):
                name = 'Average Recall (AR)' if key.startswith('AR') else 'Average Precision (AP)'
                log('{} @ [{}] = {:.3f}'.format(name, key.split('@')[1].strip('[]'), metrics[key]))
            log('Evaluated in {:.2f}s'.format(time.time() - start))
            results.append({'global_step': checkpoint['global_step'], 'metrics': metrics,
                            'ap_at_50_per_class': ap[:, 0].tolist()})
        if not watch:
            return results
        time.sleep(poll_seconds)


def main(argv=None):
    """``lumi eval`` command line (``eval.py:15-24``); same options except the TensorBoard-only ones."""
    import argparse
    from .config import get_config
    ap = argparse.ArgumentParser(prog='lumi-b200 eval', description='Evaluate trained (or training) models')
    ap.add_argument('--split', dest='dataset_split', default='val', help='Dataset split to use.')
    ap.add_argument('--config', '-c', dest='config_files', action='append', required=True, help='Config to use.')
    ap.add_argument('--watch', dest='watch', action='store_true', default=True)
    ap.add_argument('--no-watch', dest='watch', action='store_false')
    ap.add_argument('--from-global-step', type=int, default=None)
    ap.add_argument('--override', '-o', dest='override_params', action='append', default=[])
    ap.add_argument('--max-detections', type=int, default=100)
    ap.add_argument('--device', type=int, default=0)
    ap.add_argument('--max-batch', type=int, default=8)
    args = ap.parse_args(argv)
    try:
        config = get_config(args.config_files, override_params=args.override_params)
    except KeyError:
        raise KeyError('model.type should be set on the custom config.')
    res = evaluate(config, args.dataset_split, args.watch, args.from_global_step, args.max_detections, args.device,
                   args.max_batch)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
