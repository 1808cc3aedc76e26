"""``lumi predict`` on the H100 engine -- mirrors ``luminoth/predict.py`` (SURVEY.md section 8f-2 / 8f-4).

Same command line, same JSON lines (``{"file": ..., "objects": [{"bbox", "label", "prob"}]}``), same caller-side
config mutations (``--min-prob`` / ``--max-detections`` written into the config before the network is built,
``predict.py:246-259``).  What changed underneath:

* images of a run are decoded up front and sent through ``PredictorNetwork.predict_batch`` -- bucketed by
  preprocessed size, ``max_batch`` images per engine call -- instead of one ``session.run`` per file (:83);
* video frames are read ``max_batch`` at a time and predicted as one batch (:135 predicts frame by frame);
  reading / writing uses OpenCV (``skvideo`` + ffmpeg are not in this image);
* JPEG files can be decoded on the GPU with nvJPEG (``--decode nvjpeg``, ``lumi_decode_jpeg``); the default stays
  PIL like the reference (:72-79), because the two decoders differ by +-1..2 grey levels on chroma edges and the
  reference's detections are defined on PIL's pixels.
"""
import json
import os
import sys
import time

import numpy as np

from .config import get_config, override_config_params, set_prediction_filters

IMAGE_FORMATS = ['jpg', 'jpeg', 'png']
VIDEO_FORMATS = ['mov', 'mp4', 'avi']


def get_file_type(filename):
    extension = filename.split('.')[-1].lower()
    if extension in IMAGE_FORMATS:
        return 'image'
    elif extension in VIDEO_FORMATS:
        return 'video'


def resolve_files(path_or_dir):
    """``predict.py:28-55``: files of the accepted formats; directories are listed (not recursed)."""
    if not isinstance(path_or_dir, (tuple, list)):
        path_or_dir = (path_or_dir,)
    paths = []
    for entry in path_or_dir:
        if os.path.isdir(entry):
            paths.extend([os.path.join(entry, f) for f in sorted(os.listdir(entry))
                          if get_file_type(f) in ('image', 'video')])
        elif get_file_type(entry) in ('image', 'video'):
            if not os.path.exists(entry):
                print('Input {} not found, skipping.'.format(entry))
                continue
            paths.append(entry)
    return paths


def filter_classes(objects, only_classes=None, ignore_classes=None):
    if ignore_classes:
        objects = [o for o in objects if o['label'] not in ignore_classes]
    if only_classes:
        objects = [o for o in objects if o['label'] in only_classes]
    return objects


def load_image(path, decode='pil', device=0):
    """(H, W, 3) uint8 RGB.  ``decode='nvjpeg'``: baseline/progressive JPEG decoded on the GPU (other formats and any
    nvJPEG failure fall back to PIL -- a decoder choice, not a compute fallback)."""
    if decode == 'nvjpeg' and path.lower().endswith(('.jpg', '.jpeg')):
        from .engine import decode_jpeg
        with open(path, 'rb') as f:
            data = f.read()
        try:
            return decode_jpeg(data, device=device)
        except RuntimeError:
            pass
    from PIL import Image
    with open(path, 'rb') as f:
        return np.asarray(Image.open(f).convert('RGB'))


def draw_objects(image, objects):
    """Minimal stand-in for ``luminoth.vis.vis_objects`` (visualisation is out of scope): boxes + 'label prob'."""
    from PIL import Image, ImageDraw
    im = Image.fromarray(np.asarray(image, np.uint8))
    d = ImageDraw.Draw(im)
    for o in objects:
        x1, y1, x2, y2 = o['bbox']
        d.rectangle([min(x1, x2), min(y1, y2), max(x1, x2), max(y1, y2)], outline=(255, 64, 64), width=2)
        d.text((x1 + 2, y1 + 2), '{} {:.2f}'.format(o['label'], o['prob']), fill=(255, 255, 255))
    return im


def predict_images(network, paths, only_classes=None, ignore_classes=None, save_dir=None, decode='pil', echo=print):
    """All image files of a run as batched engine calls; returns [(path, objects or None)] in input order."""
    images, ok_paths, results = [], [], {}
    for path in paths:
        try:
            images.append(load_image(path, decode, network.engine.device))
            ok_paths.append(path)
        except OSError as e:
            echo('Error while processing {}: {}'.format(path, e))
            results[path] = None
    for path, image, objects in zip(ok_paths, images, network.predict_batch(images)):
        objects = filter_classes(objects, only_classes=only_classes, ignore_classes=ignore_classes)
        if save_dir:
            draw_objects(image, objects).save(os.path.join(save_dir, 'pred_{}'.format(os.path.basename(path))))
        results[path] = objects
        echo('Predicting {}... done.'.format(path))
    return [(p, results[p]) for p in paths]


def predict_image(network, path, only_classes=None, ignore_classes=None, save_path=None):
    """``predict.py:66-97`` for one file."""
    try:
        image = load_image(path)
    except OSError as e:
        print('Error while processing {}: {}'.format(path, e))
        return
    objects = filter_classes(network.predict_image(image), only_classes=only_classes, ignore_classes=ignore_classes)
    if save_path:
        draw_objects(image, objects).save(save_path)
    return objects


def predict_video(network, path, only_classes=None, ignore_classes=None, save_path=None, echo=print):
    """``predict.py:100-171`` with frame batching: ``max_batch`` consecutive frames per engine call.  Returns
    [{'frame': idx, 'objects': [...]}]."""
    import cv2
    cap = cv2.VideoCapture(path)
    if not cap.isOpened():
        raise RuntimeError('could not open video {}'.format(path))
    writer = None
    if save_path:
        save_path = os.path.splitext(save_path)[0] + '.mp4'          # hard-coded to mp4 like the reference (:104)
    else:
        echo('Video not being saved. Note that for the time being, no JSON output is being generated. '
             'Did you mean to specify `--save-path`?')
    objects_per_frame = []
    bs = network.engine.max_batch
    start_time = time.time()
    idx = 0
    while True:
        frames = []
        while len(frames) < bs:
            ok, frame = cap.read()
            if not ok:
                break
            frames.append(np.ascontiguousarray(frame[:, :, ::-1]))    # BGR -> RGB
        if not frames:
            break
        for frame, objects in zip(frames, network.predict_batch(frames)):
            objects = filter_classes(objects, only_classes=only_classes, ignore_classes=ignore_classes)
            objects_per_frame.append({'frame': idx, 'objects': objects})
            if save_path:
                if writer is None:
                    h, w = frame.shape[:2]
                    fps = cap.get(cv2.CAP_PROP_FPS) or 25.0
                    writer = cv2.VideoWriter(save_path, cv2.VideoWriter_fourcc(*'mp4v'), fps, (w, h))
                writer.write(np.asarray(draw_objects(frame, objects))[:, :, ::-1])
            idx += 1
    cap.release()
    if writer is not None:
        writer.release()
    echo('fps: {0:.1f}'.format(idx / max(time.time() - start_time, 1e-9)))
    return objects_per_frame


def main(argv=None):
    import argparse
    from .predicting import PredictorNetwork
    ap = argparse.ArgumentParser(prog='lumi-b200 predict', description="Obtain a model's predictions.")
    ap.add_argument('path_or_dir', nargs='*')
    ap.add_argument('--config', '-c', dest='config_files', action='append', default=[], help='Config to use.')
    ap.add_argument('--override', '-o', dest='override_params', action='append', default=[])
    ap.add_argument('--output', '-f', dest='output_path', default='-')
    ap.add_argument('--save-media-to', '-d')
    ap.add_argument('--min-prob', default=0.5, type=float)
    ap.add_argument('--max-detections', default=100, type=int)
    ap.add_argument('--only-class', '-k', action='append', default=None)
    ap.add_argument('--ignore-class', '-K', action='append', default=None)
    ap.add_argument('--max-batch', default=8, type=int, help='images / frames per engine call')
    ap.add_argument('--decode', default='pil', choices=['pil', 'nvjpeg'])
    ap.add_argument('--device', default=0, type=int)
    args = ap.parse_args(argv)
    if args.only_class and args.ignore_class:
        print('Only one of `only-class` or `ignore-class` may be specified.')
        return
    files = resolve_files(tuple(args.path_or_dir))
    if not files:
        print('No files to predict found. Accepted formats are: {}.'.format(', '.join(IMAGE_FORMATS + VIDEO_FORMATS)))
        return
    print('Found {} files to predict.'.format(len(files)), file=sys.stderr)
    if not args.config_files:
        # the reference falls back to the downloadable `accurate` checkpoint (predict.py:236-241); there is no
        # network here, so a config is required
        raise SystemExit('a --config is required (remote checkpoints are not available)')
    config = get_config(args.config_files)
    if args.override_params:
        config = override_config_params(config, args.override_params)
    config = set_prediction_filters(config, args.min_prob, args.max_detections)
    output = sys.stdout if args.output_path == '-' else open(args.output_path, 'w')
    if args.save_media_to:
        os.makedirs(args.save_media_to, exist_ok=True)
    network = PredictorNetwork(config, device=args.device, max_batch=args.max_batch)
    image_files = [f for f in files if get_file_type(f) == 'image']
    echo = lambda m: print(m, file=sys.stderr)
    for path, objects in predict_images(network, image_files, args.only_class, args.ignore_class, args.save_media_to,
                                        args.decode, echo):
        if objects is not None:
            output.write(json.dumps({'file': path, 'objects': objects}) + '\n')
    for path in files:
        if get_file_type(path) == 'video':
            save_path = os.path.join(args.save_media_to, 'pred_{}'.format(os.path.basename(path))) if args.save_media_to else None
            predict_video(network, path, args.only_class, args.ignore_class, save_path, echo)
    if output is not sys.stdout:
        output.close()
    network.engine.close()


if __name__ == '__main__':
    main()
