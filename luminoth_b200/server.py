"""``lumi server web`` on the H100 engine -- mirrors ``luminoth/tools/server/web.py`` (SURVEY.md section 8f-4).

Same HTTP surface: ``POST /api/<model_name>/predict/`` with a multipart ``image`` field (optional ``?total=N``)
answers ``{"objects": [{"bbox", "label", "prob"}, ...]}``; ``GET`` on it answers 400 ``Use POST method to send
image.``; a missing / undecodable file answers 400 ``Missing image`` / ``Incompatible file type`` (web.py:31-56).
The model loads on a background thread while the server already listens, and requests wait for it (:53-62); the
caller-side config mutation is ``min_prob_threshold = 0.01`` (:94-103).

What changed underneath: Flask is not in this image, so the server is the standard library's threading HTTP server;
and instead of one ``session.run`` per request, request threads hand their image to a micro-batcher -- requests that
arrive within ``batch_window_ms`` of each other run as ONE ``predict_batch`` call (size-bucketed, up to ``max_batch``
images per engine call).  One engine handle is not re-entrant; the batcher is its only caller.
"""
import io
import json
import re
import threading
import time
from concurrent.futures import Future
from email.parser import BytesParser
from email.policy import HTTP
from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer

import numpy as np

from .config import get_config, override_config_params, set_prediction_filters


class MicroBatcher(object):
    """Collects concurrently submitted images into batched ``predict_batch`` calls."""

    def __init__(self, predict_batch, max_batch=8, batch_window_ms=2.0):
        self._predict_batch = predict_batch
        self._max = int(max_batch)
        self._window = batch_window_ms / 1e3
        self._items = []
        self._cv = threading.Condition()
        self._stop = False
        self.batches = []                       # sizes of the batches run (observability / tests)
        self._thread = threading.Thread(target=self._run, daemon=True)
        self._thread.start()

    def submit(self, image):
        fut = Future()
        with self._cv:
            if self._stop:
                raise RuntimeError('batcher is closed')
            self._items.append((image, fut))
            self._cv.notify()
        return fut

    def predict(self, image):
        return self.submit(image).result()

    def _run(self):
        while True:
            with self._cv:
                while not self._items and not self._stop:
                    self._cv.wait()
                if self._stop and not self._items:
                    return
                deadline = time.monotonic() + self._window
                while len(self._items) < self._max and not self._stop:
                    left = deadline - time.monotonic()
                    if left <= 0:
                        break
                    self._cv.wait(left)
                batch, self._items = self._items[:self._max], self._items[self._max:]
            try:
                results = self._predict_batch([im for im, _ in batch])
                self.batches.append(len(batch))
                for (_, fut), res in zip(batch, results):
                    fut.set_result(res)
            except Exception as e:              # noqa: BLE001 -- every waiting request gets the error
                for _, fut in batch:
                    if not fut.done():
                        fut.set_exception(e)

    def close(self):
        with self._cv:
            self._stop = True
            self._cv.notify_all()
        self._thread.join(5)


def parse_multipart_image(content_type, body):
    """The ``image`` file field of a multipart/form-data body -> raw bytes; ValueError when absent."""
    if not content_type or 'multipart/form-data' not in content_type:
        raise ValueError('Missing image')
    msg = BytesParser(policy=HTTP).parsebytes(b'Content-Type: ' + content_type.encode() + b'\r\n\r\n' + body)
    for part in msg.iter_parts():
        if part.get_param('name', header='content-disposition') == 'image':
            data = part.get_payload(decode=True)
            if data:
                return data
    raise ValueError('Missing image')


INDEX_HTML = (b'<html><body><h3>luminoth_b200</h3><form method="post" enctype="multipart/form-data" '
              b'action="/api/model/predict/"><input type="file" name="image"><input type="submit"></form></body></html>')


class LumiServer(object):
    """The web application object: owns the network (loaded on a background thread) and the batcher."""

    def __init__(self, config, host='127.0.0.1', port=5000, device=0, max_batch=8, batch_window_ms=2.0, weights=None,
                 network_factory=None, pack_sizes=False):
        self.config = set_prediction_filters(config, 0.01, None)         # web.py:94-103
        self.network = None
        self.batcher = None
        self.error = None

        def start_network():
            try:
                if network_factory is not None:
                    self.network = network_factory(self.config)
                else:
                    from .predicting import PredictorNetwork
                    self.network = PredictorNetwork(self.config, weights=weights, device=device, max_batch=max_batch,
                                                    pack_sizes=pack_sizes)
                self.batcher = MicroBatcher(self.network.predict_batch, max_batch, batch_window_ms)
            except Exception as e:               # noqa: BLE001 -- reported to every request (web.py:64-69 kills the server)
                self.error = e

        self.start_thread = threading.Thread(target=start_network, daemon=True)
        self.start_thread.start()
        app = self

        class Handler(BaseHTTPRequestHandler):
            protocol_version = 'HTTP/1.1'

            def log_message(self, *a):          # quiet
                pass

            def _json(self, code, obj):
                data = json.dumps(obj).encode()
                self.send_response(code)
                self.send_header('Content-Type', 'application/json')
                self.send_header('Content-Length', str(len(data)))
                self.end_headers()
                self.wfile.write(data)

            def do_GET(self):
                if re.match(r'^/api/[^/]+/predict/?(\?.*)?$', self.path):
                    return self._json(400, {'error': 'Use POST method to send image.'})
                if self.path in ('/', '/index.html'):
                    self.send_response(200)
                    self.send_header('Content-Type', 'text/html')
                    self.send_header('Content-Length', str(len(INDEX_HTML)))
                    self.end_headers()
                    self.wfile.write(INDEX_HTML)
                    return
                self._json(404, {'error': 'Not found'})

            def do_POST(self):
                m = re.match(r'^/api/[^/]+/predict/?(?:\?(.*))?$', self.path)
                if not m:
                    return self._json(404, {'error': 'Not found'})
                body = self.rfile.read(int(self.headers.get('Content-Length') or 0))
                try:
                    raw = parse_multipart_image(self.headers.get('Content-Type'), body)
                except ValueError:
                    return self._json(400, {'error': 'Missing image'})
                try:
                    from PIL import Image
                    image = np.asarray(Image.open(io.BytesIO(raw)).convert('RGB'))
                except OSError:
                    return self._json(400, {'error': 'Incompatible file type'})
                total = None
                tm = re.search(r'(?:^|&)total=([^&]*)', m.group(1) or '')
                if tm:
                    try:
                        total = int(tm.group(1))
                    except ValueError:
                        total = None
                app.start_thread.join()          # wait for the model to finish loading (web.py:53)
                if app.error is not None:
                    return self._json(500, {'error': 'model failed to load: {}'.format(app.error)})
                try:
                    objects = app.batcher.predict(image)
                except Exception as e:           # noqa: BLE001
                    return self._json(500, {'error': str(e)})
                self._json(200, {'objects': objects[:total]})

        self.httpd = ThreadingHTTPServer((host, port), Handler)
        self.httpd.daemon_threads = True
        self.port = self.httpd.server_address[1]

    def serve_forever(self):
        self.httpd.serve_forever()

    def start(self):
        t = threading.Thread(target=self.httpd.serve_forever, daemon=True)
        t.start()
        return t

    def close(self):
        self.httpd.shutdown()
        self.httpd.server_close()
        self.start_thread.join()
        if self.batcher is not None:
            self.batcher.close()
        if self.network is not None and hasattr(self.network, 'engine'):
            self.network.engine.close()


def main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(prog='lumi-b200 server web', description='Start basic web application.')
    ap.add_argument('--config', '-c', dest='config_files', action='append', required=True)
    ap.add_argument('--override', '-o', dest='override_params', action='append', default=[])
    ap.add_argument('--host', default='127.0.0.1')
    ap.add_argument('--port', default=5000, type=int)
    ap.add_argument('--device', default=0, type=int)
    ap.add_argument('--max-batch', default=8, type=int)
    ap.add_argument('--pack-sizes', action='store_true', help='run images of different preprocessed sizes in one engine call, each at the top left of a shared canvas')
    ap.add_argument('--batch-window-ms', default=2.0, type=float)
    args = ap.parse_args(argv)
    config = get_config(args.config_files)
    if args.override_params:
        config = override_config_params(config, args.override_params)
    srv = LumiServer(config, args.host, args.port, args.device, args.max_batch, args.batch_window_ms,
                     pack_sizes=args.pack_sizes)
    print('listening on http://{}:{}'.format(args.host, srv.port))
    try:
        srv.serve_forever()
    except KeyboardInterrupt:
        pass
    srv.close()


if __name__ == '__main__':
    main()
