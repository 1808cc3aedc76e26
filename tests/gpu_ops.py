"""numpy-in / numpy-out wrappers over the stand-alone C-ABI operators (GPU tests only).
torch CUDA tensors are just the device containers."""
import ctypes

import numpy as np
import torch

from luminoth_b200 import engine as E


def _lib():
    return E.load_library()


def _dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a if dtype is None else a.astype(dtype)))
    return t.cuda()


def _check(rc):
    if rc != 0:
        raise RuntimeError('op failed (%d): %s' % (rc, _lib().lumi_op_last_error().decode()))


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def conv2d(x, w, stride=1, rate=1, padding='SAME', scale=None, bias=None, residual=None, act=0, impl='simt'):
    lib = _lib()
    n, h, wd, cin = x.shape
    kh, kw, _, cout = w.shape
    pad = {'VALID': 0, 'SAME': 1, 'SLIM': 2}[padding]
    xd, wdv = _dev(x, np.float32), _dev(w, np.float32)
    sd = _dev(scale, np.float32) if scale is not None else None
    bd = _dev(bias, np.float32) if bias is not None else None
    rd = _dev(residual, np.float32) if residual is not None else None
    ho, wo = ctypes.c_int(), ctypes.c_int()
    im = {'simt': 0, 'tc': 1, 'tc_streamk': 2, 'tc_split': 3, 'tc_split_epi16': 4, 'tc_split_epi16_streamk': 5, 'tc_split_cta2': 6, 'tc_split_cta2_streamk': 7,
          'tc_split_halo': 8, 'tc_split_halo_streamk': 9, 'tc_split_halo_cta2': 10, 'tc_split_halo_cta2_streamk': 11}[impl]
    _check(lib.lumi_op_conv2d(_p(xd), n, h, wd, cin, _p(wdv), kh, kw, cout, stride, rate, pad, _p(sd), _p(bd), _p(rd),
                              act, im, None, ctypes.byref(ho), ctypes.byref(wo), None))
    y = torch.empty((n, ho.value, wo.value, cout), dtype=torch.float32, device='cuda')
    _check(lib.lumi_op_conv2d(_p(xd), n, h, wd, cin, _p(wdv), kh, kw, cout, stride, rate, pad, _p(sd), _p(bd), _p(rd),
                              act, im, _p(y), ctypes.byref(ho), ctypes.byref(wo), None))
    torch.cuda.synchronize()
    return y.cpu().numpy()


def max_pool(x, k, stride, padding):
    lib = _lib()
    n, h, w, c = x.shape
    from oracle import tf_ops as T
    if padding == 'SAME':
        ho, wo = T.same_pads(h, k, stride)[0], T.same_pads(w, k, stride)[0]
    else:
        ho, wo = T.valid_out(h, k, stride), T.valid_out(w, k, stride)
    xd = _dev(x, np.float32)
    y = torch.empty((n, ho, wo, c), dtype=torch.float32, device='cuda')
    _check(lib.lumi_op_max_pool(_p(xd), n, h, w, c, k, stride, 1 if padding == 'SAME' else 0, _p(y), None))
    return y.cpu().numpy()


def roi_pool(fmap, rois, im_shape, ph, pw):
    lib = _lib()
    n, fh, fw, c = fmap.shape
    r = rois.shape[0]
    fd, rd = _dev(fmap, np.float32), _dev(rois, np.float32)
    y = torch.empty((r, pw, ph, c), dtype=torch.float32, device='cuda')
    _check(lib.lumi_op_roi_pool(_p(fd), n, fh, fw, c, _p(rd), None, r, float(im_shape[0]), float(im_shape[1]), ph, pw,
                                _p(y), None))
    return y.cpu().numpy()


def roi_kernel(c, ph, pw):
    return _lib().lumi_roi_kernel(c, ph, pw)


def roi_pool_batched(fmap, rois, counts, im_shape, ph, pw, kernel=-1, pooled=True, mean=True):
    """fmap [n, fh, fw, c], rois [n, rmax, 4], counts [n] or None -> (pooled [n*rmax, pw, ph, c] or None,
    mean [n*rmax, c] or None) as CUDA float32 tensors.  fmap / rois may be numpy arrays or CUDA tensors."""
    lib = _lib()
    n, fh, fw, c = fmap.shape
    rmax = rois.shape[1]
    fd = fmap if torch.is_tensor(fmap) else _dev(fmap, np.float32)
    rd = rois if torch.is_tensor(rois) else _dev(rois, np.float32)
    cd = _dev(np.asarray(counts), np.int32) if counts is not None else None
    y = torch.empty((n * rmax, pw, ph, c), dtype=torch.float32, device='cuda') if pooled else None
    m = torch.empty((n * rmax, c), dtype=torch.float32, device='cuda') if mean else None
    _check(lib.lumi_op_roi_pool_batched(_p(fd), n, fh, fw, c, _p(rd), _p(cd), rmax, float(im_shape[0]),
                                        float(im_shape[1]), ph, pw, kernel, _p(y), _p(m), None))
    return y, m


def spatial_mean(x):
    """x [r, h, w, c] -> [r, c] through the split planes."""
    lib = _lib()
    r, h, w, c = x.shape
    xd = _dev(x, np.float32)
    y = torch.empty((r, c), dtype=torch.float32, device='cuda')
    _check(lib.lumi_op_spatial_mean(_p(xd), r, h, w, c, _p(y), None))
    return y.cpu().numpy()


def softmax_rows(x, cols):
    """x [rows, in_stride] -> softmax of the first cols entries of each row, [rows, cols]."""
    lib = _lib()
    rows, stride = x.shape
    xd = _dev(x, np.float32)
    y = torch.empty((rows, cols), dtype=torch.float32, device='cuda')
    _check(lib.lumi_op_softmax_rows(_p(xd), rows, cols, stride, _p(y), None))
    return y.cpu().numpy()


def sort_desc(scores):
    lib = _lib()
    sd = _dev(scores, np.float32)
    idx = torch.empty((scores.shape[0],), dtype=torch.int32, device='cuda')
    _check(lib.lumi_op_sort_desc(_p(sd), scores.shape[0], _p(idx), None))
    return idx.cpu().numpy()


def nms_sorted(boxes, thr, max_out):
    lib = _lib()
    bd = _dev(boxes, np.float32)
    keep = torch.full((max_out,), -1, dtype=torch.int32, device='cuda')
    nk = torch.zeros((1,), dtype=torch.int32, device='cuda')
    _check(lib.lumi_op_nms_sorted(_p(bd), boxes.shape[0], float(thr), max_out, _p(keep), _p(nk), None))
    k = int(nk.cpu()[0])
    return keep.cpu().numpy()[:k]


def nms_path(problems, ncap, thr):
    return _lib().lumi_nms_path(problems, ncap, float(thr))


def nms_batched(boxes, nvalid, thr, max_out):
    """boxes [P, cap, 4] sorted lists, nvalid [P] -> list of P keep-index arrays."""
    lib = _lib()
    P, cap, _ = boxes.shape
    bd, nd = _dev(boxes, np.float32), _dev(np.asarray(nvalid), np.int32)
    keep = torch.full((P, max_out), -1, dtype=torch.int32, device='cuda')
    nk = torch.zeros((P,), dtype=torch.int32, device='cuda')
    _check(lib.lumi_op_nms_batched(_p(bd), _p(nd), P, cap, float(thr), max_out, _p(keep), _p(nk), None))
    keep, nk = keep.cpu().numpy(), nk.cpu().numpy()
    return [keep[p, :nk[p]] for p in range(P)]


def rpn_proposals_batched(heads, A, anchors, na, cap, im_shape, cfg, logits=True, cls_off=0, box_off=None):
    """heads [nimg, cells, hc]: the engine's fused head, class pair of anchor a at cls_off + 2a, deltas at
    box_off + 4a (default 2A).  Returns (proposals [nimg, post, 4], scores [nimg, post], counts [nimg])."""
    lib = _lib()
    nimg, cells, hc = heads.shape
    assert cells * A == na
    post = int(cfg['post_nms_top_n'])
    hd, ad = _dev(heads, np.float32), _dev(anchors, np.float32)
    props = torch.zeros((nimg, post, 4), dtype=torch.float32, device='cuda')
    scores = torch.zeros((nimg, post), dtype=torch.float32, device='cuda')
    cnt = torch.zeros((nimg,), dtype=torch.int32, device='cuda')
    _check(lib.lumi_op_rpn_proposals_batched(
        _p(hd), _p(hd), cells * hc, cells * hc, A, _p(ad), nimg, na, cap, float(im_shape[0]), float(im_shape[1]),
        int(cfg['pre_nms_top_n']), post, float(cfg['nms_threshold']), float(cfg.get('min_prob_threshold', 0.0)),
        int(bool(cfg.get('filter_outside_anchors', False))), int(bool(cfg.get('clip_after_nms', False))),
        int(bool(cfg.get('apply_nms', True))), int(logits), hc, cls_off, hc, 2 * A if box_off is None else box_off,
        _p(props), _p(scores), _p(cnt), None))
    return props.cpu().numpy(), scores.cpu().numpy(), cnt.cpu().numpy()


def class_detections_batched(boxes_in, boxes_img_stride, row_counts, deltas, delta_stride, cls_prob, nimg, r, nc,
                             im_shape, cfg, variances, shared_deltas, records=False):
    """boxes_in / deltas / cls_prob: flat float32 arrays in the engine's layouts (see lumi_op_class_detections_batched).
    Returns (objects [nimg, tm, 4], labels, probs [nimg, tm], counts [nimg], records [nimg, 1 + 6 tm] or None)."""
    lib = _lib()
    tm, cm = int(cfg['total_max_detections']), int(cfg['class_max_detections'])
    bd, dd, pd = _dev(boxes_in, np.float32), _dev(deltas, np.float32), _dev(cls_prob, np.float32)
    rc = _dev(np.asarray(row_counts), np.int32) if row_counts is not None else None
    obj = torch.zeros((nimg, tm, 4), dtype=torch.float32, device='cuda')
    lab = torch.zeros((nimg, tm), dtype=torch.int32, device='cuda')
    prob = torch.zeros((nimg, tm), dtype=torch.float32, device='cuda')
    cnt = torch.zeros((nimg,), dtype=torch.int32, device='cuda')
    rec = torch.full((nimg, 1 + 6 * tm), np.nan, dtype=torch.float32, device='cuda') if records else None
    v = variances or [1., 1.]
    _check(lib.lumi_op_class_detections_batched(
        _p(bd), boxes_img_stride, _p(rc), _p(dd), _p(pd), nimg, r, nc, float(im_shape[0]), float(im_shape[1]),
        float(v[0]), float(v[1]), float(cfg.get('min_prob_threshold') or 0.0), float(cfg['class_nms_threshold']), cm, tm,
        int(shared_deltas), nc + 1, delta_stride, _p(obj), _p(lab), _p(prob), _p(cnt), _p(rec), None))
    return (obj.cpu().numpy(), lab.cpu().numpy(), prob.cpu().numpy(), cnt.cpu().numpy(),
            rec.cpu().numpy() if records else None)


def rpn_proposals(cls_prob, bbox_pred, anchors, im_shape, cfg):
    lib = _lib()
    na = cls_prob.shape[0]
    post = int(cfg['post_nms_top_n'])
    cd, bd, ad = _dev(cls_prob, np.float32), _dev(bbox_pred, np.float32), _dev(anchors, np.float32)
    props = torch.zeros((post, 4), dtype=torch.float32, device='cuda')
    scores = torch.zeros((post,), dtype=torch.float32, device='cuda')
    cnt = torch.zeros((1,), dtype=torch.int32, device='cuda')
    _check(lib.lumi_op_rpn_proposals(_p(cd), _p(bd), _p(ad), na, float(im_shape[0]), float(im_shape[1]),
                                     int(cfg['pre_nms_top_n']), post, float(cfg['nms_threshold']),
                                     float(cfg.get('min_prob_threshold', 0.0)),
                                     int(bool(cfg.get('filter_outside_anchors', False))),
                                     int(bool(cfg.get('clip_after_nms', False))), _p(props), _p(scores), _p(cnt), None))
    k = int(cnt.cpu()[0])
    return props.cpu().numpy()[:k], scores.cpu().numpy()[:k]


def class_detections(boxes_in, deltas, cls_prob, im_shape, nc, cfg, variances, ssd=False):
    lib = _lib()
    r = boxes_in.shape[0]
    tm, cm = int(cfg['total_max_detections']), int(cfg['class_max_detections'])
    bd, dd, pd = _dev(boxes_in, np.float32), _dev(deltas, np.float32), _dev(cls_prob, np.float32)
    obj = torch.zeros((tm, 4), dtype=torch.float32, device='cuda')
    lab = torch.zeros((tm,), dtype=torch.int32, device='cuda')
    prob = torch.zeros((tm,), dtype=torch.float32, device='cuda')
    cnt = torch.zeros((1,), dtype=torch.int32, device='cuda')
    v = variances or [1., 1.]
    _check(lib.lumi_op_class_detections(_p(bd), _p(dd), _p(pd), r, nc, float(im_shape[0]), float(im_shape[1]),
                                        float(v[0]), float(v[1]), float(cfg.get('min_prob_threshold') or 0.0),
                                        float(cfg['class_nms_threshold']), cm, tm, int(ssd), _p(obj), _p(lab), _p(prob),
                                        _p(cnt), None))
    k = int(cnt.cpu()[0])
    return obj.cpu().numpy()[:k], lab.cpu().numpy()[:k], prob.cpu().numpy()[:k]


def resize_bilinear(image, nh, nw):
    lib = _lib()
    is_f32 = image.dtype != np.uint8
    src = _dev(image, np.float32 if is_f32 else np.uint8)
    dst = torch.empty((nh, nw, 3), dtype=torch.float32, device='cuda')
    _check(lib.lumi_op_resize_bilinear(_p(src), int(is_f32), image.shape[0], image.shape[1], _p(dst), nh, nw, None))
    return dst.cpu().numpy()
