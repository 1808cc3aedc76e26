"""Numpy restatement of the cross-window merge of ``lumi_predict_windows`` (DESIGN section 4.2), exact in float32:

1. each window detection is mapped to source pixels, x / s_x + x0 and y / s_y + y0 in float32;
2. per source and label, the candidates are that source's window detections with that label, in window order, then
   rank within the window;
3. each list is sorted by score, descending and stable, and greedy NMS (``tf.image.non_max_suppression``: suppress
   when IoU > thr) keeps at most ``class_max`` of it;
4. the kept lists are concatenated label-major and the top ``total_max`` by score are kept (ties: lower label, then
   earlier kept rank).
"""
import numpy as np

from oracle.tf_ops import non_max_suppression


def map_boxes(boxes, window):
    """(k, 4) float32 (x1, y1, x2, y2) window boxes -> source pixels; window = (y0, x0, s_y, s_x)."""
    y0, x0, sy, sx = (np.float32(v) for v in window)
    b = np.asarray(boxes, np.float32)
    out = np.empty_like(b)
    out[:, 0] = b[:, 0] / sx + x0
    out[:, 1] = b[:, 1] / sy + y0
    out[:, 2] = b[:, 2] / sx + x0
    out[:, 3] = b[:, 3] / sy + y0
    return out


def list_lengths(labels, counts, win_src, nsrc, nc):
    """Candidates per (source, label) list, indexed source * nc + label."""
    n = np.zeros(nsrc * nc, np.int64)
    for k, c in enumerate(counts):
        np.add.at(n, int(win_src[k]) * nc + np.asarray(labels[k][:int(c)], np.int64), 1)
    return n


def plan_groups(lengths):
    """The list groups of ``plan_window_merge``: the lists with candidates, longest first (stable on the list index),
    taken in groups whose first list's length is the group's cap; a group takes max(1, T // cap) lists (T: all
    candidates), or the rest.  Returns [(problems, cap)]."""
    lengths = [int(v) for v in lengths]
    order = sorted((p for p, v in enumerate(lengths) if v), key=lambda p: -lengths[p])
    total = sum(lengths)
    groups, i = [], 0
    while i < len(order):
        cap = lengths[order[i]]
        take = min(len(order) - i, max(1, total // cap))
        groups.append((take, cap))
        i += take
    return groups


def nms_words(n):
    """u64 words of one NMS mask row of an n-candidate list: ceil(n / 64) rounded up to even."""
    return (-(-n // 64) + 1) & ~1


def staged_fits(n):
    """The staged scan takes an n-candidate list when its shared memory (the removed words plus two chunks of 64 mask
    rows) fits in 200 KiB."""
    w = nms_words(n)
    return (w + 2 * 64 * w) * 8 <= 200 * 1024


def nms_path(problems, cap, thr):
    """``nms_path`` with LUMI_NMS_LAZY unset: 0 staged scan, 1 two-phase, 2 unstaged scan."""
    if not staged_fits(cap):
        return 2
    return 1 if cap >= 4096 and 0 < thr < float('inf') and problems >= 3 else 0


def merge_windows(boxes, scores, labels, counts, win_src, wmap, nsrc, nc, class_max, total_max, thr):
    """boxes [nwin][K][4], scores / labels [nwin][K], counts [nwin] (window pixels), win_src [nwin], wmap [nwin] =
    (y0, x0, s_y, s_x).  Returns per source (boxes (m, 4) float32, scores (m,) float32, labels (m,) int32)."""
    out = []
    for s in range(nsrc):
        cb, cs, cl = [], [], []
        for k in range(len(counts)):
            if win_src[k] != s:
                continue
            n = int(counts[k])
            cb.append(map_boxes(boxes[k, :n], wmap[k]))
            cs.append(np.asarray(scores[k, :n], np.float32))
            cl.append(np.asarray(labels[k, :n], np.int32))
        cb = np.concatenate(cb) if cb else np.zeros((0, 4), np.float32)
        cs = np.concatenate(cs) if cs else np.zeros((0,), np.float32)
        cl = np.concatenate(cl) if cl else np.zeros((0,), np.int32)
        kb, ks, kl = [], [], []
        for c in range(nc):
            sel = np.nonzero(cl == c)[0]
            if not len(sel):
                continue
            keep = non_max_suppression(cb[sel], cs[sel], class_max, thr)
            kb.append(cb[sel][keep]); ks.append(cs[sel][keep]); kl.append(np.full(len(keep), c, np.int32))
        if not kb:
            out.append((np.zeros((0, 4), np.float32), np.zeros((0,), np.float32), np.zeros((0,), np.int32)))
            continue
        kb, ks, kl = np.concatenate(kb), np.concatenate(ks), np.concatenate(kl)
        order = np.argsort(-ks, kind='stable')[:total_max]
        out.append((kb[order], ks[order], kl[order]))
    return out
