"""Box and mask mAP restated in plain numpy / Python (TEST INFRASTRUCTURE): utils/common_utils.py:107-255 as eval.py:35-69,:106
drive them, pinned to tests/golden/eval.npz.  The GPU tests use it at sizes beyond the goldens.

Masks are given either densely (uint8 [n,h,w]) or as the filled pixel rectangles of eval_set below, whose IoUs are exact
integer areas -- the same counts the reference's fp32 matmul of {0,1} masks produces below 2^24 pixels.
"""
import bisect

import numpy as np

from . import postprocess_np as pp, synth

F32 = np.float32


def box_iou(boxes_px, gt, h, w):
    """prep_metrics' box IoU (common_utils.py:175-183): gt in [0,1] scaled in fp32 (x by w, y by h) vs the int pixel boxes."""
    gb = np.asarray(gt, F32)[:, :4].copy()
    gb[:, [0, 2]] *= F32(w)
    gb[:, [1, 3]] *= F32(h)
    return pp.box_iou(np.asarray(boxes_px).astype(F32)[None], gb[None])[0]


def _iou_from_counts(inter, ca, cb):
    fi = inter.astype(F32)
    with np.errstate(invalid='ignore', divide='ignore'):
        return (fi / ((ca.astype(F32)[:, None] + cb.astype(F32)[None, :]) - fi)).astype(F32)


def mask_iou_dense(dm, gm):
    dm, gm = np.asarray(dm), np.asarray(gm)
    a = dm.reshape(len(dm), int(np.prod(dm.shape[1:]))).astype(np.int64)
    b = gm.reshape(len(gm), int(np.prod(gm.shape[1:]))).astype(np.int64)
    return _iou_from_counts(a @ b.T, a.sum(1), b.sum(1))


def mask_iou_rects(dr, gr):
    a = np.asarray(dr, np.int64).reshape(-1, 4)
    b = np.asarray(gr, np.int64).reshape(-1, 4)
    area = lambda r: np.maximum(r[:, 2] - r[:, 0], 0) * np.maximum(r[:, 3] - r[:, 1], 0)
    iw = np.maximum(np.minimum(a[:, None, 2], b[None, :, 2]) - np.maximum(a[:, None, 0], b[None, :, 0]), 0)
    ih = np.maximum(np.minimum(a[:, None, 3], b[None, :, 3]) - np.maximum(a[:, None, 1], b[None, :, 1]), 0)
    return _iou_from_counts(iw * ih, area(a), area(b))


def eval_set(seed, num_images=5, num_classes=8, dets_per_image=24, sizes=((333, 500), (480, 640)), max_gt=6, empty_image=2):
    """Deterministic synthetic inputs of eval.py's loop body (after_nms outputs + ground truth), drawn from oracle/synth.py's
    counter-based generator.  Per image a dict:
    h, w; ids [d] int64 (0-based class) and scores [d] float32 in the given detection order; boxes_px [d,4] int32 pixel boxes;
    det_rects [d,4] int32 mask rectangles [x1,y1,x2,y2) in pixels; gt [g,5] float32 ([0,1] box, class); gt_rects [g,4] int32.
    Masks are filled rectangles (rect_masks), so exact mask IoUs are also integer rectangle areas.
    Covers: detections that are jittered copies of gts (IoU ~0.4-1.0), duplicates, wrong-class detections and pure false
    positives, scores quantised to 1/20 (ties within and across images), IoUs of exactly 11/20, 12/20 and 16/20 for boxes and
    masks (fp32(x) > x / 100 in double but not in fp32) in class C-3, zero-area boxes and empty masks (NaN IoUs), a class with
    only gts (C-2) and one with only detections (C-1), and image `empty_image` without detections."""
    out = []
    C = num_classes
    for k in range(num_images):
        h, w = sizes[k % len(sizes)]
        u = lambda stream, shape: synth.uniform(seed, 1000 * k + stream, shape)
        g = 1 + int(u(1, ())[()] * max_gt) if max_gt > 0 else 0
        x1 = np.floor(u(2, (g,)) * (w * 0.6)).astype(np.int64)
        y1 = np.floor(u(3, (g,)) * (h * 0.6)).astype(np.int64)
        x2 = np.minimum(x1 + 8 + np.floor(u(4, (g,)) * (w * 0.35)).astype(np.int64), w)
        y2 = np.minimum(y1 + 8 + np.floor(u(5, (g,)) * (h * 0.35)).astype(np.int64), h)
        gcls = np.floor(u(6, (g,)) * (C - 3)).astype(np.int64)
        gt_px = np.stack([x1, y1, x2, y2], 1)
        gt_rects = np.stack([x1 + 1, y1, np.maximum(x2 - 1, x1 + 1), y2], 1)
        if k == 0:                      # a gt of the gt-only class
            gcls[-1] = C - 2
        ids, boxes, rects = [], [], []
        nd = 0 if k == empty_image else dets_per_image
        r = u(7, (max(nd, 1), 8))
        for i in range(nd):
            j = int(r[i, 0] * g)
            if r[i, 1] < 0.15:          # pure false positive
                bx = np.floor(r[i, 2:6] * np.array([w * 0.7, h * 0.7, w * 0.3, h * 0.3])).astype(np.int64)
                b = np.array([bx[0], bx[1], bx[0] + 4 + bx[2], bx[1] + 4 + bx[3]])
                c = int(r[i, 6] * (C - 3)) if r[i, 7] < 0.8 else C - 1
            else:                       # jittered copy (duplicates when j repeats), sometimes with the wrong class
                bw, bh = gt_px[j, 2] - gt_px[j, 0], gt_px[j, 3] - gt_px[j, 1]
                jit = (r[i, 2:6] - 0.5) * 0.5 * np.array([bw, bh, bw, bh])
                b = np.round(gt_px[j] + jit).astype(np.int64)
                c = int(gcls[j]) if r[i, 6] > 0.12 else int((gcls[j] + 1) % (C - 3))
            b = np.clip(b, 0, [w, h, w, h])
            b[2], b[3] = max(b[2], b[0]), max(b[3], b[1])
            mr = b + np.round((r[i, [3, 4, 5, 2]] - 0.5) * 4).astype(np.int64)
            mr = np.clip(mr, 0, [w, h, w, h])
            mr[2], mr[3] = max(mr[2], mr[0]), max(mr[3], mr[1])
            ids.append(c); boxes.append(b); rects.append(mr)
        scores = (np.floor(u(8, (nd,)) * 20) / 20 + 0.05).astype(np.float32)
        if nd and k in (0, 1):
            # exact-threshold pairs in class C-3: gt box 20 x 15 px at the image corner (w = 640, h = 480 keep gt * size exact),
            # gt mask 20 x 1 px; detections [0,0,11,15] (box 0.55) with mask 12 px (0.6), [0,0,16,15] (0.8) with 11 px (0.55)
            gpx = np.array([[0, 0, 20, 15]])
            gt_px = np.concatenate([gt_px, gpx]); gt_rects = np.concatenate([gt_rects, [[0, 0, 20, 1]]])
            gcls = np.concatenate([gcls, [C - 3]])
            ids[0], boxes[0], rects[0] = C - 3, np.array([0, 0, 11, 15]), np.array([0, 0, 12, 1])
            ids[1], boxes[1], rects[1] = C - 3, np.array([0, 0, 16, 15]), np.array([0, 0, 11, 1])
            # zero-area gt with an empty mask, a zero-area detection with an empty mask (0/0 = NaN for both IoU types)
            gt_px = np.concatenate([gt_px, [[30, 30, 30, 40]]]); gt_rects = np.concatenate([gt_rects, [[30, 30, 30, 40]]])
            gcls = np.concatenate([gcls, [C - 3]])
            ids[2], boxes[2], rects[2] = C - 3, np.array([30, 30, 30, 40]), np.array([30, 30, 30, 40])
        gt = np.concatenate([gt_px[:, [0, 2]] / w, gt_px[:, [1, 3]] / h], 1)[:, [0, 2, 1, 3]]
        gt = np.concatenate([gt, gcls[:, None]], 1).astype(np.float32)
        out.append({'h': h, 'w': w, 'ids': np.array(ids, np.int64), 'scores': scores,
                    'boxes_px': np.array(boxes, np.int64).reshape(-1, 4).astype(np.int32),
                    'det_rects': np.array(rects, np.int64).reshape(-1, 4).astype(np.int32), 'gt': gt,
                    'gt_rects': np.asarray(gt_rects, np.int64).reshape(-1, 4).astype(np.int32)})
    return out


def rect_masks(rects, h, w):
    """Filled rectangles [x1,y1,x2,y2) -> uint8 masks [n,h,w]."""
    ys, xs = np.arange(h)[None, :, None], np.arange(w)[None, None, :]
    r = np.asarray(rects, np.int64).reshape(-1, 4)
    return ((xs >= r[:, 0, None, None]) & (xs < r[:, 2, None, None]) & (ys >= r[:, 1, None, None]) & (ys < r[:, 3, None, None])).astype(np.uint8)


class EvalOracle:
    """ap_data of the reference: per (type, threshold, class) the pushed (score, is_true) points and the gt count."""

    def __init__(self, num_classes, iou_thres):
        self.C, self.thr = num_classes, list(iou_thres)
        T = len(self.thr)
        self.points = [[[[] for _ in range(num_classes)] for _ in range(T)] for _ in range(2)]
        self.num_gt = np.zeros((2, T, num_classes), np.int64)

    def add_image(self, ids, scores, box_iou_m, mask_iou_m, gt_classes):
        """One image of eval.py's loop: ids / scores in detection order, [d,g] fp32 IoU matrices, gt classes."""
        ids = [int(c) for c in ids]
        if len(ids) == 0:                                   # eval.py:53: no prep_metrics, the gts are never counted
            return
        gt_classes = [int(c) for c in gt_classes]
        scores = [float(s) for s in scores]
        for c in set(ids + gt_classes):
            ngt = gt_classes.count(c)
            for t, thr in enumerate(self.thr):
                for typ, iou in enumerate((box_iou_m, mask_iou_m)):
                    used = [False] * len(gt_classes)
                    self.num_gt[typ, t, c] += ngt
                    pts = self.points[typ][t][c]
                    for i, pc in enumerate(ids):
                        if pc != c:
                            continue
                        best, bj = thr, -1
                        for j, gc in enumerate(gt_classes):
                            if used[j] or gc != c:
                                continue
                            v = float(iou[i, j])
                            if v > best:
                                best, bj = v, j
                        if bj >= 0:
                            used[bj] = True
                        pts.append((scores[i], bj >= 0))

    def add_synth(self, im, dense=False):
        """An image of eval_set."""
        if dense:
            miou = mask_iou_dense(rect_masks(im['det_rects'], im['h'], im['w']), rect_masks(im['gt_rects'], im['h'], im['w']))
        else:
            miou = mask_iou_rects(im['det_rects'], im['gt_rects'])
        self.add_image(im['ids'], im['scores'], box_iou(im['boxes_px'], im['gt'], im['h'], im['w']), miou,
                       np.asarray(im['gt'])[:, 4].astype(np.int32))

    def is_empty(self, typ, t, c):
        return len(self.points[typ][t][c]) == 0 and self.num_gt[typ, t, c] == 0

    def get_ap(self, typ, t, c):
        ngt = int(self.num_gt[typ, t, c])
        if ngt == 0:
            return 0.0
        pts = sorted(self.points[typ][t][c], key=lambda x: -x[0])        # stable: ties keep push order
        prec, rec, nt = [], [], 0
        for k, (_, tp) in enumerate(pts):
            nt += bool(tp)
            prec.append(nt / (k + 1))
            rec.append(nt / ngt)
        for i in range(len(prec) - 1, 0, -1):
            prec[i - 1] = max(prec[i - 1], prec[i])
        y = [0] * 101
        for x in range(101):
            idx = bisect.bisect_left(rec, x / 100)                      # np.searchsorted(recalls, x / 100, side='left')
            if idx < len(prec):
                y[x] = prec[idx]
        return sum(y) / len(y)                                          # Python's sum(): compensated (Neumaier) since 3.12

    def ap_array(self):
        T = len(self.thr)
        ap = np.array([[[self.get_ap(typ, t, c) for c in range(self.C)] for t in range(T)] for typ in range(2)], np.float64)
        nonempty = np.array([not self.is_empty(0, 0, c) for c in range(self.C)])
        return ap, nonempty


def map_rows(ap, nonempty, iou_thres):
    """calc_map's rows (common_utils.py:219-255) from ap [2,T,C] and nonempty [C]: per threshold the mean over non-empty classes
    (x 100), 'all' = mean of the thresholds, each rounded to 2 places."""
    rows = []
    for typ, name in enumerate(('box', 'mask')):
        maps = []
        for t in range(len(iou_thres)):
            vals = [float(ap[typ, t, c]) for c in range(ap.shape[2]) if nonempty[c]]
            maps.append(sum(vals) / len(vals) * 100 if vals else 0)
        rows.append([name] + [round(v, 2) for v in [sum([0] + maps) / len(maps)] + maps])
    return rows[0], rows[1]
