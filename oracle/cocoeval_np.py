"""COCO's own mAP (pycocotools' COCOeval with its default Params, iouType 'bbox' and 'segm') restated in plain Python / numpy
(TEST INFRASTRUCTURE).  Written from the evaluation rules, not from pycocotools' source: per (image, category, area range) the
greedy matching of the score-sorted detections against the ignore-sorted gts, then per (category, area range, maxDets) the
cross-image precision / recall scan sampled at 101 recall thresholds.  The CUDA path (csrc/cocoeval.cu behind
utils/cocoeval.CocoEvaluator) must equal it bit for bit.

    gts  list of {'image_id', 'category' (0-based), 'bbox' [x,y,w,h] float, 'area' float, 'iscrowd', 'mask' or 'rect'} in
         annotation-file order
    dts  list of {'image_id', 'category', 'bbox' [x,y,w,h], 'score', 'mask' or 'rect'} in the order they were produced
    precision, recall = evaluate(gts, dts, img_ids, num_classes, 'bbox' | 'segm')

A mask is a dense {0,1} array [h,w] ('mask') or a filled pixel rectangle x1,y1,x2,y2 ('rect'); a rectangle's pixel counts are
exact integer areas, so both give the same IoUs.
"""
from collections import defaultdict

import numpy as np

IOU_THRS = np.linspace(.5, .95, 10)
REC_THRS = np.linspace(0, 1, 101)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0, 1e10], [0, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e10]]
EPS = np.spacing(1)


def _counts(d, g):
    """(|d & g|, |d|, |g|) of two masks."""
    if 'rect' in d:
        a, b = [int(v) for v in d['rect']], [int(v) for v in g['rect']]
        area = lambda r: max(r[2] - r[0], 0) * max(r[3] - r[1], 0)
        inter = max(min(a[2], b[2]) - max(a[0], b[0]), 0) * max(min(a[3], b[3]) - max(a[1], b[1]), 0)
        return inter, area(a), area(b)
    dm, gm = np.asarray(d['mask'], bool), np.asarray(g['mask'], bool)
    return int(np.count_nonzero(dm & gm)), int(np.count_nonzero(dm)), int(np.count_nonzero(gm))


def iou(d, g, iou_type):
    """IoU of detection d and gt g; a crowd gt divides by the detection's own area."""
    crowd = bool(g['iscrowd'])
    if iou_type == 'bbox':
        dx, dy, dw, dh = (float(v) for v in d['bbox'])
        gx, gy, gw, gh = (float(v) for v in g['bbox'])
        w = min(dx + dw, gx + gw) - max(dx, gx)
        if w <= 0:
            return 0.0
        h = min(dy + dh, gy + gh) - max(dy, gy)
        if h <= 0:
            return 0.0
        i = w * h
        u = dw * dh if crowd else dw * dh + gw * gh - i
        return i / u
    i, cd, cg = _counts(d, g)
    if i == 0:
        return 0.0
    u = cd if crowd else cd + cg - i
    return float(i) / float(u)


def det_area(d, iou_type):
    if iou_type == 'bbox':
        return float(d['bbox'][2]) * float(d['bbox'][3])
    if 'rect' in d:
        return float(_counts(d, d)[1])
    return float(np.count_nonzero(d['mask']))


def _evaluate_img(gt, dt, ious, a_rng, iou_type):
    """One (image, category, area range): dt in score order (already truncated), gt in annotation order, ious[d][g] in those
    orders.  The gts are stably reordered with the non-ignored ones first."""
    if not gt and not dt:
        return None
    lo, hi = a_rng
    g_ign = [1 if g['iscrowd'] or g['area'] < lo or g['area'] > hi else 0 for g in gt]
    gtind = list(np.argsort(g_ign, kind='mergesort'))
    g_ign = [g_ign[i] for i in gtind]
    iscrowd = [int(bool(gt[i]['iscrowd'])) for i in gtind]
    T, G, D = len(IOU_THRS), len(gt), len(dt)
    gtm = np.zeros((T, G), bool)
    dtm = np.zeros((T, D), bool)
    dt_ig = np.zeros((T, D), bool)
    for tind, t in enumerate(IOU_THRS):
        for dind in range(D):
            best = min(t, 1 - 1e-10)
            m = -1
            for gind in range(G):
                if gtm[tind, gind] and not iscrowd[gind]:
                    continue
                if m > -1 and g_ign[m] == 0 and g_ign[gind] == 1:
                    break
                v = ious[dind][gtind[gind]]
                if v < best:
                    continue
                best, m = v, gind
            if m == -1:
                continue
            dt_ig[tind, dind] = g_ign[m]
            dtm[tind, dind] = True
            gtm[tind, m] = True
    outside = np.array([det_area(d, iou_type) < lo or det_area(d, iou_type) > hi for d in dt], bool).reshape(1, D)
    dt_ig = dt_ig | (~dtm & outside)
    return {'scores': np.array([d['score'] for d in dt], np.float64), 'dtm': dtm, 'dt_ig': dt_ig, 'g_ign': np.array(g_ign, int)}


def evaluate(gts, dts, img_ids, num_classes, iou_type):
    """-> (precision [10,101,K,4,3], recall [10,K,4,3]) float64, -1 where no non-ignored gt exists."""
    img_ids = sorted(img_ids)
    by_gt, by_dt = defaultdict(list), defaultdict(list)
    for g in gts:
        by_gt[g['image_id'], g['category']].append(g)
    for d in dts:
        by_dt[d['image_id'], d['category']].append(d)
    K, A, M, T, R = num_classes, len(AREA_RNG), len(MAX_DETS), len(IOU_THRS), len(REC_THRS)
    evals = {}
    for img in img_ids:
        for k in range(K):
            gt, dt = by_gt.get((img, k), []), by_dt.get((img, k), [])
            if not gt and not dt:
                continue
            order = np.argsort([-float(d['score']) for d in dt], kind='mergesort')
            dt = [dt[i] for i in order[:MAX_DETS[-1]]]
            ious = [[iou(d, g, iou_type) for g in gt] for d in dt]
            for a, rng in enumerate(AREA_RNG):
                evals[img, k, a] = _evaluate_img(gt, dt, ious, rng, iou_type)
    precision = -np.ones((T, R, K, A, M))
    recall = -np.ones((T, K, A, M))
    for k in range(K):
        for a in range(A):
            E = [evals[img, k, a] for img in img_ids if evals.get((img, k, a)) is not None]
            if not E:
                continue
            for m, max_det in enumerate(MAX_DETS):
                scores = np.concatenate([e['scores'][:max_det] for e in E])
                inds = np.argsort(-scores, kind='mergesort')
                dtm = np.concatenate([e['dtm'][:, :max_det] for e in E], axis=1)[:, inds]
                dt_ig = np.concatenate([e['dt_ig'][:, :max_det] for e in E], axis=1)[:, inds]
                npig = int(np.count_nonzero(np.concatenate([e['g_ign'] for e in E]) == 0))
                if npig == 0:
                    continue
                tp_sum = np.cumsum(dtm & ~dt_ig, axis=1).astype(np.float64)
                fp_sum = np.cumsum(~dtm & ~dt_ig, axis=1).astype(np.float64)
                for t in range(T):
                    tp, fp = tp_sum[t], fp_sum[t]
                    nd = len(tp)
                    rc = tp / npig
                    pr = (tp / (fp + tp + EPS)).tolist()
                    recall[t, k, a, m] = rc[-1] if nd else 0
                    for i in range(nd - 1, 0, -1):
                        if pr[i] > pr[i - 1]:
                            pr[i - 1] = pr[i]
                    q = np.zeros(R)
                    for r, pi in enumerate(np.searchsorted(rc, REC_THRS, side='left')):
                        if pi < nd:
                            q[r] = pr[pi]
                    precision[t, :, k, a, m] = q
    return precision, recall

