#!/usr/bin/env python
"""Golden vectors of the mAP stage (TEST INFRASTRUCTURE).  Runs only where a read-only checkout of the reference is named by
$YOLACT_REFERENCE; it writes tests/golden/eval.npz and touches no other fixture.

    python tests/golden/make_golden_eval.py

It imports the UNMODIFIED reference utils/common_utils.py (with stub pycocotools / terminaltables modules in sys.modules: the
functions minted here use neither) and runs eval.py's loop body (:57-69) and calc_map (:106) on CPU tensors for the inputs of
oracle/eval_np.eval_set(seed).  The tests rebuild the inputs from the seeds.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ['YOLACT_REFERENCE']
sys.path.insert(0, ROOT)

from oracle.eval_np import eval_set, rect_masks  # noqa: E402

SEEDS = (1, 2, 3)
NUM_CLASSES = 8
IOU_THRES = [x / 100 for x in range(50, 100, 5)]          # eval.py:24


def import_reference():
    scratch = '/tmp/yolact_ref_cwd'
    os.makedirs(scratch, exist_ok=True)
    os.chdir(scratch)                                        # config.py mkdirs in CWD on import (config.py:6-15)
    sys.modules.setdefault('pycocotools', types.ModuleType('pycocotools'))
    tt = types.ModuleType('terminaltables')
    tt.AsciiTable = lambda rows: types.SimpleNamespace(table='\n'.join(' '.join(str(v) for v in r) for r in rows))
    sys.modules['terminaltables'] = tt
    sys.path.insert(0, REF)
    from utils import common_utils as rcu
    return rcu


def run_case(rcu, seed):
    images = eval_set(seed, num_classes=NUM_CLASSES)
    ap_data = {'box': [[rcu.APDataObject() for _ in range(NUM_CLASSES)] for _ in IOU_THRES],
               'mask': [[rcu.APDataObject() for _ in range(NUM_CLASSES)] for _ in IOU_THRES]}
    for im in images:
        if len(im['ids']) == 0:                              # eval.py:53: after_nms returned None
            continue
        h, w = im['h'], im['w']
        ids_p = list(im['ids'].astype(int))                  # eval.py:57-58
        class_p = list(im['scores'].astype(float))
        boxes_p = torch.from_numpy(im['boxes_px'])
        masks_p = torch.from_numpy(rect_masks(im['det_rects'], h, w).astype(np.float32))
        gt = torch.from_numpy(im['gt'].copy())
        gt_masks = torch.from_numpy(rect_masks(im['gt_rects'], h, w).astype(np.float32))
        rcu.prep_metrics(ap_data, ids_p, class_p, boxes_p, masks_p, gt, gt_masks, h, w, IOU_THRES)
    out = {}
    scores, tps, offs, num_gt, empty = [], [], [0], [], []
    for typ in ('box', 'mask'):
        for t in range(len(IOU_THRES)):
            for c in range(NUM_CLASSES):
                o = ap_data[typ][t][c]
                scores += [p[0] for p in o.data_points]
                tps += [bool(p[1]) for p in o.data_points]
                offs.append(len(scores))
                num_gt.append(o.num_gt_positives)
                empty.append(o.is_empty())
    shape = (2, len(IOU_THRES), NUM_CLASSES)
    aps = [ap_data[typ][t][c].get_ap() for typ in ('box', 'mask') for t in range(len(IOU_THRES)) for c in range(NUM_CLASSES)]
    _, box_row, mask_row = rcu.calc_map(ap_data, IOU_THRES, NUM_CLASSES, step=None)
    p = f'seed{seed}/'
    out[p + 'point_score'] = np.array(scores, np.float64)
    out[p + 'point_tp'] = np.array(tps, bool)
    out[p + 'point_offset'] = np.array(offs, np.int64)
    out[p + 'num_gt'] = np.array(num_gt, np.int64).reshape(shape)
    out[p + 'is_empty'] = np.array(empty, bool).reshape(shape)
    out[p + 'ap'] = np.array(aps, np.float64).reshape(shape)
    out[p + 'box_row'] = np.array(box_row[1:], np.float64)
    out[p + 'mask_row'] = np.array(mask_row[1:], np.float64)
    return out


def make_json_records(rcu):
    """MakeJson.add_bbox (common_utils.py:76-86) on a few detections of eval_set(1)."""
    mj = rcu.MakeJson()
    im = eval_set(1, num_classes=NUM_CLASSES)[3]
    ids, scores = list(im['ids'].astype(int)), list(im['scores'].astype(float))
    for j in range(6):
        mj.add_bbox(1000 + j, ids[j] * 9 % 80, im['boxes_px'][j, :], scores[j])
    rec = mj.bbox_data
    return {'json/image_id': np.array([r['image_id'] for r in rec], np.int64),
            'json/category_id': np.array([r['category_id'] for r in rec], np.int64),
            'json/bbox': np.array([r['bbox'] for r in rec], np.float64),
            'json/score': np.array([r['score'] for r in rec], np.float64)}


def main():
    rcu = import_reference()
    out = {'seeds': np.array(SEEDS, np.int64), 'num_classes': np.array(NUM_CLASSES), 'iou_thres': np.array(IOU_THRES)}
    for s in SEEDS:
        out.update(run_case(rcu, s))
    out.update(make_json_records(rcu))
    np.savez_compressed(os.path.join(HERE, 'eval.npz'), **out)
    print('wrote', os.path.join(HERE, 'eval.npz'), sorted(out))


if __name__ == '__main__':
    main()
