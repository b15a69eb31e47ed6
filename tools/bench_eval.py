#!/usr/bin/env python
"""Time box + mask mAP on a synthetic COCO-val-like set: 5000 images of 480x640, ~7 gts and 100 detections each, packed masks
already on the device.  Three arms:
  batched    MapEvaluator.add at B=64 over all images + MapEvaluator.ap()
  per_image  the reference's call pattern: prep_metrics once per image (host lists, packed masks) + calc_map
  oracle     oracle/eval_np.py (the plain restatement of the reference's loops) on the CPU over the first --oracle-images images
GPU arms are timed with CUDA events after a synchronise.  The batched and per-image results must be identical, and the batched
result on the oracle's subset must equal the oracle.  Prints one JSON line (GPU name and power limit read in the same run).

    python tools/bench_eval.py [--images 5000] [--batch 64] [--oracle-images 192] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import eval_np as ev  # noqa: E402
from yolact_minimal_b200.utils import common_utils as cu  # noqa: E402
from yolact_minimal_b200.utils.mask_utils import pack_masks  # noqa: E402

THR = [x / 100 for x in range(50, 100, 5)]
C = 80


def rect_bits(rects, h, w, dev):
    r = torch.from_numpy(np.asarray(rects, np.int64).reshape(-1, 4)).to(dev)
    ys = torch.arange(h, device=dev)[None, :, None]
    xs = torch.arange(w, device=dev)[None, None, :]
    m = (xs >= r[:, 0, None, None]) & (xs < r[:, 2, None, None]) & (ys >= r[:, 1, None, None]) & (ys < r[:, 3, None, None])
    return pack_masks(m.to(torch.uint8))


def power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=5000)
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--oracle-images', type=int, default=192)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    D = 100
    t0 = time.perf_counter()
    images = ev.eval_set(2024, num_images=a.images, num_classes=C, dets_per_image=D, sizes=((480, 640),), max_gt=13, empty_image=-1)
    gen_s = time.perf_counter() - t0
    dmasks = [rect_bits(im['det_rects'], im['h'], im['w'], dev) for im in images]
    gmasks = [rect_bits(im['gt_rects'], im['h'], im['w'], dev) for im in images]
    batches = []
    for i in range(0, len(images), a.batch):
        ims = images[i:i + a.batch]
        B = len(ims)
        cls = np.zeros((B, D), np.int32); score = np.zeros((B, D), np.float32); boxes = np.zeros((B, D, 4), np.int32)
        for b, im in enumerate(ims):
            d = len(im['ids'])
            cls[b, :d], score[b, :d], boxes[b, :d] = im['ids'], im['scores'], im['boxes_px']
        t = lambda x: torch.from_numpy(x).to(dev)
        det = {'count': t(np.array([len(im['ids']) for im in ims], np.int32)), 'cls': t(cls), 'score': t(score)}
        gt = t(np.concatenate([im['gt'] for im in ims]))
        off = np.concatenate([[0], np.cumsum([len(im['gt']) for im in ims])]).tolist()
        batches.append((det, t(boxes), dmasks[i:i + B], gt, off, gmasks[i:i + B], [(im['h'], im['w']) for im in ims]))
    per_image = [(list(im['ids'].astype(int)), list(im['scores'].astype(float)), torch.from_numpy(im['boxes_px']).to(dev),
                  torch.from_numpy(im['gt']).to(dev)) for im in images]

    def run_batched(subset=None):
        m = cu.MapEvaluator(C, THR, capacity=len(images) * D)
        for bt in (batches if subset is None else subset):
            m.add(*bt)
        return m.ap()

    def run_per_image():
        ap_data = {'box': [[cu.APDataObject() for _ in range(C)] for _ in THR], 'mask': [[cu.APDataObject() for _ in range(C)] for _ in THR]}
        for k, (ids, scores, boxes, gt) in enumerate(per_image):
            cu.prep_metrics(ap_data, ids, scores, boxes, dmasks[k], gt, gmasks[k], 480, 640, THR)
        return cu.evaluator_of(ap_data).ap()

    def timed(fn, reps=3):
        fn()                                                       # warm-up (allocations, library load)
        best = None
        for _ in range(reps):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            h0 = time.perf_counter()
            e0.record()
            out = fn()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1)
            wall = (time.perf_counter() - h0) * 1e3
            best = (ms, wall, out) if best is None or wall < best[1] else best
        return best

    b_ms, b_wall, b_out = timed(run_batched)
    p_ms, p_wall, p_out = timed(run_per_image, reps=1)
    same = bool(np.array_equal(b_out[0], p_out[0]) and np.array_equal(b_out[1], p_out[1]))
    # oracle on the CPU over the first oracle-images images, and the batched evaluator on the same subset
    n_or = min(a.oracle_images, len(images))
    h0 = time.perf_counter()
    o = ev.EvalOracle(C, THR)
    for im in images[:n_or]:
        o.add_synth(im)
    want = o.ap_array()
    or_s = time.perf_counter() - h0
    sub = batches[:n_or // a.batch]
    got = run_batched(sub) if n_or % a.batch == 0 else None
    match = None if got is None else bool(np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]))
    ndet = sum(len(im['ids']) for im in images)
    ngt = sum(len(im['gt']) for im in images)
    res = {'workload': 'map_eval_synthetic_coco_val', 'gpu': torch.cuda.get_device_name(0), 'power_limit_w': power_limit(),
           'images': len(images), 'detections': ndet, 'gts': ngt, 'img_hw': [480, 640], 'iou_thresholds': len(THR), 'classes': C,
           'batched_B': a.batch, 'batched_ms': round(b_ms, 3), 'batched_wall_ms': round(b_wall, 3),
           'batched_images_per_s': round(len(images) / (b_wall / 1e3), 1),
           'per_image_ms': round(p_ms, 3), 'per_image_wall_ms': round(p_wall, 3),
           'per_image_images_per_s': round(len(images) / (p_wall / 1e3), 1),
           'oracle_cpu_images': n_or, 'oracle_cpu_s': round(or_s, 3), 'oracle_cpu_ms_per_image': round(or_s * 1e3 / n_or, 3),
           'batched_equals_per_image': same, 'batched_equals_oracle_on_subset': match,
           'box_map50': round(float(b_out[0][0, 0][b_out[1]].mean() * 100), 4), 'mask_map50': round(float(b_out[0][1, 0][b_out[1]].mean() * 100), 4),
           'input_generation_s': round(gen_s, 1)}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
