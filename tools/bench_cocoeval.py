#!/usr/bin/env python
"""Time COCO's own mAP (CocoEvaluator: csrc/cocoeval.cu) on a synthetic COCO-val-like set: 5000 images of 480x640 / 640x480, ~7
annotations each (some crowd, areas over small / medium / large), 100 detections each, detection masks packed on the device.
  gpu      CocoEvaluator.add at B=64 over all images + accumulate() + summarize(), CUDA events after a synchronise
  oracle   oracle/cocoeval_np.py (the plain restatement of COCOeval's loops) on the CPU over the first --oracle-images images,
           and the GPU path on the same subset, which must give identical arrays
  pycocotools  not measured when it is not importable
Prints one JSON line with the GPU name and power limit read in the same run.

    python tools/bench_cocoeval.py [--images 5000] [--batch 64] [--oracle-images 192] [--out FILE]
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import cocoeval_np as ce  # noqa: E402
from yolact_minimal_b200.utils.cocoeval import CocoEvaluator  # noqa: E402
from yolact_minimal_b200.utils.mask_utils import pack_masks, pack_masks_host  # noqa: E402

K, D = 80, 100
IDENTITY = {k + 1: k + 1 for k in range(K)}


def power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def rect_bits(rects, h, w, dev):
    r = torch.from_numpy(np.asarray(rects, np.int64).reshape(-1, 4)).to(dev)
    ys = torch.arange(h, device=dev)[None, :, None]
    xs = torch.arange(w, device=dev)[None, None, :]
    m = (xs >= r[:, 0, None, None]) & (xs < r[:, 2, None, None]) & (ys >= r[:, 1, None, None]) & (ys < r[:, 3, None, None])
    return pack_masks(m.to(torch.uint8))


def make_images(seed, n):
    rng = np.random.RandomState(seed)
    images = []
    for b in range(n):
        h, w = ((480, 640), (640, 480))[b % 2]
        pool = rng.randint(0, K, size=8)
        gts = []
        for _ in range(max(1, rng.poisson(7))):
            side = int(rng.choice([rng.randint(4, 32), rng.randint(32, 96), rng.randint(96, 300)]))   # small / medium / large
            bw, bh = min(side + rng.randint(-3, 4), w), min(side, h)
            bw = max(bw, 1)
            x1, y1 = rng.randint(0, w - bw + 1), rng.randint(0, h - bh + 1)
            gts.append({'cls': int(rng.choice(pool)), 'bbox': [x1 + .5 * rng.randint(2), y1 + 0.0, bw - .5 * rng.randint(2), bh + 0.0],
                        'area': float(bw * bh - rng.randint(0, 3)), 'crowd': int(rng.rand() < .05), 'rect': (x1, y1, x1 + bw, y1 + bh)})
        dets = []
        for _ in range(D):
            g = gts[rng.randint(len(gts))]['rect']
            if rng.rand() < .5:
                j = rng.randint(-6, 7, size=4)
                x1, y1 = int(np.clip(g[0] + j[0], 0, w - 1)), int(np.clip(g[1] + j[1], 0, h - 1))
                x2, y2 = int(np.clip(g[2] + j[2], x1 + 1, w)), int(np.clip(g[3] + j[3], y1 + 1, h))
            else:
                x1, y1 = rng.randint(0, w - 1), rng.randint(0, h - 1)
                x2, y2 = rng.randint(x1 + 1, w + 1), rng.randint(y1 + 1, h + 1)
            dets.append({'cls': int(rng.choice(pool)), 'score': np.float32(rng.randint(1, 1000) / 1000), 'box': (x1, y1, x2, y2)})
        images.append({'id': 1000 + 7 * b, 'h': h, 'w': w, 'gts': gts, 'dets': dets})
    return images


class Batch:
    """What CocoEvaluator.add reads of a PackedValBatch, page-locked as DataLoader(pin_memory=True) leaves it."""

    def __init__(self, ims):
        self.ids, self.sizes = [im['id'] for im in ims], [(im['h'], im['w']) for im in ims]
        g = [im['gts'] for im in ims]
        self.ann_offset = np.concatenate([[0], np.cumsum([len(x) for x in g])]).astype(int).tolist()
        self.ann_cls = torch.tensor([a['cls'] for x in g for a in x], dtype=torch.int32).pin_memory()
        self.ann_box = torch.tensor([a['bbox'] for x in g for a in x], dtype=torch.float64).reshape(-1, 4).pin_memory()
        self.ann_area = torch.tensor([a['area'] for x in g for a in x], dtype=torch.float64).pin_memory()
        self.ann_crowd = torch.tensor([a['crowd'] for x in g for a in x], dtype=torch.int32).pin_memory()
        bits = []
        for im in ims:
            m = np.zeros((len(im['gts']), im['h'], im['w']), np.uint8)
            for i, a in enumerate(im['gts']):
                x1, y1, x2, y2 = a['rect']
                m[i, y1:y2, x1:x2] = 1
            bits.append(pack_masks_host(m))
        self.ann_mask_off = np.concatenate([[0], np.cumsum([x.size for x in bits])]).astype(int).tolist()
        self.ann_masks = torch.from_numpy(np.concatenate([x.reshape(-1) for x in bits])).pin_memory()

    def __len__(self):
        return len(self.ids)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=5000)
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--oracle-images', type=int, default=192)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    t0 = time.perf_counter()
    images = make_images(2024, a.images)
    batches = []
    for i in range(0, len(images), a.batch):
        ims = images[i:i + a.batch]
        B = len(ims)
        cls = np.zeros((B, D), np.int32); score = np.zeros((B, D), np.float32); boxes = np.zeros((B, D, 4), np.int32)
        for b, im in enumerate(ims):
            for j, d in enumerate(im['dets']):
                cls[b, j], score[b, j], boxes[b, j] = d['cls'], d['score'], d['box']
        t = lambda x: torch.from_numpy(x).to(dev)
        det = {'count': t(np.full(B, D, np.int32)), 'cls': t(cls), 'score': t(score)}
        masks = [rect_bits([d['box'] for d in im['dets']], im['h'], im['w'], dev) for im in ims]
        batches.append((det, t(boxes), masks, Batch(ims)))
    gen_s = time.perf_counter() - t0

    def coco():
        class C:
            imgToAnns = {im['id']: [{'category_id': g['cls'] + 1, 'area': g['area'], 'iscrowd': g['crowd']} for g in im['gts']]
                         for im in images}
        return C()

    def run(sub):
        ev = CocoEvaluator(coco(), IDENTITY, dev, capacity=len(images) * D)
        for bt in sub:
            ev.add(*bt)
        with contextlib.redirect_stdout(io.StringIO()):
            stats = ev.summarize()
        return ev.accumulate(), stats

    run(batches[:2])                                               # warm-up: library load, allocations, CUB
    best = None
    for _ in range(3):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        h0 = time.perf_counter()
        e0.record()
        out, stats = run(batches)
        e1.record()
        torch.cuda.synchronize()
        ms, wall = e0.elapsed_time(e1), (time.perf_counter() - h0) * 1e3
        best = (ms, wall, out, stats) if best is None or wall < best[1] else best
    g_ms, g_wall, _, stats = best

    # oracle on the CPU over the first oracle-images images (whole batches), against the GPU path on the same images; the
    # annotation set stays the whole set, so the images never added still count as gts to find
    nb = max(1, a.oracle_images // a.batch)
    sub = images[:nb * a.batch]
    gts = [{'image_id': im['id'], 'category': g['cls'], 'bbox': g['bbox'], 'area': g['area'], 'iscrowd': g['crowd'], 'rect': g['rect']}
           for im in images for g in im['gts']]
    dts = [{'image_id': im['id'], 'category': d['cls'], 'bbox': [d['box'][0], d['box'][1], d['box'][2] - d['box'][0], d['box'][3] - d['box'][1]],
            'score': float(d['score']), 'rect': d['box']} for im in sub for d in im['dets']]
    h0 = time.perf_counter()
    want = {t: ce.evaluate(gts, dts, [im['id'] for im in images], K, t) for t in ('bbox', 'segm')}
    or_s = time.perf_counter() - h0
    got, _ = run(batches[:nb])
    match = all(np.array_equal(got[t]['precision'], want[t][0]) and np.array_equal(got[t]['recall'], want[t][1]) for t in want)
    try:
        import pycocotools  # noqa: F401
        pyc = 'importable, not timed by this tool'
    except ImportError:
        pyc = 'not measured (pycocotools not importable)'
    res = {'workload': 'cocoeval_synthetic_coco_val', 'gpu': torch.cuda.get_device_name(0), 'power_limit_w': power_limit(),
           'images': len(images), 'detections': len(images) * D, 'annotations': sum(len(im['gts']) for im in images),
           'crowd': sum(g['crowd'] for im in images for g in im['gts']), 'img_hw': [[480, 640], [640, 480]], 'classes': K, 'batch': a.batch,
           'gpu_ms': round(g_ms, 3), 'gpu_wall_ms': round(g_wall, 3), 'gpu_images_per_s': round(len(images) / (g_wall / 1e3), 1),
           'oracle_cpu_images': len(sub), 'oracle_cpu_s': round(or_s, 3), 'oracle_cpu_ms_per_image': round(or_s * 1e3 / len(sub), 3),
           'gpu_equals_oracle_on_subset': bool(match), 'pycocotools': pyc,
           'bbox_ap': round(float(stats[0][0]), 6), 'segm_ap': round(float(stats[1][0]), 6), 'input_generation_s': round(gen_s, 1)}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')
    if not match:
        sys.exit('GPU result differs from the oracle on the subset')


if __name__ == '__main__':
    main()
