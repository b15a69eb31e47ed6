#!/usr/bin/env python
"""Time the GPU training augmentation (yb_train_aug) on a seeded COCO-like batch.

    python tools/bench_train_aug.py [--batch 64] [--size 550] [--iters 200] [--out profiles/h100_bench_train_aug.json]
    python tools/bench_train_aug.py --cpu-reference DIR     # the reference's own train_aug per image, on the CPU

The batch: B images with sizes drawn from {480x640, 427x640, 640x480, 640x640} and 1-20 elliptical masks each
(oracle/augment_np.synthetic_sample), plans drawn by train_aug_plan under a fixed seed.  The GPU mode times, with
CUDA events, yb_train_aug over many launches, the packed uint8 H2D copy from pinned and from pageable memory, and
train_aug_batch on a pinned batch; it times on the host the pin_memory() copy that the DataLoader's pin thread
makes.  It reports bytes written over kernel time against the data sheet's 3.35 TB/s, plus the host planner's microseconds per image.  Prints one JSON line (GPU name
and power limit read in the same run).  --cpu-reference DIR imports train_aug from the reference checkout at DIR
(needs cv2) and times it per image on the same inputs; it never touches a GPU.
"""
import argparse
import copy
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import augment_np as an  # noqa: E402
from yolact_minimal_b200.utils.augmentations import train_aug_plan  # noqa: E402

SIZES = ((480, 640), (427, 640), (640, 480), (640, 640))
HBM_TBPS = 3.35


def power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def inputs(B, seed=2024):
    rng = random.Random(seed)
    out = []
    for i in range(B):
        h, w = rng.choice(SIZES)
        img, masks, boxes, labels = an.synthetic_sample(5000 + i, h, w, rng.randint(1, 20))
        out.append((img, masks, boxes, labels, rng.randint(0, 10 ** 9)))
    return out


def plans(raw, S):
    samples, t0 = [], time.perf_counter()
    calls = 0
    for img, masks, boxes, labels, seed in raw:
        random.seed(seed)
        while True:
            calls += 1
            p = train_aug_plan(img.shape[0], img.shape[1], boxes, labels, S)
            if p is not None:
                break
        samples.append((img, masks, p))
    return samples, (time.perf_counter() - t0) * 1e6 / calls


def gpu(args):
    import torch
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils.augmentations import PackedTrainBatch, train_aug_batch
    dev = torch.device('cuda:0')
    S, B = args.size, args.batch
    samples, plan_us = plans(inputs(B), S)
    packed = PackedTrainBatch(samples)
    G = int(packed.keep.shape[0])
    L = _lib.lib()
    pageable = packed.buffer
    pin_ms = []
    for _ in range(3):                                # what DataLoader(pin_memory=True)'s pin thread does per batch
        t0 = time.perf_counter()
        host = pageable.pin_memory()
        pin_ms.append((time.perf_counter() - t0) * 1e3)
    pin_ms = min(pin_ms)
    src = torch.empty_like(host, device=dev)
    ws_bytes = int(L.yb_train_aug_workspace_bytes(B, G))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    img = torch.empty(B, 3, S, S, device=dev)
    msk = torch.empty(G, S, S, device=dev)
    stream = torch.cuda.current_stream()
    keep_p = packed.keep_ptr()

    def launch():
        _lib.check(L.yb_train_aug(src.data_ptr(), src.numel(), packed.items_ptr(), B, keep_p, S, ws.data_ptr(), ws_bytes, img.data_ptr(),
                                  msk.data_ptr(), stream.cuda_stream), 'yb_train_aug')

    def timed(fn, iters):
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    h2d_ms = timed(lambda: src.copy_(host, non_blocking=True), args.iters)
    h2d_pageable_ms = timed(lambda: src.copy_(pageable), max(10, args.iters // 10))
    kern_ms = timed(launch, args.iters)
    written = (B * 3 + G) * S * S * 4
    read = packed.buffer.numel()
    pinned = copy.copy(packed)
    pinned.buffer = host
    batch_ms = timed(lambda: train_aug_batch(pinned, S, dev), max(10, args.iters // 10))
    res = {'workload': f'train_aug_B{B}_S{S}_coco_like', 'gpu': torch.cuda.get_device_name(0), 'power_limit_w': power_limit(),
           'batch': B, 'img_size': S, 'masks_out': G, 'src_mb': round(read / 1e6, 2), 'out_mb': round(written / 1e6, 1),
           'kernel_ms': round(kern_ms, 4), 'kernel_gbps_written': round(written / kern_ms / 1e6, 1),
           'frac_of_3.35TBps': round(written / kern_ms / 1e9 / HBM_TBPS, 3), 'bound_ms_at_3.35TBps': round(written / HBM_TBPS / 1e9, 4),
           'h2d_ms': round(h2d_ms, 4), 'h2d_gbps': round(read / h2d_ms / 1e6, 1),
           'h2d_pageable_ms': round(h2d_pageable_ms, 3), 'host_pin_ms': round(pin_ms, 2), 'train_aug_batch_ms_pinned': round(batch_ms, 3), 'planner_us_per_image': round(plan_us, 1),
           'img_per_s_kernel': round(B / kern_ms * 1e3, 0), 'iters': args.iters}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


def cpu_reference(args):
    os.chdir(os.environ.get('TMPDIR', '/tmp'))             # the reference's config.py makes directories in the CWD
    sys.path.insert(0, args.cpu_reference)
    import cv2
    from utils.augmentations import train_aug
    raw = inputs(args.batch)
    _, plan_us = plans(raw, args.size)
    t0 = time.perf_counter()
    n = 0
    for img, masks, boxes, labels, seed in raw:
        random.seed(seed)
        train_aug(img.copy(), masks.copy(), boxes.copy(), labels.copy(), args.size)
        n += 1
    ms = (time.perf_counter() - t0) * 1e3 / n
    print(json.dumps({'workload': f'reference_train_aug_cpu_S{args.size}', 'cpu_count': os.cpu_count(), 'cv2_threads': cv2.getNumThreads(),
                      'images': n, 'ms_per_image': round(ms, 2), 'planner_us_per_image': round(plan_us, 1)}))


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--size', type=int, default=550)
    ap.add_argument('--iters', type=int, default=200)
    ap.add_argument('--out', default=None)
    ap.add_argument('--cpu-reference', default=None)
    a = ap.parse_args()
    cpu_reference(a) if a.cpu_reference else gpu(a)
