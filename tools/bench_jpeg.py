#!/usr/bin/env python
"""JPEG encoding on the device (yb_jpeg_encode_batch) against cv2.imencode on the host, quality 95 (cv2's default).

Images are the three photos of tests/golden/ resized (INTER_LINEAR) to each size and cycled through the batch.  For batches of 32
and 64 images at 480x640, 640x480, 427x640 and 1080x1920: GPU time of one encode call (CUDA events, median of --iters after
--warmup), the images/s and raw input bytes/s that implies, and the mean file size.  Every GPU file is checked against
cv2.imencode first.  cv2.imencode's time per image on this host (one thread, median) is measured at each size.  Prints one JSON
line (GPU name and power limit read in the same run) and writes it to --out.

    python tools/bench_jpeg.py [--iters 20] [--warmup 3] [--out profiles/h100_bench_jpeg.json]
"""
import argparse
import glob
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from bench_val import power_limit  # noqa: E402
from yolact_minimal_b200.utils.augmentations import pack_images  # noqa: E402
from yolact_minimal_b200.utils.output_utils import imencode_batched  # noqa: E402

SIZES = ((480, 640), (640, 480), (427, 640), (1080, 1920))
BATCHES = (32, 64)
Q = 95


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100_bench_jpeg.json'))
    args = ap.parse_args()
    import cv2
    cv2.setNumThreads(1)
    photos = [cv2.imread(p) for p in sorted(glob.glob(os.path.join(ROOT, 'tests', 'golden', '0*.jpg')))]
    dev = torch.device('cuda')
    result = {'gpu': torch.cuda.get_device_name(0), 'power_limit_w': power_limit(), 'quality': Q,
              'content': 'tests/golden photos resized to each size', 'gpu_encode': {}, 'cv2_imencode_ms_per_image': {}}
    for h, w in SIZES:
        imgs = [cv2.resize(p, (w, h), interpolation=cv2.INTER_LINEAR) for p in photos]
        ts = []
        for _ in range(max(args.iters, 5)):
            for img in imgs:
                t0 = time.perf_counter()
                cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, Q])
                ts.append(time.perf_counter() - t0)
        result['cv2_imencode_ms_per_image'][f'{h}x{w}'] = round(1e3 * float(np.median(ts)), 3)
        for bs in BATCHES:
            batch = [imgs[i % len(imgs)] for i in range(bs)]
            buf, items = pack_images(batch)
            src = buf.to(dev)
            data, off, lens = imencode_batched(src, items, Q)
            got, lens = data.cpu().numpy(), lens.cpu().numpy()
            for i, img in enumerate(batch[:len(imgs)]):
                assert got[off[i]:off[i] + lens[i]].tobytes() == cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, Q])[1].tobytes()
            for _ in range(args.warmup):
                imencode_batched(src, items, Q)
            ms = []
            for _ in range(args.iters):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                imencode_batched(src, items, Q)
                b.record()
                b.synchronize()
                ms.append(a.elapsed_time(b))
            t = float(np.median(ms))
            result['gpu_encode'][f'{h}x{w}_bs{bs}'] = {
                'ms_per_batch': round(t, 3), 'images_per_s': round(bs / t * 1e3, 1),
                'input_gb_per_s': round(bs * h * w * 3 / t / 1e6, 2), 'mean_file_bytes': int(lens.mean())}
    line = json.dumps(result)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        f.write(line + '\n')


if __name__ == '__main__':
    main()
