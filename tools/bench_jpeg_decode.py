#!/usr/bin/env python
"""JPEG decoding on the device (yb_jpeg_decode_batch) against cv2.imread on the host.

Files are the three photos of tests/golden/ resized (INTER_AREA) to 480x640, 640x480 and 427x640 and re-encoded by cv2 at q 95 in
4:2:0 and 4:4:4, cycled through batches of 8, 32 and 64.  For each: time of one decode call (CUDA events around it on its stream,
so the host's header parse and staging are included; median of --iters after --warmup; the H2D copy of the file bytes excluded), the images/s, compressed MB/s in and raw GB/s out that implies, the
worst number of synchronisation rounds of the Huffman decode in the batch, and the H2D bytes saved against copying the pixels.
Every decoded image is checked against cv2.imread first.  cv2.imread's time per image on this host (one thread, median) is
measured for each size and layout.  Prints one JSON line (GPU name and power limit read in the same run) and writes it to --out.

    python tools/bench_jpeg_decode.py [--iters 20] [--warmup 3] [--out profiles/h100_bench_jpeg_decode.json]
"""
import argparse
import ctypes
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from bench_val import power_limit  # noqa: E402
import jpeg_decode_corpus  # noqa: E402
from yolact_minimal_b200 import _lib  # noqa: E402
from yolact_minimal_b200.utils.augmentations import VAL_ITEM_DTYPE, imdecode_batched, jpeg_header  # noqa: E402

BATCHES = (8, 32, 64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=os.path.join(ROOT, 'profiles', 'h100_bench_jpeg_decode.json'))
    args = ap.parse_args()
    import cv2
    cv2.setNumThreads(1)
    dev = torch.device('cuda')
    files = jpeg_decode_corpus.photo_files()
    groups = {}
    for name, data in files:
        key = name.split('_', 1)[1]                   # '{h}x{w}_{layout}'
        groups.setdefault(key, []).append(data)
    result = {'gpu': torch.cuda.get_device_name(0), 'power_limit_w': power_limit(), 'quality': 95,
              'content': 'tests/golden photos resized (INTER_AREA) and re-encoded by cv2', 'gpu_decode': {},
              'cv2_imread_ms_per_image': {}}
    tmp = tempfile.mkdtemp()
    worst_rounds = 0
    for key, datas in groups.items():
        paths = []
        for i, d in enumerate(datas):
            p = os.path.join(tmp, f'{key}_{i}.jpg')
            with open(p, 'wb') as f:
                f.write(d)
            paths.append(p)
        ts = []
        for _ in range(max(args.iters, 5)):
            for p in paths:
                t0 = time.perf_counter()
                cv2.imread(p)
                ts.append(time.perf_counter() - t0)
        result['cv2_imread_ms_per_image'][key] = round(1e3 * float(np.median(ts)), 3)
        want = [cv2.imread(p) for p in paths]
        for bs in BATCHES:
            batch = [datas[i % len(datas)] for i in range(bs)]
            src = torch.from_numpy(np.concatenate([np.frombuffer(d, np.uint8) for d in batch])).pin_memory()
            src_off = np.concatenate([[0], np.cumsum([len(d) for d in batch])]).astype(np.int64)
            items = np.zeros(bs, VAL_ITEM_DTYPE)
            o = 0
            for i, d in enumerate(batch):
                h, w = jpeg_header(np.frombuffer(d, np.uint8))
                items[i] = (o, h, w)
                o += h * w * 3
            out, status = imdecode_batched(src, src_off, items, dev)
            got = out.cpu().numpy()
            assert np.all(status.cpu().numpy() == 0), key
            for i in range(bs):
                off, h, w = items[i].tolist()
                assert np.array_equal(got[off:off + h * w * 3].reshape(h, w, 3), want[i % len(want)]), (key, bs, i)
            # timed calls on a workspace of our own: its first bs int32 hold the synchronisation rounds afterwards
            L = _lib.lib()
            host = src.numpy()
            off_p = src_off.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))
            ws_bytes = int(L.yb_jpeg_decode_workspace_bytes(host.ctypes.data, off_p, bs))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            st = torch.empty(bs, dtype=torch.int32, device=dev)
            src_d = src.to(dev)
            call = lambda: _lib.check(L.yb_jpeg_decode_batch(host.ctypes.data, src_d.data_ptr(), off_p, bs,
                                                             items.ctypes.data_as(ctypes.POINTER(_lib.ValAugItem)), out.data_ptr(),
                                                             out.numel(), ws.data_ptr(), ws_bytes, st.data_ptr(),
                                                             torch.cuda.current_stream().cuda_stream), 'decode')
            for _ in range(args.warmup):
                call()
            torch.cuda.synchronize()
            times = []
            for _ in range(args.iters):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                call()
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
            rounds = ws[:4 * bs].view(torch.int32).cpu().numpy()
            worst_rounds = max(worst_rounds, int(rounds.max()))
            ms = float(np.median(times))
            comp, raw = int(src_off[-1]), int(o)
            result['gpu_decode'][f'{key}@{bs}'] = {
                'ms': round(ms, 4), 'images_per_s': round(bs / ms * 1e3, 1), 'compressed_mb_per_s_in': round(comp / ms / 1e3, 1),
                'raw_gb_per_s_out': round(raw / ms / 1e6, 2), 'max_sync_rounds': int(rounds.max()),
                'mean_sync_rounds': round(float(rounds.mean()), 2), 'h2d_bytes_files': comp, 'h2d_bytes_pixels': raw,
                'h2d_bytes_saved': raw - comp}
    result['max_sync_rounds'] = worst_rounds
    line = json.dumps(result)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        f.write(line + '\n')


if __name__ == '__main__':
    main()
