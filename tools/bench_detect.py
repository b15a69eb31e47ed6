#!/usr/bin/env python
"""Batched detection (python -m yolact_minimal_b200.detect) against the reference's per-image loop (tests/detect_loop.py), res101_coco
550 fp16 with synthetic weights, visual_thre 0.3 (detect.py's default):

  images   256 JPEGs of 480x640 / 640x480 / 427x640 in a temporary folder, read, detected, drawn and JPEG-encoded to results/images
  video    a 1080x1920 MJPG clip, decoded, detected, drawn and encoded with VideoWriter (mp4v)

Arms: the per-image loop and det_bs 1, 8 and 32, end to end (images or frames per second, host clock around the whole run, which
ends after the last write).  For each det_bs, a separate instrumented pass times every device stage of a batch with CUDA events
(mean ms per batch) and the host pass of a batch (cv2 labels plus encode, mean ms).  Prints one JSON line (GPU name and power
limit read in the same run) and writes it to --out.

    python tools/bench_detect.py [--images 256] [--frames 64] [--out profiles/h100_bench_detect.json]

With --jpeg_gpu it runs the image arms only, at det_bs 8 and 32, both with cv2.imwrite and with detect --jpeg_gpu (images/s end to
end), and splits the host pass of a batch into the cv2 labels and the encode: cv2.imencode of each drawn image, or the JpegWriter's
packing and queueing (mean ms per batch).  Its default --out is profiles/h100_bench_detect_jpeg.json.

With --decode_gpu it runs the image arms only, at det_bs 8 and 32 with 2 loader workers (detect's default): cv2.imread in the
workers against detect --decode_gpu, each with cv2.imwrite and with --jpeg_gpu (images/s end to end), and what one worker does per
image to read it (cv2.imread, or np.fromfile plus yb_jpeg_header; median ms on one thread).  Its default --out is
profiles/h100_bench_detect_decode.json.
"""
import argparse
import glob
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
from detect_loop import per_frame_detect, per_image_detect  # noqa: E402
from oracle import forward_torch as ft  # noqa: E402
from yolact_minimal_b200 import detect as yd  # noqa: E402
from yolact_minimal_b200.config import make_config  # noqa: E402
from yolact_minimal_b200.modules.yolact import Yolact  # noqa: E402
from yolact_minimal_b200.utils import output_utils as ou  # noqa: E402
from yolact_minimal_b200.utils.augmentations import val_aug_batch  # noqa: E402
from yolact_minimal_b200.utils.coco import DetectImages, detect_collate  # noqa: E402

SIZES = ((480, 640), (640, 480), (427, 640))
STAGES = ('h2d', 'val_aug', 'forward', 'detect', 'visible', 'masks', 'overlay', 'd2h')
BATCHES = (1, 8, 32)


def scene(k, h, w, rng):
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([128 + 100 * np.sin(xx / (7 + k % 5) + c) * np.cos(yy / (11 + c)) for c in range(3)], -1)
    return np.clip(base + rng.normal(0, 20, size=(h, w, 3)), 0, 255).astype(np.uint8)


def stage_times(net, cfg, packed_batches):
    """Mean device ms per batch of each stage, and mean host ms of the cv2 pass, over the given batches (after one warm-up)."""
    import cv2
    dev = next(net.parameters()).device
    host = yd._HostBuffers()
    acc, host_ms = {s: 0.0 for s in STAGES}, 0.0
    for i, packed in enumerate(packed_batches):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(STAGES) + 1)]
        ev[0].record()
        src = packed.buffer.to(dev, non_blocking=True)
        ev[1].record()
        with torch.no_grad():
            images = val_aug_batch(src, packed.items, cfg.img_size, dev)
            ev[2].record()
            class_p, box_p, coef_p, proto_p = net(images)
        ev[3].record()
        det = ou.detect_batched(class_p, box_p, coef_p, net.anchors, cfg)
        ev[4].record()
        det = dict(det, count=ou.visible_count(det, cfg.visual_thre))
        ev[5].record()
        boxes_px, masks = ou.after_nms_batched(det, proto_p, packed.sizes)
        ev[6].record()
        frames = ou.blend_masks_batched(src, packed.items, det, masks, cfg.num_classes)
        ev[7].record()
        res = {k: host.take(k, v) for k, v in dict(count=det['count'], cls=det['cls'], score=det['score'], boxes=boxes_px,
                                                    frames=frames).items()}
        ev[8].record()
        p = yd._Pending(packed=packed, src=src, det=det, masks=masks, res=res, done=ev[8])
        t0 = time.perf_counter()
        yd.finish(p, cfg, lambda name, img: cv2.imencode('.jpg', img))
        if i == 0:
            continue
        host_ms += (time.perf_counter() - t0) * 1e3
        for k, s in enumerate(STAGES):
            acc[s] += ev[k].elapsed_time(ev[k + 1])
    n = len(packed_batches) - 1
    return {s: round(v / n, 4) for s, v in acc.items()}, round(host_ms / n, 3)


def host_split(net, cfg, batches):
    """Mean ms per batch of the host pass: cv2 labels (finish with the device already done), then the encode of the drawn
    images: cv2.imencode each, or JpegWriter.put_host + flush (packing into page-locked memory and queueing the encode)."""
    import cv2
    hosts = (yd._HostBuffers(), yd._HostBuffers())
    labels, cv2_enc, gpu_enc = [], [], []
    writer = yd.JpegWriter()
    for i, packed in enumerate(batches):
        p = yd.enqueue(net, cfg, packed, hosts[i % 2])
        torch.cuda.synchronize()
        drawn = []
        t0 = time.perf_counter()
        yd.finish(p, cfg, lambda name, img: drawn.append((name, img.copy())))
        labels.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        for _, img in drawn:
            cv2.imencode('.jpg', img)
        cv2_enc.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for name, img in drawn:
            writer.put_host(f'results/images/{name}', img)
        writer.flush()
        gpu_enc.append(time.perf_counter() - t0)
    writer.close()
    ms = lambda v: round(1e3 * float(np.mean(v[1:])), 3)
    return {'labels_ms': ms(labels), 'cv2_encode_ms': ms(cv2_enc), 'jpeg_gpu_queue_ms': ms(gpu_enc)}


def jpeg_arm(args, net, cfg, rng):
    import cv2
    result = {'gpu': torch.cuda.get_device_name(0), 'power_limit_w': power_limit(), 'model': 'res101_coco 550 fp16, synthetic weights',
              'visual_thre': 0.3, 'images': args.images}
    with tempfile.TemporaryDirectory() as tmp:
        folder = os.path.join(tmp, 'images')
        os.makedirs(folder)
        for k in range(args.images):
            cv2.imwrite(os.path.join(folder, f'{k:04d}.jpg'), scene(k, *SIZES[k % len(SIZES)], rng))
        os.chdir(tmp)
        os.makedirs('results/images')
        cfg.image = folder
        for jpeg_gpu in (False, True):                                             # warm-up
            cfg.jpeg_gpu = jpeg_gpu
            yd.detect_images(net, cfg, 32)
        e2e = {}
        for bs in (8, 32):
            for jpeg_gpu in (False, True):
                cfg.jpeg_gpu = jpeg_gpu
                t0 = time.perf_counter()
                yd.detect_images(net, cfg, bs)
                e2e[f'det_bs{bs}' + ('_jpeg_gpu' if jpeg_gpu else '')] = round(args.images / (time.perf_counter() - t0), 2)
        cfg.jpeg_gpu = False
        result['images_per_s'] = e2e
        ds = DetectImages(cfg)
        split = {}
        for bs in (8, 32):
            batches = [detect_collate([ds[i] for i in range(j, min(j + bs, len(ds)))]).pin_memory()
                       for j in range(0, min(len(ds), 9 * bs), bs)]
            split[f'det_bs{bs}'] = host_split(net, cfg, batches)
        result['host_pass_ms_per_batch'] = split
        os.chdir(ROOT)
    return result


def decode_arm(args, net, cfg, rng):
    import cv2
    from bench_val import read_ms
    result = {'gpu': torch.cuda.get_device_name(0), 'power_limit_w': power_limit(), 'model': 'res101_coco 550 fp16, synthetic weights',
              'visual_thre': 0.3, 'images': args.images, 'workers': 2, 'files': 'cv2.imwrite defaults (q95, 4:2:0)'}
    with tempfile.TemporaryDirectory() as tmp:
        folder = os.path.join(tmp, 'images')
        os.makedirs(folder)
        for k in range(args.images):
            cv2.imwrite(os.path.join(folder, f'{k:04d}.jpg'), scene(k, *SIZES[k % len(SIZES)], rng))
        result['worker_read_ms_per_image'] = read_ms(sorted(glob.glob(os.path.join(folder, '*.jpg')))[:64])
        os.chdir(tmp)
        os.makedirs('results/images')
        cfg.image = folder
        for decode_gpu in (False, True):                                           # warm-up
            cfg.decode_gpu = decode_gpu
            yd.detect_images(net, cfg, 32)
        e2e = {}
        for bs in (8, 32):
            for jpeg_gpu in (False, True):
                for decode_gpu in (False, True):
                    cfg.jpeg_gpu, cfg.decode_gpu = jpeg_gpu, decode_gpu
                    t0 = time.perf_counter()
                    yd.detect_images(net, cfg, bs)
                    key = f'det_bs{bs}' + ('_jpeg_gpu' if jpeg_gpu else '') + ('_decode_gpu' if decode_gpu else '')
                    e2e[key] = round(args.images / (time.perf_counter() - t0), 2)
        cfg.jpeg_gpu = cfg.decode_gpu = False
        result['images_per_s'] = e2e
        os.chdir(ROOT)
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=256)
    ap.add_argument('--frames', type=int, default=64)
    ap.add_argument('--jpeg_gpu', action='store_true')
    ap.add_argument('--decode_gpu', action='store_true')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if args.out is None:
        args.out = os.path.join(ROOT, 'profiles', 'h100_bench_detect_decode.json' if args.decode_gpu else
                                'h100_bench_detect_jpeg.json' if args.jpeg_gpu else 'h100_bench_detect.json')
    import cv2
    dev = torch.device('cuda')
    cfg = make_config('res101_coco', 550, mode='detect', visual_thre=0.3)
    cfg.precision, cfg.max_batch = 'fp16', max(BATCHES)
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict('res101', seed=0), strict=True)
    net = net.to(dev).eval()
    rng = np.random.RandomState(5)
    if args.decode_gpu or args.jpeg_gpu:
        result = decode_arm(args, net, cfg, rng) if args.decode_gpu else jpeg_arm(args, net, cfg, rng)
        line = json.dumps(result)
        print(line)
        with open(args.out, 'w') as f:
            f.write(line + '\n')
        return
    result = {'gpu': torch.cuda.get_device_name(0), 'power_limit_w': power_limit(), 'model': 'res101_coco 550 fp16, synthetic weights',
              'visual_thre': 0.3, 'images': args.images, 'frames': args.frames}
    with tempfile.TemporaryDirectory() as tmp:
        folder = os.path.join(tmp, 'images')
        os.makedirs(folder)
        for k in range(args.images):
            cv2.imwrite(os.path.join(folder, f'{k:04d}.jpg'), scene(k, *SIZES[k % len(SIZES)], rng))
        video = os.path.join(tmp, 'clip.avi')
        vw = cv2.VideoWriter(video, cv2.VideoWriter_fourcc(*'MJPG'), 30, (1920, 1080))
        for k in range(args.frames):
            vw.write(scene(k % 5, 1080, 1920, rng))
        vw.release()
        os.chdir(tmp)
        os.makedirs('results/images'), os.makedirs('results/videos')
        cfg.image, cfg.video = folder, video
        paths = sorted(glob.glob(folder + '/*.jpg'))
        per_image_detect(net, cfg, paths[:8])                                    # warm-up
        yd.detect_images(net, cfg, max(BATCHES))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        per_image_detect(net, cfg, paths)
        torch.cuda.synchronize()
        e2e = {'per_image': round(args.images / (time.perf_counter() - t0), 2)}
        for bs in BATCHES:
            t0 = time.perf_counter()
            yd.detect_images(net, cfg, bs)
            e2e[f'det_bs{bs}'] = round(args.images / (time.perf_counter() - t0), 2)
        result['images_per_s'] = e2e
        ds = DetectImages(cfg)
        stages = {}
        for bs in BATCHES:
            batches = [detect_collate([ds[i] for i in range(j, min(j + bs, len(ds)))]).pin_memory()
                       for j in range(0, min(len(ds), 9 * bs), bs)]
            st, host_ms = stage_times(net, cfg, batches)
            stages[f'det_bs{bs}'] = {'device_ms_per_batch': st, 'device_ms_total': round(sum(st.values()), 3),
                                     'host_labels_encode_ms_per_batch': host_ms}
        result['stages'] = stages
        vfps = {}
        t0 = time.perf_counter()
        per_frame_detect(net, cfg, video, cv2.VideoWriter('results/videos/ref.mp4', cv2.VideoWriter_fourcc(*'mp4v'), 30, (1920, 1080)))
        vfps['per_frame'] = round(args.frames / (time.perf_counter() - t0), 2)
        for bs in BATCHES:
            t0 = time.perf_counter()
            yd.detect_video(net, cfg, bs)
            vfps[f'det_bs{bs}'] = round(args.frames / (time.perf_counter() - t0), 2)
        result['video_1080x1920_frames_per_s'] = vfps
        os.chdir(ROOT)
    line = json.dumps(result)
    print(line)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
        f.write(line + '\n')


if __name__ == '__main__':
    main()
