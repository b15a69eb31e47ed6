#!/usr/bin/env python
"""Time batched COCO-style evaluation (yolact_minimal_b200.eval's per-batch body) against the reference's per-image loop.

Workload: res101_coco 550, fp16, synthetic weights (oracle.forward_torch.synth_state_dict), B = 64, --images synthetic images of
COCO sizes (480x640, 640x480, 427x640, 640x427) with gts built from a first detection pass (shifted boxes of some detections
plus an unrelated box).  The batches are packed (PackedValBatch) and pinned before timing, so the numbers cover the GPU side and
not JPEG decoding.  Arms:
  batched    per batch: val_aug_batch, net(images), detect_batched, after_nms_batched, MapEvaluator.add; CUDA-event time per stage
  per_image  tests/val_loop.py: val_aug, net(img[None]), nms, after_nms with float masks, prep_metrics per image
Both arms end in calc_map; their (box_row, mask_row) must be identical.  Prints one JSON line (GPU name and power limit read in
the same run) and writes it to --out.

    python tools/bench_val.py [--images 1024] [--batch 64] [--out profiles/h100_bench_val.json]

With --decode_gpu it instead times evaluate(net, cfg) end to end on the same images written as JPEG files (cv2.imwrite: q95,
4:2:0) with a stub COCO of their gts, 4 loader workers as evaluate's default: once with cv2.imread in the workers and once with
--decode_gpu (the workers read the files' bytes, each batch is decoded on the device).  Images/s by the host clock around the
whole call, after a warm-up call of each; the rows of both must be identical.  It also times what one worker does per image to
read it (cv2.imread, or np.fromfile plus yb_jpeg_header).  Its default --out is profiles/h100_bench_val_decode.json.
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
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from oracle import forward_torch as ft  # noqa: E402
from val_loop import per_image_evaluate  # noqa: E402
from yolact_minimal_b200.config import make_config  # noqa: E402
from yolact_minimal_b200.eval import iou_thres  # noqa: E402
from yolact_minimal_b200.modules.yolact import Yolact  # noqa: E402
from yolact_minimal_b200.utils.augmentations import PackedValBatch, val_aug_batch  # noqa: E402
from yolact_minimal_b200.utils.common_utils import APDataObject, _bind, calc_map  # noqa: E402
from yolact_minimal_b200.utils.mask_utils import pack_masks_host  # noqa: E402
from yolact_minimal_b200.utils.output_utils import after_nms_batched, detect_batched  # noqa: E402

SIZES = ((480, 640), (640, 480), (427, 640), (640, 427))
STAGES = ('preprocess', 'forward', 'detect', 'masks', 'match')


def power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def images(n, seed=5):
    """Smooth-plus-noise BGR images of COCO sizes: enough structure for the synthetic net to detect things."""
    rng = np.random.RandomState(seed)
    out = []
    for k in range(n):
        h, w = SIZES[k % len(SIZES)]
        yy, xx = np.mgrid[0:h, 0:w]
        img = np.stack([128 + 100 * np.sin(xx / (7 + k % 5) + c) * np.cos(yy / (11 + c)) for c in range(3)], -1)
        out.append(np.clip(img + rng.normal(0, 20, size=(h, w, 3)), 0, 255).astype(np.uint8))
    return out


def samples(net, cfg, imgs, batch, dev):
    """COCOValDetection-style items whose gts come from a first detection pass, as in tests/test_eval_gpu.py: the class and the
    shifted box of every third detection, plus one unrelated box, with rectangular masks."""
    from yolact_minimal_b200.utils.augmentations import pack_images
    out = []
    for i in range(0, len(imgs), batch):
        chunk = imgs[i:i + batch]
        buf, items = pack_images(chunk)
        with torch.no_grad():
            cls, box, coef, _ = net(val_aug_batch(buf, items, cfg.img_size, dev))
        det = detect_batched(cls, box, coef, net.anchors, cfg)
        count, ids, boxes = det['count'].cpu().numpy(), det['cls'].cpu().numpy(), det['box'].cpu().numpy().astype(np.float64)
        for b, img in enumerate(chunk):
            h, w = img.shape[:2]
            sel = list(range(0, int(count[b]), 3))
            px = np.trunc(boxes[b, sel] * max(h, w))
            px = np.concatenate([np.clip(px + np.array([2, -1, 3, 1]), 0, [w, h, w, h]), [[5, 5, 40, 30]]])
            labels = np.array([ids[b, j] for j in sel] + [(7 * (i + b)) % 80], np.float64)
            rects = np.floor(px).astype(np.int64)
            masks = np.zeros((len(rects), h, w), np.uint8)
            for g, (x1, y1, x2, y2) in enumerate(rects):
                masks[g, y1:y2, x1:x2] = 1
            gt = np.hstack((px / np.array([w, h, w, h]), labels[:, None])).astype(np.float32)
            out.append((img, gt, pack_masks_host(masks), (h, w), i + b))
    return out


def new_ap_data(cfg, dev):
    ap_data = {'box': [[APDataObject() for _ in cfg.class_names] for _ in iou_thres],
               'mask': [[APDataObject() for _ in cfg.class_names] for _ in iou_thres]}
    return ap_data, _bind(ap_data, iou_thres, dev)


def batched(net, cfg, batches, dev, events=None):
    ap_data, ev = new_ap_data(cfg, dev)
    rec = (lambda i: events[i].record()) if events is not None else (lambda i: None)
    for packed in batches:
        rec(0)
        with torch.no_grad():
            x = val_aug_batch(packed.buffer, packed.items, cfg.img_size, dev)
            rec(1)
            class_p, box_p, coef_p, proto_p = net(x)
        rec(2)
        det = detect_batched(class_p, box_p, coef_p, net.anchors, cfg)
        rec(3)
        boxes_px, masks = after_nms_batched(det, proto_p, packed.sizes)
        rec(4)
        gt, gt_masks = packed.gt_to(dev)
        ev.add(det, boxes_px, masks, gt, packed.gt_offset, gt_masks, packed.sizes)
        rec(5)
        if events is not None:
            events = events[6:]
    return ap_data


def read_ms(paths):
    """Median ms per image, on one thread, of what a worker does to read an image: cv2.imread, or the bytes and the header."""
    import cv2
    from yolact_minimal_b200.utils.augmentations import read_image
    cv2.setNumThreads(1)
    out = {}
    for key, fn in (('cv2_imread', cv2.imread), ('decode_gpu_read', lambda p: read_image(p, decode_gpu=True))):
        ts = []
        for p in paths:
            t0 = time.perf_counter()
            fn(p)
            ts.append(time.perf_counter() - t0)
        out[key] = round(1e3 * float(np.median(ts)), 3)
    return out


def decode_arm(a, net, cfg, dev):
    import tempfile
    import cv2
    from test_val_batch_gpu import _StubCOCO
    from yolact_minimal_b200.config import COCO_LABEL_MAP
    from yolact_minimal_b200.eval import evaluate
    from yolact_minimal_b200.utils.coco import COCOValDetection
    coco_id = {label - 1: cid for cid, label in COCO_LABEL_MAP.items()}
    items = samples(net, cfg, images(a.images), a.batch, dev)
    res = dict(bench='bench_val --decode_gpu', gpu=torch.cuda.get_device_name(0), power_limit_w=power_limit(), arch='res101_coco',
               img_size=550, precision='fp16', val_bs=a.batch, images=a.images, sizes=[list(s) for s in SIZES], workers=4,
               files='cv2.imwrite defaults (q95, 4:2:0)')
    with tempfile.TemporaryDirectory() as tmp:
        meta, nbytes = {}, 0
        for k, (img, gt, _, (h, w), _) in enumerate(items):
            name = f'{k:05d}.jpg'
            cv2.imwrite(os.path.join(tmp, name), img)
            nbytes += os.path.getsize(os.path.join(tmp, name))
            anns = []
            for row in gt.astype(np.float64):
                x1, y1, x2, y2 = row[:4] * [w, h, w, h]
                anns.append(dict(bbox=[x1, y1, x2 - x1, y2 - y1], category_id=coco_id[int(row[4])], iscrowd=0, _hw=(h, w)))
            meta[k] = (name, h, w, anns)
        res['file_mb'] = round(nbytes / 1e6, 2)
        res['pixel_mb'] = round(sum(it[0].nbytes for it in items) / 1e6, 2)
        res['worker_read_ms_per_image'] = read_ms([os.path.join(tmp, meta[k][0]) for k in range(min(64, len(meta)))])
        coco = _StubCOCO(meta)
        cfg.val_imgs, cfg.val_bs, cfg.val_num = tmp, a.batch, -1
        rows, ips = {}, {}
        for decode_gpu in (False, True):
            cfg.decode_gpu = decode_gpu
            ds = COCOValDetection(cfg, coco=coco, decode_gpu=decode_gpu)
            evaluate(net, cfg, dataset=ds)                                 # warm-up: workers, engine, workspaces
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rows[decode_gpu] = evaluate(net, cfg, dataset=ds)
            torch.cuda.synchronize()
            ips['decode_gpu' if decode_gpu else 'cv2_imread'] = round(a.images / (time.perf_counter() - t0), 1)
        cfg.decode_gpu = False
    assert rows[True] == rows[False], (rows[True][1:], rows[False][1:])
    assert rows[False][1][1] > 0, 'the workload has no matches: the row comparison would be vacuous'
    res.update(images_per_s_end_to_end=ips, rows_equal=True, box_row=rows[False][1], mask_row=rows[False][2],
               batched_gpu_images_per_s='profiles/h100_bench_val.json')
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=1024)
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--decode_gpu', action='store_true')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if a.out is None:
        a.out = os.path.join(ROOT, 'profiles', 'h100_bench_val_decode.json' if a.decode_gpu else 'h100_bench_val.json')
    dev = torch.device('cuda:0')
    cfg = make_config('res101_coco', 550, mode='val')
    cfg.precision, cfg.max_batch = 'fp16', a.batch
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict('res101', seed=0), strict=True)
    net = net.to(dev).eval()
    if a.decode_gpu:
        line = json.dumps(decode_arm(a, net, cfg, dev))
        print(line)
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')
        return
    items = samples(net, cfg, images(a.images), a.batch, dev)
    batches = [PackedValBatch(items[i:i + a.batch]).pin_memory() for i in range(0, len(items), a.batch)]

    batched(net, cfg, batches[:1], dev)                                     # warm-up: engine finalize, workspaces, anchors
    torch.cuda.synchronize()
    events = [torch.cuda.Event(enable_timing=True) for _ in range(6 * len(batches))]
    t0 = time.perf_counter()
    ap_data = batched(net, cfg, batches, dev, events)
    torch.cuda.synchronize()
    host_s = time.perf_counter() - t0
    stage_ms = {s: 0.0 for s in STAGES}
    for b in range(len(batches)):
        e = events[6 * b:6 * b + 6]
        for i, s in enumerate(STAGES):
            stage_ms[s] += e[i].elapsed_time(e[i + 1])
    gpu_ms = events[0].elapsed_time(events[-1])
    _, box_b, mask_b = calc_map(ap_data, iou_thres, len(cfg.class_names), step=None)

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    _, box_p, mask_p = per_image_evaluate(net, cfg, items)
    per_image_s = time.perf_counter() - t0
    assert (box_b, mask_b) == (box_p, mask_p), (box_b, mask_b, box_p, mask_p)
    assert box_b[1] > 0 and mask_b[1] > 0, 'the workload has no matches: the row comparison would be vacuous'

    res = dict(bench='bench_val', gpu=torch.cuda.get_device_name(0), power_limit_w=power_limit(), arch='res101_coco', img_size=550,
               precision='fp16', batch=a.batch, images=a.images, sizes=[list(s) for s in SIZES],
               batched=dict(gpu_ms=round(gpu_ms, 3), host_s=round(host_s, 4), images_per_s=round(a.images / (gpu_ms / 1e3), 1),
                            stage_ms={k: round(v, 3) for k, v in stage_ms.items()},
                            stage_ms_per_batch={k: round(v / len(batches), 3) for k, v in stage_ms.items()}),
               per_image=dict(s=round(per_image_s, 3), images_per_s=round(a.images / per_image_s, 1)),
               speedup=round(per_image_s / (gpu_ms / 1e3), 2), box_row=box_b, mask_row=mask_b, rows_equal=True,
               end_to_end_with_coco_loader='not measured')
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
