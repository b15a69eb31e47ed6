#!/usr/bin/env python
"""Time draw_img's device overlay (csrc/draw.cu) against the host path detect.py took before it.

Inputs: synthetic 'stress' head outputs (oracle/synth.py) at 544x544 through the package's nms and after_nms, keeping the top 20
or 100 detections, at 480x640 and 1080x1920.  after_nms runs with no_crop: the synthetic boxes are small, and the uncropped masks
cover large, overlapping areas -- the heavier case for the packed-bit path, which skips all-zero words.
  kernel     k_draw_masks per mask format (float32 / uint8 / bits), CUDA events over many launches of yb_draw_masks; algorithmic
             bytes = masks + image read + image written, and their rate as a share of the H100 SXM data sheet's 3.35 TB/s
  draw_img   per frame on a host clock around a synchronised call, image H2D and D2H and the cv2 label pass included, for float32
             masks (what after_nms returns by default) and packed bits
  host       the path detect.py took before: the float32 masks and the detections .cpu() plus oracle/draw_np.draw (numpy overlay
             + the same cv2 label pass), same frames, same run; its image must equal draw_img's
Prints one JSON line (GPU name and power limit read in the same run).

    python tools/bench_draw.py [--frames 20] [--host-frames 3] [--out FILE]
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

from oracle import draw_np as dn, postprocess_np as pp, synth  # noqa: E402
from yolact_minimal_b200 import _lib  # noqa: E402
from yolact_minimal_b200.config import COLORS, make_config  # noqa: E402
from yolact_minimal_b200.utils.output_utils import after_nms, draw_img, nms  # noqa: E402

HBM_TB_S = 3.35
WORKLOADS = ((480, 640, 20), (480, 640, 100), (1080, 1920, 20), (1080, 1920, 100))


def power_limit():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def detections(dev, S=544, seed=3):
    cfg = make_config('res101_coco', S)
    anchors = torch.from_numpy(pp.make_anchors(S)).to(dev)
    cls, box, coef = synth.head_outputs(seed, anchors.shape[0])
    proto = synth.proto(seed, (S + 3) // 4)
    t = lambda a: torch.from_numpy(a).to(dev)
    out = nms(t(cls), t(box), t(coef), t(proto), anchors, cfg)
    assert out[0] is not None and out[0].shape[0] == 100
    cfg.no_crop = True
    return out, cfg


def kernel_ms(img, ids32, masks, fmt, pal, nc, reps):
    L = _lib.lib()
    h, w = img.shape[:2]
    out = torch.empty_like(img)
    s = torch.cuda.current_stream().cuda_stream
    call = lambda: L.yb_draw_masks(img.data_ptr(), h, w, masks.data_ptr(), fmt, ids32.shape[0], ids32.data_ptr(), pal.data_ptr(), nc,
                                   out.data_ptr(), s)
    for _ in range(5):
        _lib.check(call())
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=20)
    ap.add_argument('--host-frames', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_draw needs a CUDA device')
    dev = torch.device('cuda:0')
    (ids_all, scores_all, box_all, coef_all, proto), cfg = detections(dev)
    pal = torch.from_numpy(COLORS.reshape(-1).copy()).to(dev)
    nc = cfg.num_classes - 1
    rows = []
    for h, w, n in WORKLOADS:
        args = (ids_all[:n], scores_all[:n], box_all[:n], coef_all[:n], proto, h, w, cfg)
        dets = {k: after_nms(*args, mask_dtype=dt) for k, dt in (('f32', torch.float32), ('u8', torch.uint8), ('bits', 'bits'))}
        img = np.random.default_rng(h + n).integers(0, 256, (h, w, 3), dtype=np.uint8)
        img_d = torch.from_numpy(img).to(dev)
        ids32 = dets['f32'][0].to(torch.int32)
        row = {'h': h, 'w': w, 'detections': n, 'mask_coverage': round(float(dets['u8'][3].float().mean()), 4),
               'max_overlap': int(dets['u8'][3].sum(0, dtype=torch.int32).max()), 'kernel': {}}
        for fmt_name, code in (('f32', 1), ('u8', 0), ('bits', 2)):
            m = dets[fmt_name][3]
            ms = kernel_ms(img_d, ids32, m, code, pal, nc, reps=100 if h > 500 else 400)
            nbytes = m.numel() * m.element_size() + 2 * img.nbytes
            row['kernel'][fmt_name] = {'ms': round(ms, 5), 'bytes': nbytes, 'tb_s': round(nbytes / ms / 1e9, 3),
                                       'share_of_3.35_tb_s': round(nbytes / ms / 1e9 / HBM_TB_S, 4)}
        row['draw_img_ms'] = {}
        for fmt_name in ('f32', 'bits'):
            i, s, b, m = dets[fmt_name]
            for _ in range(3):
                draw_img(i, s, b, m, img, cfg)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.frames):
                got = draw_img(i, s, b, m, img, cfg)
            torch.cuda.synchronize()
            row['draw_img_ms'][fmt_name] = round((time.perf_counter() - t0) * 1e3 / a.frames, 3)
        i, s, b, m = dets['f32']
        want = None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.host_frames):
            want, _ = dn.draw(i.cpu().numpy(), s.cpu().numpy(), b.cpu().numpy(), m.cpu().numpy(), img, cfg, COLORS)
        row['host_path_ms'] = round((time.perf_counter() - t0) * 1e3 / a.host_frames, 3)
        row['draw_img_f32_equals_host_path'] = bool(np.array_equal(draw_img(i, s, b, m, img, cfg), want))
        row['host_over_draw_img_f32'] = round(row['host_path_ms'] / row['draw_img_ms']['f32'], 2)
        rows.append(row)
        del dets, img_d
        torch.cuda.empty_cache()
    res = {'workload': 'draw_img_synthetic_stress_no_crop', 'gpu': torch.cuda.get_device_name(0), 'power_limit_w': power_limit(),
           'hbm_data_sheet_tb_s': HBM_TB_S, 'frames': a.frames, 'host_frames': a.host_frames, 'rows': rows}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
