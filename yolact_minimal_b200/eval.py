"""COCO evaluation in batches on the GPU: the reference's eval.py `evaluate(net, cfg, step=None)` with the same signature, return
value `(table, box_row, mask_row)` and progress line, fed `cfg.val_bs` images at a time:

    val_aug_batch -> net(images) -> detect_batched -> after_nms_batched -> MapEvaluator.add        (per batch, no host sync)
    calc_map(ap_data, ...)                                                                          (once, through ap_data)

The rows equal the reference's per-image loop (eval.py:42-69,106 with val_aug, nms, after_nms, prep_metrics) bit for bit: the
forward is batch-invariant, detect_batched treats images independently, after_nms_batched equals after_nms per image and
MapEvaluator appends the images in order (DESIGN.md, batched evaluation).  With cfg.coco_api the detections go to MakeJson and
pycocotools' COCOeval instead, as in the reference.  With cfg.coco_gpu (--coco_gpu) they go to utils.cocoeval.CocoEvaluator, which
computes COCOeval's bbox and segm results on the GPU from the same detections, with no JSON and no COCOeval; evaluate() then
prints COCOeval's two summaries and returns their stats (box_stats, mask_stats), float64 [12] each.  With cfg.decode_gpu
(--decode_gpu) the workers read the JPEG files' bytes and each batch is decoded on the device (yb_jpeg_decode_batch, the pixels
cv2.imread returns); the decode statuses are read once at the end, and a file with corrupt entropy-coded data raises.

    python -m yolact_minimal_b200.eval --weight weights/best_30.5_res101_coco_392000.pth --val_bs 64
"""
import argparse
import re
import time

import numpy as np
import torch
from torch.utils.data import DataLoader

from .utils import mask_utils
from .utils.augmentations import val_aug_batch
from .utils.coco import COCOValDetection, val_collate
from .utils.cocoeval import CocoEvaluator
from .utils.common_utils import APDataObject, MakeJson, ProgressBar, _bind, calc_map
from .utils.output_utils import after_nms_batched, detect_batched

iou_thres = [x / 100 for x in range(50, 100, 5)]


def _add_json(make_json, packed, det, boxes_px, masks):
    """eval.py:60-67 for a batch: boxes and RLE masks of the detections with a positive box area."""
    count = det['count'].cpu().numpy()
    cls, score, boxes = det['cls'].cpu().numpy(), det['score'].cpu().numpy(), boxes_px.cpu().numpy()
    for b, n in enumerate(count):
        keep = [j for j in range(int(n)) if (boxes[b, j, 3] - boxes[b, j, 1]) * (boxes[b, j, 2] - boxes[b, j, 0]) > 0]
        if not keep:
            continue
        h, w = packed.sizes[b]
        rles = mask_utils.encode_rle(masks[b][keep].contiguous(), h, w)
        for j, rle in zip(keep, rles):
            make_json.add_bbox(packed.ids[b], cls[b, j], boxes[b, j, :], float(score[b, j]))
            make_json.add_mask_rle(packed.ids[b], cls[b, j], rle, float(score[b, j]))


def evaluate(net, cfg, step=None, *, dataset=None, num_workers=4):
    """Box and mask mAP of `net` on COCO val (cfg.val_imgs / cfg.val_ann, cfg.val_num images), cfg.val_bs images per batch.
    `dataset` replaces COCOValDetection(cfg) (any object with its item format; with cfg.coco_gpu, COCOValDetection's
    coco_eval=True format and a `coco` attribute), `num_workers` the loader's workers."""
    coco_gpu = bool(getattr(cfg, 'coco_gpu', False))
    if coco_gpu and cfg.coco_api:
        raise ValueError('evaluate: coco_api and coco_gpu are alternatives; set one')
    decode_gpu = bool(getattr(cfg, 'decode_gpu', False))
    dataset = COCOValDetection(cfg, coco_eval=coco_gpu, decode_gpu=decode_gpu) if dataset is None else dataset
    data_loader = DataLoader(dataset, int(cfg.val_bs), num_workers=num_workers, shuffle=False, pin_memory=True,
                             collate_fn=val_collate)
    ds = len(data_loader)
    progress_bar = ProgressBar(40, max(ds, 1))
    dev = next(net.parameters()).device
    ap_data = {'box': [[APDataObject() for _ in cfg.class_names] for _ in iou_thres],
               'mask': [[APDataObject() for _ in cfg.class_names] for _ in iou_thres]}
    evaluator = None if cfg.coco_api or coco_gpu else _bind(ap_data, iou_thres, dev)
    coco_ev = CocoEvaluator(dataset.coco, cfg.continuous_id, dev) if coco_gpu else None
    make_json = MakeJson() if cfg.coco_api else None
    start, seen = None, 0
    statuses = []                                 # (device status, image ids of its entries) of the batches decoded on the device
    for i, packed in enumerate(data_loader):
        if i == 1:
            start, seen = time.perf_counter(), 0
        with torch.no_grad():
            if packed.mixed is not None:
                buffer, status = packed.to_device(dev)
                if status is not None:
                    statuses.append((status, [packed.ids[int(k)] for k in packed.mixed.encoded]))
            else:
                buffer = packed.buffer
            images = val_aug_batch(buffer, packed.items, cfg.img_size, dev)
            class_p, box_p, coef_p, proto_p = net(images)
        det = detect_batched(class_p, box_p, coef_p, net.anchors, cfg)
        boxes_px, masks = after_nms_batched(det, proto_p, packed.sizes)
        if cfg.coco_api:
            _add_json(make_json, packed, det, boxes_px, masks)
        elif coco_gpu:
            coco_ev.add(det, boxes_px, masks, packed)
        else:
            gt, gt_masks = packed.gt_to(dev)
            evaluator.add(det, boxes_px, masks, gt, packed.gt_offset, gt_masks, packed.sizes)
        seen += len(packed)
        if i > 0:
            # host time of the batches after the first: the device runs behind the host by at most the queue depth
            fps = seen / (time.perf_counter() - start)
            print(f'\rTesting: {progress_bar.get_bar(i + 1)} {i + 1}/{ds}, total fps: {fps:.2f}', end='')

    if statuses:
        codes = torch.cat([s for s, _ in statuses]).cpu().numpy()
        ids = [i for _, b in statuses for i in b]
        bad = [ids[k] for k in np.flatnonzero(codes)]
        if bad:
            raise RuntimeError(f'corrupt JPEG data in the images with ids {bad}')
    if coco_gpu:
        print()
        box_stats, mask_stats = coco_ev.summarize()
        return box_stats, mask_stats
    if cfg.coco_api:
        from pycocotools.coco import COCO
        from pycocotools.cocoeval import COCOeval
        make_json.dump()
        print(f'\nJson files dumped, saved in: \'results/\', start evaluating.')

        gt_annotations = COCO(cfg.val_ann)
        bbox_dets = gt_annotations.loadRes(f'results/bbox_detections.json')
        mask_dets = gt_annotations.loadRes(f'results/mask_detections.json')

        print('\nEvaluating BBoxes:')
        bbox_eval = COCOeval(gt_annotations, bbox_dets, 'bbox')
        bbox_eval.evaluate()
        bbox_eval.accumulate()
        bbox_eval.summarize()

        print('\nEvaluating Masks:')
        bbox_eval = COCOeval(gt_annotations, mask_dets, 'segm')
        bbox_eval.evaluate()
        bbox_eval.accumulate()
        bbox_eval.summarize()
    else:
        table, box_row, mask_row = calc_map(ap_data, iou_thres, len(cfg.class_names), step=step)
        print(table)
        return table, box_row, mask_row


def main(argv=None):
    from .config import get_config, make_output_dirs
    from .modules.yolact import Yolact
    parser = argparse.ArgumentParser(description='YOLACT COCO Evaluation')
    parser.add_argument('--img_size', type=int, default=544, help='The image size for validation.')
    parser.add_argument('--weight', type=str, default='weights/best_30.5_res101_coco_392000.pth')
    parser.add_argument('--traditional_nms', default=False, action='store_true', help='Whether to use traditional nms.')
    parser.add_argument('--val_num', default=-1, type=int, help='The number of images for test, set to -1 for all.')
    parser.add_argument('--coco_api', action='store_true', help='Whether to use cocoapi to evaluate results.')
    parser.add_argument('--coco_gpu', action='store_true', help='Compute COCOeval\'s box and mask mAP on the GPU (no JSON, '
                        'no pycocotools for the metric).')
    parser.add_argument('--val_bs', default=1, type=int, help='Images per batch on the GPU.')
    parser.add_argument('--decode_gpu', action='store_true', help='Decode the JPEG files on the GPU (the same pixels cv2.imread '
                        'returns).')
    args = parser.parse_args(argv)
    if args.coco_api and args.coco_gpu:
        parser.error('--coco_api and --coco_gpu are alternatives')
    prefix = re.findall(r'best_\d+\.\d+_', args.weight)[0]
    suffix = re.findall(r'_\d+\.pth', args.weight)[0]
    args.cfg = args.weight.split(prefix)[-1].split(suffix)[0]
    cfg = get_config(args, mode='val')
    cfg.val_bs = args.val_bs
    cfg.coco_gpu = args.coco_gpu
    cfg.decode_gpu = args.decode_gpu
    if cfg.coco_api:
        make_output_dirs()

    net = Yolact(cfg)
    net.load_weights(cfg.weight, cfg.cuda)
    net.eval()
    net = net.cuda()
    evaluate(net, cfg)


if __name__ == '__main__':
    main()
