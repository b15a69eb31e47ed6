"""The reference's utils/common_utils.py API -- ProgressBar, save_best, save_latest, MakeJson, APDataObject, prep_metrics, calc_map
(:16-255), the names eval.py:14 and train.py:18 import -- with box and mask mAP computed on the GPU behind yb_eval_match /
yb_eval_ap (include/yolact_b200.h, csrc/eval.cu).

    ap_data = {'box': [[APDataObject() for _ in cfg.class_names] for _ in iou_thres], 'mask': [...]}     # eval.py:35-36
    prep_metrics(ap_data, ids_p, class_p, boxes_p, masks_p, gt, gt_masks, img_h, img_w, iou_thres)     # per image, eval.py:69
    table, box_row, mask_row = calc_map(ap_data, iou_thres, len(cfg.class_names), step)                 # eval.py:106

Every AP value and calc_map row equals the reference's float64 value bit for bit (DESIGN.md, evaluation stage).  Differences:
  * the matching runs on the device; APDataObject holds no data points, so push / add_gt_positives raise;
  * prep_metrics does not scale `gt` in place (the reference multiplies gt[:, :4] by the image size, :175-177);
  * an image with no detections contributes nothing, exactly as eval.py:53 skips it before prep_metrics (its gts are never
    counted); this holds for MapEvaluator.add and for a direct prep_metrics call alike;
  * scores are float32, the dtype nms produces, so ties are ties of float32 values;
  * calc_map's table is plain text (terminaltables is not a dependency); the rows are the reference's.
MapEvaluator is the batched form: it appends a batch of images with no host synchronisation.
"""
import ctypes
import glob
import json
import os
from collections import OrderedDict

import numpy as np
import torch

from .. import _lib
from ..config import COCO_LABEL_MAP
from . import mask_utils


# ---------------------------------------------------------------------------------------------------------------------------
# host-only helpers
# ---------------------------------------------------------------------------------------------------------------------------
class ProgressBar:
    """A text bar of `length` cells showing cur_val / max_val (the reference's eval.py / train.py progress display)."""

    def __init__(self, length, max_val):
        self.length, self.max_val = length, max_val
        self.cur_val = 0
        self.cur_num_bars = -1
        self.update_str()

    def update_str(self):
        filled = int(self.length * (self.cur_val / self.max_val))
        if filled != self.cur_num_bars:
            self.cur_num_bars = filled
            self.string = '█' * filled + '░' * (self.length - filled)

    def get_bar(self, new_val):
        self.cur_val = min(new_val, self.max_val)
        self.update_str()
        return self.string


def _weights_of(prefix, cfg_name):
    found = [p for p in glob.glob(f'weights/{prefix}*') if cfg_name in p]
    assert len(found) <= 1, f'Error, multiple {prefix} weight found.'
    return found


def save_best(net, mask_map, cfg_name, step):
    """Keep one weights/best_{mask_map}_{cfg_name}_{step}.pth: replace the stored one when mask_map is at least its mAP."""
    found = _weights_of('best', cfg_name)
    stored = float(os.path.basename(found[0]).split('_')[1]) if found else 0.
    if mask_map >= stored:
        for p in found:
            os.remove(p)
        print(f'\nSaving the best model as \'best_{mask_map}_{cfg_name}_{step}.pth\'.\n')
        torch.save(net.state_dict(), f'weights/best_{mask_map}_{cfg_name}_{step}.pth')


def save_latest(net, cfg_name, step):
    """Keep one weights/latest_{cfg_name}_{step}.pth."""
    for p in _weights_of('latest', cfg_name):
        os.remove(p)
    print(f'\nSaving the latest model as \'latest_{cfg_name}_{step}.pth\'.\n')
    torch.save(net.state_dict(), f'weights/latest_{cfg_name}_{step}.pth')


class MakeJson:
    """COCO result records for --coco_api (eval.py:60-67): boxes as [x, y, w, h] rounded to 0.1 px, masks as COCO RLE, classes
    mapped back to COCO category ids through COCO_LABEL_MAP."""

    def __init__(self):
        self.bbox_data, self.mask_data = [], []
        self.coco_cats = {label - 1: coco_id for coco_id, label in COCO_LABEL_MAP.items()}

    def add_bbox(self, image_id, category_id, bbox, score):
        x1, y1, x2, y2 = bbox[0], bbox[1], bbox[2], bbox[3]
        xywh = [round(float(v) * 10) / 10 for v in (x1, y1, x2 - x1, y2 - y1)]
        self.bbox_data.append({'image_id': int(image_id), 'category_id': self.coco_cats[int(category_id)], 'bbox': xywh,
                               'score': float(score)})

    def add_mask(self, image_id, category_id, segmentation, score):
        """segmentation: the full [h, w] {0,1} mask, a numpy array or a tensor; run-length encoded on the GPU
        (mask_utils.encode_rle: the object pycocotools.mask.encode returns, counts as str)."""
        if isinstance(segmentation, torch.Tensor):
            seg = segmentation.detach()
        else:
            seg = torch.from_numpy(np.ascontiguousarray(np.asarray(segmentation).astype(np.uint8)))
        if not seg.is_cuda:
            if not torch.cuda.is_available():
                raise _lib.YolactB200Error('MakeJson.add_mask encodes on a CUDA device (no CPU fallback)')
            seg = seg.cuda()
        h, w = seg.shape
        self.add_mask_rle(image_id, category_id, mask_utils.encode_rle(mask_utils.pack_masks(seg[None]), h, w)[0], score)

    def add_mask_rle(self, image_id, category_id, rle, score):
        """A mask record from its COCO RLE (mask_utils.encode_rle of packed masks)."""
        self.mask_data.append({'image_id': int(image_id), 'category_id': self.coco_cats[int(category_id)], 'segmentation': rle,
                               'score': float(score)})

    def dump(self):
        for data, path in ((self.bbox_data, 'results/bbox_detections.json'), (self.mask_data, 'results/mask_detections.json')):
            with open(path, 'w') as f:
                json.dump(data, f)


# ---------------------------------------------------------------------------------------------------------------------------
# the batched device accumulator
# ---------------------------------------------------------------------------------------------------------------------------
def _host_list(x):
    if x is None:
        return None
    if isinstance(x, torch.Tensor):
        if x.is_cuda:
            return None
        x = x.tolist()
    return [int(v) for v in x]


def _upload(values, dtype, device):
    """Host ints -> device tensor through pinned memory (asynchronous, no stream synchronisation)."""
    t = torch.tensor(values, dtype=dtype)
    if torch.cuda.is_available():
        t = t.pin_memory()
    return t.to(device, non_blocking=True)


def _flat_masks(masks, sizes, name, counts=None):
    """A list of per-image packed masks [n_b, h_b, ceil(w_b/32)] -> (flat int32 words, word offsets [B+1]).  The geometry of
    every entry must match `sizes`."""
    offs, parts = [0], []
    for b, (m, (h, w)) in enumerate(zip(masks, sizes)):
        if not (isinstance(m, torch.Tensor) and m.is_cuda):
            raise _lib.YolactB200Error(f'{name}[{b}] must be a CUDA tensor (no CPU fallback)')
        if m.dim() != 3 or tuple(m.shape[1:]) != (h, (w + 31) // 32) or m.dtype != torch.int32:
            raise _lib.YolactB200Error(f'{name}[{b}]: packed int32 masks [n,{h},{(w + 31) // 32}] expected for an image of {h}x{w}, '
                                       f'got {tuple(m.shape)} {m.dtype}')
        if counts is not None and m.shape[0] != counts[b]:
            raise _lib.YolactB200Error(f'{name}[{b}] holds {m.shape[0]} masks, the image has {counts[b]}')
        parts.append(m.reshape(-1))
        offs.append(offs[-1] + m.numel())
    flat = parts[0] if len(parts) == 1 else torch.cat(parts)
    return flat.contiguous(), offs


class MapEvaluator:
    """Box and mask AP of every (IoU type, threshold, class), accumulated on the device over batches of images.

        ev = MapEvaluator(num_classes, iou_thres)
        ev.add(det, boxes_px, masks, gt, gt_offset, gt_masks, sizes)     # any number of batches, no host sync
        ap, nonempty = ev.ap()                                           # float64 [2, T, C] (box, mask), bool [C]

    ap[type, t, c] is APDataObject.get_ap() of ap_data[type][t][c] after the same images went through eval.py's loop, and
    nonempty[c] is `not is_empty()`.  The record buffers grow from the host-known bound B * max_det per batch, so add() never
    waits for the device."""

    def __init__(self, num_classes, iou_thres, device=None, capacity=1024):
        thr = [float(x) for x in iou_thres]
        if not 1 <= len(thr) <= _lib.EVAL_MAX_THR:
            raise _lib.YolactB200Error(f'MapEvaluator: {len(thr)} IoU thresholds (1..{_lib.EVAL_MAX_THR} supported)')
        if num_classes < 1:
            raise _lib.YolactB200Error(f'MapEvaluator: num_classes={num_classes}')
        self.num_classes, self.iou_thres = int(num_classes), thr
        self.params = _lib.EvalParams(self.num_classes, len(thr), (ctypes.c_double * _lib.EVAL_MAX_THR)(*thr))
        self.device = None if device is None else torch.device(device)
        self._capacity0 = max(1, int(capacity))
        self._ws = None
        self._state = None
        self.reset()

    def reset(self):
        self._bound = 0
        self._result = None
        self._rec = None
        if self._state is not None:
            self._state.zero_()

    def _ensure(self, device):
        if self.device is None:
            self.device = device
        if device != self.device:
            raise _lib.YolactB200Error(f'MapEvaluator lives on {self.device}, got tensors on {device}')
        if self._state is None:
            L = _lib.lib()
            self._state = torch.zeros(int(L.yb_eval_state_bytes(ctypes.byref(self.params))), dtype=torch.uint8, device=self.device)

    def _reserve(self, extra):
        need = self._bound + extra
        cap = 0 if self._rec is None else self._rec[0].numel()
        if need <= cap:
            return
        new = max(need, 2 * cap, self._capacity0)
        rec = (torch.empty(new, dtype=torch.float32, device=self.device), torch.empty(new, dtype=torch.int32, device=self.device),
               torch.empty(new, dtype=torch.int32, device=self.device))
        if self._rec is not None and self._bound:
            for dst, src in zip(rec, self._rec):
                dst[:self._bound].copy_(src[:self._bound])
        self._rec = rec

    def _workspace(self, nbytes):
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
        return self._ws

    @property
    def capacity(self):
        return 0 if self._rec is None else self._rec[0].numel()

    def add(self, det, boxes_px, masks, gt, gt_offset, gt_masks, sizes):
        """Append a batch of B images.
          det        detect_batched's dict (count [B], cls [B,D], score [B,D]); only the first count[b] detections of image b count
          boxes_px   [B,D,4] int32 pixel boxes (after_nms' boxes of every image, padded to D)
          masks      list of B packed CUDA masks [n_b, h_b, ceil(w_b/32)] int32 with n_b >= count[b] (after_nms(..., 'bits'))
          gt         [G,5] float32 CUDA: x1,y1,x2,y2 in [0,1] and the class, all images back to back
          gt_offset  [B+1]: image b owns gt rows gt_offset[b] .. gt_offset[b+1] (list, CPU or CUDA tensor; None = from gt_masks)
          gt_masks   list of B packed CUDA gt masks [g_b, h_b, ceil(w_b/32)] int32
          sizes      list of B (h, w)
        An image with count 0 contributes nothing (eval.py:53)."""
        count, cls, score = det['count'], det['cls'], det['score']
        for name, t in (('count', count), ('cls', cls), ('score', score), ('boxes_px', boxes_px), ('gt', gt)):
            if not (isinstance(t, torch.Tensor) and t.is_cuda):
                raise _lib.YolactB200Error(f'MapEvaluator.add: {name} must be a CUDA tensor (no CPU fallback)')
        B, D = cls.shape
        sizes = [(int(h), int(w)) for h, w in sizes]
        if not (count.shape == (B,) and score.shape == (B, D) and tuple(boxes_px.shape) == (B, D, 4) and len(masks) == B
                and len(gt_masks) == B and len(sizes) == B):
            raise _lib.YolactB200Error(f'MapEvaluator.add: inconsistent batch: count {tuple(count.shape)}, cls {tuple(cls.shape)}, '
                                       f'score {tuple(score.shape)}, boxes {tuple(boxes_px.shape)}, {len(masks)} / {len(gt_masks)} '
                                       f'mask entries, {len(sizes)} sizes')
        if gt.dim() != 2 or gt.shape[1] != 5:
            raise _lib.YolactB200Error(f'MapEvaluator.add: gt must be [G,5], got {tuple(gt.shape)}')
        if B == 0:
            return
        self._ensure(gt.device)
        G = gt.shape[0]
        g_counts = [int(m.shape[0]) for m in gt_masks]
        host_off = _host_list(gt_offset)
        if gt_offset is None:
            host_off = np.concatenate([[0], np.cumsum(g_counts)]).astype(int).tolist()
        if host_off is not None:
            if len(host_off) != B + 1 or host_off[0] != 0 or host_off[-1] != G or \
                    [host_off[b + 1] - host_off[b] for b in range(B)] != g_counts:
                raise _lib.YolactB200Error(f'MapEvaluator.add: gt_offset {host_off} does not match gt [{G},5] and the gt masks {g_counts}')
        elif sum(g_counts) != G:
            raise _lib.YolactB200Error(f'MapEvaluator.add: {sum(g_counts)} gt masks for {G} gt rows')
        dmask, doff = _flat_masks(masks, sizes, 'masks')
        gmask, goff = _flat_masks(gt_masks, sizes, 'gt_masks')
        offs = _upload(doff + goff, torch.int64, self.device)
        ints = _upload([v for hw in sizes for v in hw] + (host_off or []), torch.int32, self.device)
        hw = ints[:2 * B]
        goff_dev = (ints[2 * B:] if host_off is not None else gt_offset.to(device=self.device, dtype=torch.int32)).contiguous()
        self._reserve(B * D)
        count = count.to(torch.int32).contiguous()
        cls = cls.to(torch.int32).contiguous()
        score = score.to(torch.float32).contiguous()
        boxes = boxes_px.to(torch.int32).contiguous()
        gtf = gt.to(torch.float32).contiguous()
        L = _lib.lib()
        p = ctypes.byref(self.params)
        with torch.cuda.device(self.device):
            ws = self._workspace(L.yb_eval_match_workspace_bytes(B, D, G, p))
            rs, rc, rt = self._rec
            _lib.check(L.yb_eval_match(p, B, D, count.data_ptr(), cls.data_ptr(), score.data_ptr(), boxes.data_ptr(),
                                       dmask.data_ptr() if dmask.numel() else None, offs[:B + 1].data_ptr(), dmask.numel(),
                                       hw.data_ptr(), gtf.data_ptr() if G else None, goff_dev.data_ptr(), G,
                                       gmask.data_ptr() if gmask.numel() else None, offs[B + 1:].data_ptr(), gmask.numel(),
                                       rs.data_ptr(), rc.data_ptr(), rt.data_ptr(), rs.numel(), self._state.data_ptr(),
                                       ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream), 'yb_eval_match')
        self._bound += B * D
        self._result = None

    def ap(self):
        """-> (ap float64 numpy [2, T, C], nonempty bool numpy [C]); computed once per state (synchronises)."""
        if self._result is not None:
            return self._result
        T, C = len(self.iou_thres), self.num_classes
        if self._state is None:
            self._result = (np.zeros((2, T, C)), np.zeros(C, bool))
            return self._result
        L = _lib.lib()
        p = ctypes.byref(self.params)
        n = self._bound
        out = torch.empty(2 * T * C, dtype=torch.float64, device=self.device)
        nonempty = torch.empty(C, dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            ws = torch.empty(int(L.yb_eval_ap_workspace_bytes(n, p)), dtype=torch.uint8, device=self.device)
            rs, rc, rt = self._rec if self._rec is not None else (None, None, None)
            _lib.check(L.yb_eval_ap(p, rs.data_ptr() if n else None, rc.data_ptr() if n else None, rt.data_ptr() if n else None, n,
                                    self._state.data_ptr(), ws.data_ptr(), ws.numel(), out.data_ptr(), nonempty.data_ptr(),
                                    torch.cuda.current_stream().cuda_stream), 'yb_eval_ap')
        flags = int(self._state[12:16].view(torch.int32).item())
        if flags:
            raise _lib.YolactB200Error(f'MapEvaluator: the record buffers overflowed (flags {flags})' if flags & 1 else
                                       f'MapEvaluator: an image\'s mask or gt offsets lie outside its buffers (flags {flags})')
        self._result = (out.cpu().numpy().reshape(2, T, C), nonempty.cpu().numpy().astype(bool))
        return self._result

    def num_records(self):
        """Records appended so far (synchronises)."""
        return 0 if self._state is None else int(self._state[:8].view(torch.int64).item())


# ---------------------------------------------------------------------------------------------------------------------------
# the reference's per-image API on top of MapEvaluator
# ---------------------------------------------------------------------------------------------------------------------------
_TYPES = ('box', 'mask')


class APDataObject:
    """One (IoU type, threshold, class) entry of ap_data.  prep_metrics binds it to the MapEvaluator that accumulates the whole
    ap_data on the device; is_empty() / get_ap() read that evaluator's result."""

    def __init__(self):
        self._ev = None
        self._key = None

    def _bind(self, ev, typ, t, c):
        self._ev, self._key = ev, (typ, t, c)

    def push(self, score, is_true):
        raise _lib.YolactB200Error('APDataObject.push: detections are matched and accumulated on the GPU by prep_metrics / '
                                   'MapEvaluator; there is no host-side list of data points')

    def add_gt_positives(self, num_positives):
        raise _lib.YolactB200Error('APDataObject.add_gt_positives: gt counts are accumulated on the GPU by prep_metrics / '
                                   'MapEvaluator')

    def is_empty(self):
        if self._ev is None:
            return True
        return not bool(self._ev.ap()[1][self._key[2]])

    def get_ap(self):
        if self._ev is None:
            return 0
        return float(self._ev.ap()[0][self._key])


def evaluator_of(ap_data):
    """The MapEvaluator ap_data is bound to (None before the first prep_metrics)."""
    return ap_data['box'][0][0]._ev


def _bind(ap_data, iou_thres, device):
    ev = evaluator_of(ap_data)
    if ev is not None:
        return ev
    T, C = len(ap_data['box']), len(ap_data['box'][0])
    if len(iou_thres) != T or len(ap_data['mask']) != T:
        raise _lib.YolactB200Error(f'prep_metrics: ap_data has {T} thresholds, iou_thres {len(iou_thres)}')
    ev = MapEvaluator(C, iou_thres, device=device)
    for typ, name in enumerate(_TYPES):
        for t in range(T):
            for c in range(C):
                ap_data[name][t][c]._bind(ev, typ, t, c)
    return ev


def _packed(m, h, w, what):
    if not (isinstance(m, torch.Tensor) and m.is_cuda):
        raise _lib.YolactB200Error(f'prep_metrics: {what} must be a CUDA tensor (no CPU fallback)')
    if m.dtype == torch.int32:                                    # after_nms(..., mask_dtype='bits'); geometry checked by add()
        return m
    if m.numel() != m.shape[0] * h * w:
        raise _lib.YolactB200Error(f'prep_metrics: {what} {tuple(m.shape)} does not hold [n,{h},{w}] masks')
    return mask_utils.pack_masks(m.reshape(m.shape[0], h, w))


def prep_metrics(ap_data, ids_p, classes_p, boxes_p, masks_p, gt, gt_masks, height, width, iou_thres):
    """utils/common_utils.py:174-216 for one image, on the GPU.  ids_p / classes_p: Python lists (eval.py:57-58); boxes_p: int32
    CUDA pixel boxes [d,4]; masks_p: CUDA {0,1} masks [d,h,w] (float, uint8 or bool) or after_nms' packed int32 masks
    [d,h,ceil(w/32)]; gt: CUDA [g,5] with the box in [0,1] (not modified, unlike the reference); gt_masks: CUDA {0,1} masks
    [g,h,w].  Binds ap_data to one MapEvaluator on the first call; nothing synchronises until an AP is read."""
    h, w = int(height), int(width)
    dev = boxes_p.device if isinstance(boxes_p, torch.Tensor) else None
    if not (isinstance(boxes_p, torch.Tensor) and boxes_p.is_cuda and isinstance(gt, torch.Tensor) and gt.is_cuda):
        raise _lib.YolactB200Error('prep_metrics: boxes_p and gt must be CUDA tensors (no CPU fallback)')
    ev = _bind(ap_data, iou_thres, dev)
    d = len(ids_p)
    if len(classes_p) != d or boxes_p.shape[0] != d:
        raise _lib.YolactB200Error(f'prep_metrics: {d} ids, {len(classes_p)} scores, {boxes_p.shape[0]} boxes')
    bits = _packed(masks_p, h, w, 'masks_p')
    gbits = _packed(gt_masks, h, w, 'gt_masks')
    D = max(d, 1)
    rec = np.zeros(1 + 2 * D, np.int32)
    rec[0] = d
    rec[1:1 + d] = np.asarray(ids_p, np.int64)
    rec[1 + D:1 + D + d] = np.asarray(classes_p, np.float32).view(np.int32)
    r = _upload(rec.tolist(), torch.int32, gt.device)
    det = {'count': r[:1], 'cls': r[1:1 + D].view(1, D), 'score': r[1 + D:].view(torch.float32).view(1, D)}
    boxes = boxes_p.to(torch.int32).contiguous().view(1, d, 4) if d else torch.zeros(1, 1, 4, dtype=torch.int32, device=gt.device)
    ev.add(det, boxes, [bits], gt.reshape(-1, 5), [0, gt.shape[0]], [gbits], [(h, w)])


def _table(rows):
    cols = [max(len(str(r[i])) for r in rows) for i in range(len(rows[0]))]
    line = '+' + '+'.join('-' * (c + 2) for c in cols) + '+'
    fmt = lambda r: '| ' + ' | '.join(str(v).ljust(c) for v, c in zip(r, cols)) + ' |'
    return '\n'.join([line, fmt(rows[0]), line] + [fmt(r) for r in rows[1:]] + [line])


def calc_map(ap_data, iou_thres, num_classes, step):
    """utils/common_utils.py:219-255: per IoU threshold the mean AP (x 100) over the non-empty classes, 'all' = the mean over
    the thresholds, rounded to 2 places.  Returns (table_str, box_row, mask_row) with rows ['box', all, 50, 55, ..., 95]."""
    print('\nCalculating mAP...')
    aps = [{'box': [], 'mask': []} for _ in iou_thres]
    for c in range(num_classes):
        for t in range(len(iou_thres)):
            for name in _TYPES:
                obj = ap_data[name][t][c]
                if not obj.is_empty():
                    aps[t][name].append(obj.get_ap())
    all_maps = {'box': OrderedDict(), 'mask': OrderedDict()}
    for name in _TYPES:
        all_maps[name]['all'] = 0
        for t, thr in enumerate(iou_thres):
            vals = aps[t][name]
            all_maps[name][int(thr * 100)] = sum(vals) / len(vals) * 100 if vals else 0
        all_maps[name]['all'] = sum(all_maps[name].values()) / (len(all_maps[name]) - 1)
    header = [f'{step // 1000}k' if step else ''] + list(all_maps['box'].keys())
    box_row = ['box'] + [round(v, 2) for v in all_maps['box'].values()]
    mask_row = ['mask'] + [round(v, 2) for v in all_maps['mask'].values()]
    return _table([header, box_row, mask_row]), box_row, mask_row
