"""COCO's own box and mask mAP on the GPU: what `--coco_api` gets from pycocotools' COCOeval (default Params, iouType 'bbox' and
'segm'), computed from the batched evaluation loop's device tensors with no result JSON, behind yb_cocoeval_match /
yb_cocoeval_accumulate (include/yolact_b200.h, csrc/cocoeval.cu).

    ev = CocoEvaluator(coco, cfg.continuous_id, device)
    ev.add(det, boxes_px, masks, packed)        # per batch (COCOValDetection(..., coco_eval=True) batches), no host sync
    arrays = ev.accumulate()                    # {'bbox': {'precision', 'recall'}, 'segm': {...}}, numpy float64
    stats = ev.summarize()                      # [2, 12]: COCOeval.stats of bbox and segm, printed as COCOeval prints them

precision / recall equal COCOeval's arrays for the detections eval.py's --coco_api path writes, bit for bit, and the stats are
computed from them on the host exactly as COCOeval.summarize does (DESIGN.md, COCO mAP on the GPU).  The evaluation parameters
are COCOeval's defaults and are not settable: IoU thresholds np.linspace(.5, .95, 10), recall thresholds np.linspace(0, 1, 101),
maxDets 1 / 10 / 100, area ranges all / small / medium / large.
"""
import ctypes

import numpy as np
import torch

from .. import _lib
from .common_utils import _flat_masks, _upload

IOU_THRS = np.linspace(.5, .95, 10)
REC_THRS = np.linspace(0, 1, 101)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0, 1e10], [0, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e10]]
AREA_LBL = ['all', 'small', 'medium', 'large']
TYPES = ('bbox', 'segm')


def _summarize_one(precision, recall, ap, iou_idx=None, area='all', max_dets=100):
    """One line of COCOeval.summarize: the mean of the entries > -1 (numpy's pairwise sum), or -1."""
    a, m = [AREA_LBL.index(area)], [MAX_DETS.index(max_dets)]
    if ap:
        s = precision if iou_idx is None else precision[[iou_idx]]
        s = s[:, :, :, a, m]
    else:
        s = recall if iou_idx is None else recall[[iou_idx]]
        s = s[:, :, a, m]
    mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
    iou_str = f'{IOU_THRS[0]:0.2f}:{IOU_THRS[-1]:0.2f}' if iou_idx is None else f'{IOU_THRS[iou_idx]:0.2f}'
    title, kind = ('Average Precision', '(AP)') if ap else ('Average Recall', '(AR)')
    line = ' {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}'.format(title, kind, iou_str, area, max_dets, mean_s)
    return mean_s, line


def summarize(precision, recall):
    """COCOeval.summarize for one iouType: -> (stats float64 [12], the 12 printed lines).  @.5 and @.75 are iouThrs[0] and [5]."""
    specs = [(1, None, 'all', 100), (1, 0, 'all', 100), (1, 5, 'all', 100), (1, None, 'small', 100), (1, None, 'medium', 100),
             (1, None, 'large', 100), (0, None, 'all', 1), (0, None, 'all', 10), (0, None, 'all', 100), (0, None, 'small', 100),
             (0, None, 'medium', 100), (0, None, 'large', 100)]
    stats, lines = np.zeros((12,)), []
    for i, (ap, t, area, md) in enumerate(specs):
        stats[i], line = _summarize_one(precision, recall, ap, t, area, md)
        lines.append(line)
    return stats, lines


def _params(num_classes, num_images):
    p = _lib.CocoEvalParams()
    p.num_classes, p.num_images = int(num_classes), int(num_images)
    for i, v in enumerate(IOU_THRS):
        p.iou_thr[i] = float(v)
    for i, v in enumerate(REC_THRS):
        p.rec_thr[i] = float(v)
    for i, (lo, hi) in enumerate(AREA_RNG):
        p.area_rng[i][0], p.area_rng[i][1] = float(lo), float(hi)
    for i, v in enumerate(MAX_DETS):
        p.max_dets[i] = v
    return p


def _pinned_to(t, device):
    """Host tensor -> device without a stream synchronisation (page-locked first when it is not)."""
    return (t if t.is_pinned() else t.pin_memory()).to(device, non_blocking=True)


class CocoEvaluator:
    """COCOeval's precision / recall for bbox and segm, accumulated on the device over batches of images.

    coco           any object with `imgToAnns` (image id -> annotations with 'category_id', 'area', 'iscrowd'): the annotation set.
                   Its images, in ascending id order, are COCOeval's imgIds; every non-crowd annotation counts as a gt to find,
                   also in images never added.
    continuous_id  COCO category id -> 1-based continuous label (cfg.continuous_id); the labels are COCOeval's catIds in order.
    The record buffers grow from the host-known bound B * max_det per batch, so add() never waits for the device."""

    def __init__(self, coco, continuous_id, device=None, capacity=1024):
        ids = sorted(coco.imgToAnns.keys())
        if not ids:
            raise _lib.YolactB200Error('CocoEvaluator: the annotation set has no image')
        self.rank = {img: r for r, img in enumerate(ids)}
        self.num_classes = int(max(continuous_id.values()))
        npig = np.zeros((self.num_classes, len(AREA_RNG)), np.int64)
        for img in ids:
            for a in coco.imgToAnns[img]:
                if a['iscrowd']:
                    continue
                k = continuous_id[a['category_id']] - 1
                for r, (lo, hi) in enumerate(AREA_RNG):
                    if lo <= a['area'] <= hi:
                        npig[k, r] += 1
        self.npig = npig
        self.params = _params(self.num_classes, len(ids))
        self.device = None if device is None else torch.device(device)
        self._capacity0 = max(1, int(capacity))
        self._state = self._npig = self._rec = self._ws = None
        self._bound = 0
        self._result = None

    def _ensure(self, device):
        if self.device is None:
            self.device = device
        if device != self.device:
            raise _lib.YolactB200Error(f'CocoEvaluator lives on {self.device}, got tensors on {device}')
        if self._state is None:
            self._state = torch.zeros(int(_lib.lib().yb_cocoeval_state_bytes()), dtype=torch.uint8, device=device)
            self._npig = _upload(self.npig.reshape(-1).tolist(), torch.int64, device)

    def _reserve(self, extra):
        need = self._bound + extra
        cap = 0 if self._rec is None else self._rec.numel() // _lib.COCOEVAL_RECORD_BYTES
        if need <= cap:
            return
        new = max(need, 2 * cap, self._capacity0)
        rec = torch.empty(new * _lib.COCOEVAL_RECORD_BYTES, dtype=torch.uint8, device=self.device)
        if self._rec is not None and self._bound:
            n = self._bound * _lib.COCOEVAL_RECORD_BYTES
            rec[:n].copy_(self._rec[:n])
        self._rec = rec

    def _workspace(self, nbytes):
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
        return self._ws

    def add(self, det, boxes_px, masks, packed):
        """Append a batch of B images.
          det       detect_batched's dict (count [B], cls [B,D], score [B,D]); only the first count[b] detections of image b count
          boxes_px  [B,D,4] int32 pixel boxes (after_nms_batched)
          masks     list of B packed CUDA masks [n_b, h_b, ceil(w_b/32)] int32 with n_b >= count[b] (after_nms_batched)
          packed    the batch's PackedValBatch from COCOValDetection(..., coco_eval=True): image ids, sizes and every annotation
        Detections are kept as the result JSON would keep them: (y2-y1)*(x2-x1) > 0, at most 100 per (image, class)."""
        count, cls, score = det['count'], det['cls'], det['score']
        for name, t in (('count', count), ('cls', cls), ('score', score), ('boxes_px', boxes_px)):
            if not (isinstance(t, torch.Tensor) and t.is_cuda):
                raise _lib.YolactB200Error(f'CocoEvaluator.add: {name} must be a CUDA tensor (no CPU fallback)')
        if getattr(packed, 'ann_cls', None) is None:
            raise _lib.YolactB200Error('CocoEvaluator.add: the batch carries no annotations (COCOValDetection(..., coco_eval=True))')
        B, D = cls.shape
        sizes = [(int(h), int(w)) for h, w in packed.sizes]
        if not (count.shape == (B,) and score.shape == (B, D) and tuple(boxes_px.shape) == (B, D, 4) and len(masks) == B
                and len(packed) == B):
            raise _lib.YolactB200Error(f'CocoEvaluator.add: inconsistent batch: count {tuple(count.shape)}, cls {tuple(cls.shape)}, '
                                       f'score {tuple(score.shape)}, boxes {tuple(boxes_px.shape)}, {len(masks)} mask entries, '
                                       f'{len(packed)} images')
        missing = [i for i in packed.ids if i not in self.rank]
        if missing:
            raise _lib.YolactB200Error(f'CocoEvaluator.add: image ids {missing[:5]} are not in the annotation set')
        if B == 0:
            return
        self._ensure(count.device)
        G = int(packed.ann_cls.shape[0])
        dmask, doff = _flat_masks(masks, sizes, 'masks')
        offs = _upload(doff + list(packed.ann_mask_off), torch.int64, self.device)
        ints = _upload([v for hw in sizes for v in hw] + [self.rank[i] for i in packed.ids] + list(packed.ann_offset), torch.int32,
                       self.device)
        gcls, gbox, garea, gcrowd, gmask = (_pinned_to(t, self.device) for t in (packed.ann_cls, packed.ann_box, packed.ann_area,
                                                                                   packed.ann_crowd, packed.ann_masks))
        self._reserve(B * D)
        count = count.to(torch.int32).contiguous()
        cls = cls.to(torch.int32).contiguous()
        score = score.to(torch.float32).contiguous()
        boxes = boxes_px.to(torch.int32).contiguous()
        L = _lib.lib()
        p = ctypes.byref(self.params)
        ptr = lambda t: t.data_ptr() if t.numel() else None
        with torch.cuda.device(self.device):
            ws = self._workspace(L.yb_cocoeval_match_workspace_bytes(B, D, G))
            cap = self._rec.numel() // _lib.COCOEVAL_RECORD_BYTES
            _lib.check(L.yb_cocoeval_match(p, B, D, count.data_ptr(), cls.data_ptr(), score.data_ptr(), boxes.data_ptr(), ptr(dmask),
                                           offs[:B + 1].data_ptr(), dmask.numel(), ints[:2 * B].data_ptr(), ints[2 * B:3 * B].data_ptr(),
                                           ptr(gcls), ptr(gbox), ptr(garea), ptr(gcrowd), ints[3 * B:].data_ptr(), G, ptr(gmask),
                                           offs[B + 1:].data_ptr(), gmask.numel(), self._rec.data_ptr(), cap, self._state.data_ptr(),
                                           ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream), 'yb_cocoeval_match')
        self._bound += B * D
        self._result = None

    def accumulate(self):
        """-> {'bbox': {'precision' [10,101,K,4,3], 'recall' [10,K,4,3]}, 'segm': {...}}: COCOeval.eval's arrays, numpy float64
        (synchronises; computed once per state)."""
        if self._result is not None:
            return self._result
        self._ensure(self.device or torch.device('cuda', torch.cuda.current_device()))
        K, n = self.num_classes, self._bound
        T, R, A, M = len(IOU_THRS), len(REC_THRS), len(AREA_RNG), len(MAX_DETS)
        L = _lib.lib()
        prec = torch.empty(2 * T * R * K * A * M, dtype=torch.float64, device=self.device)
        rec = torch.empty(2 * T * K * A * M, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            ws = torch.empty(int(L.yb_cocoeval_accumulate_workspace_bytes(n)), dtype=torch.uint8, device=self.device)
            _lib.check(L.yb_cocoeval_accumulate(ctypes.byref(self.params), self._rec.data_ptr() if n else None, n, self._state.data_ptr(),
                                                self._npig.data_ptr(), ws.data_ptr(), ws.numel(), prec.data_ptr(), rec.data_ptr(),
                                                torch.cuda.current_stream().cuda_stream), 'yb_cocoeval_accumulate')
        flags = int(self._state[12:16].view(torch.int32).item())
        if flags:
            what = ['the record buffers overflowed', 'an image\'s mask or annotation offsets lie outside its buffers',
                    'an image rank lies outside the annotation set']
            raise _lib.YolactB200Error(f'CocoEvaluator: {"; ".join(w for i, w in enumerate(what) if flags >> i & 1)} (flags {flags})')
        prec = prec.cpu().numpy().reshape(2, T, R, K, A, M)
        rec = rec.cpu().numpy().reshape(2, T, K, A, M)
        self._result = {name: {'precision': prec[i], 'recall': rec[i]} for i, name in enumerate(TYPES)}
        return self._result

    def summarize(self):
        """COCOeval.summarize for bbox and segm: prints both blocks under eval.py's headers, returns stats float64 [2, 12]."""
        res = self.accumulate()
        out = np.zeros((2, 12))
        for i, (name, header) in enumerate(zip(TYPES, ('\nEvaluating BBoxes:', '\nEvaluating Masks:'))):
            out[i], lines = summarize(res[name]['precision'], res[name]['recall'])
            print(header)
            print('\n'.join(lines))
        return out
