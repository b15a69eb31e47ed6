"""Post-process API kept from the reference's utils/output_utils.py -- `nms` (:126-163),
`after_nms` (:200-233) and `draw_img` (:308-369) -- with the work done by the CUDA kernels behind
yb_detect / yb_mask_assemble / yb_draw_masks (include/yolact_b200.h).  Same arguments, same return
tuples, same "(None, ...)" convention for "no detections".  `detect_batched` and `after_nms_batched`
are the batched forms the reference lacks (its nms() squeezes a batch of 1, output_utils.py:127-130);
`blend_masks` is draw_img's overlay on device-resident frames, `blend_masks_batched` the same for a batch of images of any sizes,
and `lincomb_batched` draw_lincomb (cfg.save_lincomb) for a batch.

All inputs must be CUDA tensors (draw_img also takes numpy arrays, which it uploads); nothing here
falls back to the CPU.
"""
import ctypes

import torch

from .. import _lib
from .box_utils import anchors_tensor

_ws_cache = {}
_anchor_cache = {}
_palette_cache = {}


def _params(cfg, num_classes, coef_dim, no_clip=False):
    return _lib.DetectParams(float(cfg.nms_score_thre), float(cfg.nms_iou_thre), int(cfg.top_k),
                             int(cfg.max_detections), int(num_classes), int(coef_dim),
                             1 if getattr(cfg, 'traditional_nms', False) else 0, float(getattr(cfg, 'img_size', 0)), 1 if no_clip else 0)


def _workspace(nbytes, device):
    key = (device.index, 'detect')
    buf = _ws_cache.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
        _ws_cache[key] = buf
    return buf


def _device_anchors(anchors, device):
    if isinstance(anchors, torch.Tensor) and anchors.is_cuda and anchors.dtype == torch.float32:
        return anchors.reshape(-1, 4).contiguous()
    key = (id(anchors), len(anchors), device.index)
    hit = _anchor_cache.get(key)
    if hit is None:
        hit = anchors_tensor(anchors, device)
        _anchor_cache.clear()
        _anchor_cache[key] = hit
    return hit


def _require_cuda(*tensors):
    for t in tensors:
        if not (isinstance(t, torch.Tensor) and t.is_cuda):
            raise _lib.YolactB200Error('yolact_minimal_b200 post-process needs CUDA tensors (no CPU fallback)')


def record_fields(B, D, K):
    """(name, int32 offset, element count, shape, dtype) of every field of the flat detection record.  Field offsets are
    16-byte aligned: the post-process kernels store boxes / coefficients with 128-bit vector writes."""
    fields, o = [], 0
    for name, n, shape, dt in (('count', B, (B,), torch.int32), ('cls', B * D, (B, D), torch.int32), ('anchor', B * D, (B, D), torch.int32),
                               ('score', B * D, (B, D), torch.float32), ('box', B * D * 4, (B, D, 4), torch.float32),
                               ('coef', B * D * K, (B, D, K), torch.float32)):
        fields.append((name, o, n, shape, dt))
        o += (n + 3) // 4 * 4
    return fields, o


def record_numel(B, D, K):
    return record_fields(B, D, K)[1]


def record_views(flat, B, D, K):
    """Typed views of a flat int32 detection record -> the detect_batched dict; '_flat' is the buffer itself."""
    out = {'_flat': flat}
    for name, o, n, shape, dt in record_fields(B, D, K)[0]:
        out[name] = flat[o:o + n].view(dt).view(shape)
    return out


def detect_batched(class_pred, box_pred, coef_pred, anchors, cfg, no_clip=False):
    """Batched decode + (Fast|traditional) NMS + top-k.
    class_pred [B,A,C] (post-softmax), box_pred [B,A,4], coef_pred [B,A,K].
    Returns dict of padded tensors: count [B] int32, class [B,D] int32, anchor [B,D] int32,
    score [B,D], box [B,D,4], coef [B,D,K]  (D = cfg.max_detections)."""
    _require_cuda(class_pred, box_pred, coef_pred)
    dev = class_pred.device
    cls = class_pred.detach().to(torch.float32).contiguous()
    box = box_pred.detach().to(torch.float32).contiguous()
    coef = coef_pred.detach().to(torch.float32).contiguous()
    if cls.dim() == 2:
        cls, box, coef = cls[None], box[None], coef[None]
    B, A, C = cls.shape
    K = coef.shape[-1]
    anc = _device_anchors(anchors, dev)
    if anc.shape[0] != A:
        raise ValueError(f'anchors has {anc.shape[0]} rows, predictions have {A}')
    p = _params(cfg, C, K, no_clip)
    D = p.max_det
    L = _lib.lib()
    # ONE flat int32 buffer [count B | class B*D | anchor B*D | score B*D | box B*D*4 | coef B*D*K]; the dict entries are typed views
    # of it, so the kernels write the record that dist.gather_detections all-gathers directly (no pack pass)
    out = record_views(torch.empty(record_numel(B, D, K), dtype=torch.int32, device=dev), B, D, K)
    with torch.cuda.device(dev):
        nbytes = L.yb_detect_workspace_bytes(B, A, ctypes.byref(p))
        ws = _workspace(nbytes, dev)
        _lib.check(L.yb_detect(cls.data_ptr(), box.data_ptr(), coef.data_ptr(), anc.data_ptr(), B, A, ctypes.byref(p),
                               ws.data_ptr(), ws.numel(), out['count'].data_ptr(), out['cls'].data_ptr(),
                               out['anchor'].data_ptr(), out['score'].data_ptr(), out['box'].data_ptr(),
                               out['coef'].data_ptr(), torch.cuda.current_stream().cuda_stream), 'yb_detect')
    return out


def nms(class_pred, box_pred, coef_pred, proto_out, anchors, cfg):
    """Reference signature (utils/output_utils.py:126).  Batch of one image.
    Returns (class_ids int64 [d], scores [d], boxes [d,4], coefs [d,K], proto [P,P,K]) or
    (None,)*5 when nothing passes the score filter (:155)."""
    cls = class_pred.squeeze(0) if class_pred.dim() == 3 else class_pred
    box = box_pred.squeeze(0) if box_pred.dim() == 3 else box_pred
    coef = coef_pred.squeeze(0) if coef_pred.dim() == 3 else coef_pred
    proto = proto_out.squeeze(0) if proto_out.dim() == 4 else proto_out
    r = detect_batched(cls[None], box[None], coef[None], anchors, cfg)
    d = int(r['count'][0].item())          # the reference syncs here too (boolean-mask compaction)
    if d == 0:
        return None, None, None, None, None
    return (r['cls'][0, :d].long(), r['score'][0, :d].clone(), r['box'][0, :d].clone(), r['coef'][0, :d].clone(), proto)


def after_nms(ids_p, class_p, box_p, coef_p, proto_p, img_h, img_w, cfg=None, img_name=None, mask_dtype=torch.float32):
    """Reference signature (utils/output_utils.py:200).  Returns (ids, scores, boxes int32 [d,4]
    in pixels of max(img_h,img_w), masks [d,img_h,img_w] with values {0,1}) or (None,)*4.
    `mask_dtype=torch.uint8` writes byte masks instead of the reference's float32 (4x less HBM
    traffic), `mask_dtype='bits'` bit-packed masks [d,img_h,ceil(img_w/32)] (32x less; utils/mask_utils.py has
    the IoU / RLE stage that consumes them); unlike the reference, box_p is not modified in place."""
    if ids_p is None:
        return None, None, None, None
    _require_cuda(box_p, coef_p, proto_p)
    if cfg is not None and getattr(cfg, 'visual_thre', 0) > 0:              # :204-212
        keep = class_p >= cfg.visual_thre
        if not bool(keep.any()):
            return None, None, None, None
        ids_p, class_p, box_p, coef_p = ids_p[keep], class_p[keep], box_p[keep], coef_p[keep]
    dev = proto_p.device
    proto = proto_p.detach().to(torch.float32).contiguous()
    coef = coef_p.detach().to(torch.float32).contiguous()
    if cfg is not None and getattr(cfg, 'save_lincomb', False):                   # :214-215
        import cv2
        lincomb = lincomb_batched(proto[None], {'coef': coef[None]})
        cv2.imwrite(f'results/images/lincomb_{img_name}', lincomb[0].cpu().numpy())
    box = box_p.detach().to(torch.float32).contiguous()
    d, K = coef.shape
    P = proto.shape[0]
    if proto.shape[1] != P or proto.shape[2] != K:
        raise ValueError(f'proto {tuple(proto.shape)} does not match coef {tuple(coef.shape)}')
    crop = 0 if (cfg is not None and getattr(cfg, 'no_crop', False)) else 1
    f32 = mask_dtype == torch.float32
    fmt = 2 if isinstance(mask_dtype, str) and mask_dtype == 'bits' else (1 if f32 else 0)
    if fmt == 2:
        masks = torch.empty(d, int(img_h), (int(img_w) + 31) // 32, dtype=torch.int32, device=dev)
    else:
        masks = torch.empty(d, int(img_h), int(img_w), dtype=torch.float32 if f32 else torch.uint8, device=dev)
    boxes_px = torch.empty(d, 4, dtype=torch.int32, device=dev)
    L = _lib.lib()
    with torch.cuda.device(dev):
        ws = torch.empty(int(L.yb_mask_workspace_bytes(d, P)), dtype=torch.uint8, device=dev)
        _lib.check(L.yb_mask_assemble(proto.data_ptr(), coef.data_ptr(), box.data_ptr(), d, P, K, int(img_h), int(img_w),
                                      crop, fmt, ws.data_ptr(), ws.numel(), masks.data_ptr(),
                                      boxes_px.data_ptr(), torch.cuda.current_stream().cuda_stream), 'yb_mask_assemble')
    return ids_p, class_p, boxes_px, masks


def after_nms_batched(det, proto, sizes, crop=True):
    """after_nms for a whole detect_batched record, bit-packed masks, with no host sync on the counts (yb_mask_assemble_batch).
    det: detect_batched's dict (count [B], box [B,D,4], coef [B,D,K]); proto [B,P,P,K] (Yolact.forward's proto); sizes: B (h, w).
    Returns (boxes_px [B,D,4] int32: pixel boxes of max(h_b, w_b), zero at or past count[b]; a list of B packed-mask views
    [D, h_b, ceil(w_b/32)] int32 into one buffer, of which the first count[b] masks are written) -- the boxes_px and masks
    MapEvaluator.add takes.  Image b's first count[b] masks and boxes equal after_nms(..., mask_dtype='bits') on that image."""
    import numpy as np
    count, box, coef = det['count'], det['box'], det['coef']
    _require_cuda(count, box, coef, proto)
    dev = proto.device
    B, D, K = coef.shape
    proto = proto.detach().to(torch.float32).contiguous()
    P = proto.shape[1]
    if tuple(proto.shape) != (B, P, P, K) or tuple(box.shape) != (B, D, 4) or tuple(count.shape) != (B,):
        raise ValueError(f'proto {tuple(proto.shape)}, box {tuple(box.shape)}, count {tuple(count.shape)} do not match coef {tuple(coef.shape)}')
    hw = np.ascontiguousarray(np.asarray(sizes, dtype=np.int64).reshape(-1, 2))
    if hw.shape[0] != B or (hw <= 0).any() or (hw > 65535).any():
        raise ValueError(f'sizes must hold {B} (h, w) pairs in 1..65535, got {sizes}')
    n_words = D * hw[:, 0] * ((hw[:, 1] + 31) // 32)
    off = np.concatenate([[0], np.cumsum(n_words)]).astype(np.int64)
    hw32 = hw.astype(np.int32)
    count, box, coef = (t.to(dt).contiguous() for t, dt in ((count, torch.int32), (box, torch.float32), (coef, torch.float32)))
    masks = torch.empty(int(off[-1]), dtype=torch.int32, device=dev)
    boxes_px = torch.empty(B, D, 4, dtype=torch.int32, device=dev)
    L = _lib.lib()
    with torch.cuda.device(dev):
        ws = torch.empty(int(L.yb_mask_assemble_batch_workspace_bytes(B, D, P)), dtype=torch.uint8, device=dev)
        _lib.check(L.yb_mask_assemble_batch(proto.data_ptr(), coef.data_ptr(), box.data_ptr(), count.data_ptr(), B, D, P, K, hw32.ctypes.data, off.ctypes.data, masks.numel(), 1 if crop else 0, ws.data_ptr(),
                                            ws.numel(), masks.data_ptr(), boxes_px.data_ptr(), torch.cuda.current_stream().cuda_stream),
                   'yb_mask_assemble_batch')
    views = [masks[int(off[b]):int(off[b + 1])].view(D, int(h), (int(w) + 31) // 32) for b, (h, w) in enumerate(hw)]
    return boxes_px, views


# ---------------------------------------------------------------------------------------------------------------------------
# The ONNX / TensorRT callers' numpy twins (utils/output_utils.py:46-81,:166-197,:236-273; detect_with_onnx.py, detect_with_trt.py):
# numpy arrays in, numpy arrays out, same return conventions -- computed by the same CUDA kernels.  Semantics kept from the
# reference: NO clip of the decoded boxes to [0,1] (compare :186-190 with :153) and boolean masks.  Two documented differences:
# the reference decodes in float64 (its anchors are a float64 array) and resizes the masks with cv2.INTER_LINEAR; here the decode
# is the fp32 kernel and the resize the same half-pixel bilinear kernel as after_nms (boxes agree to ~1e-6, masks to a few pixels
# on the contour).
# ---------------------------------------------------------------------------------------------------------------------------
def _np_dev():
    if not torch.cuda.is_available():
        raise _lib.YolactB200Error('the numpy post-process twins run on a CUDA device (no CPU fallback)')
    return torch.device('cuda', torch.cuda.current_device())


def nms_numpy(class_pred, box_pred, coef_pred, proto_out, anchors, cfg):
    """utils/output_utils.py:166-197.  Returns (class_ids, class_thre, box_thre, coef_thre, proto_p) as numpy arrays or (None,)*5."""
    import numpy as np
    assert not getattr(cfg, 'traditional_nms', False), 'Traditional nms is not supported with numpy.'          # :193
    dev = _np_dev()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32))).to(dev)
    cls, box, coef = t(np.squeeze(class_pred)), t(np.squeeze(box_pred)), t(np.squeeze(coef_pred))
    proto = np.squeeze(np.asarray(proto_out))
    anc = t(np.asarray(anchors, dtype=np.float64).reshape(-1, 4))
    r = detect_batched(cls[None], box[None], coef[None], anc, cfg, no_clip=True)
    d = int(r['count'][0].item())
    if d == 0:
        return None, None, None, None, None
    return (r['cls'][0, :d].cpu().numpy().astype(np.int64), r['score'][0, :d].cpu().numpy(), r['box'][0, :d].cpu().numpy(),
            r['coef'][0, :d].cpu().numpy(), proto)


def after_nms_numpy(ids_p, class_p, box_p, coef_p, proto_p, img_h, img_w, cfg=None):
    """utils/output_utils.py:236-273.  Returns (ids, scores, boxes int32 [d,4], masks bool [d,img_h,img_w]) or (None,)*4."""
    import numpy as np
    if ids_p is None:
        return None, None, None, None
    if cfg and getattr(cfg, 'visual_thre', 0) > 0:
        keep = class_p >= cfg.visual_thre
        if not keep.any():
            return None, None, None, None
        ids_p, class_p, box_p, coef_p = ids_p[keep], class_p[keep], box_p[keep], coef_p[keep]
    assert not (cfg and getattr(cfg, 'save_lincomb', False)), 'save_lincomb is not supported in onnx mode.'   # :253
    dev = _np_dev()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32))).to(dev)
    r = after_nms(ids_p, class_p, t(box_p), t(coef_p), t(proto_p), img_h, img_w, cfg=None if cfg is None else _NoVisual(cfg), mask_dtype=torch.uint8)
    return ids_p, class_p, r[2].cpu().numpy().astype(np.int32), r[3].cpu().numpy().astype(bool)


class _NoVisual:
    """cfg view for after_nms_numpy: the score filter was already applied on the numpy side."""

    def __init__(self, cfg):
        self._cfg = cfg

    def __getattr__(self, k):
        if k == 'visual_thre':
            return 0
        return getattr(self._cfg, k)


# ---------------------------------------------------------------------------------------------------------------------------
# Drawing (utils/output_utils.py:308-369).  The mask overlay and the cutout matting run on the device (csrc/draw.cu); the box,
# label and fps pass is the reference's cv2 calls in the reference's order on the host image, which the caller needs there anyway
# (cv2.imwrite, VideoWriter).  Colours come from config.COLORS, this package's palette.
# ---------------------------------------------------------------------------------------------------------------------------
def _palette(num_classes, device):
    from ..config import COLORS
    nc = int(num_classes) - 1
    if not 1 <= nc <= len(COLORS):
        raise ValueError(f'num_classes={num_classes}: the palette has {len(COLORS)} colours')
    key = device.index
    pal = _palette_cache.get(key)
    if pal is None:
        pal = torch.from_numpy(COLORS.reshape(-1).copy()).to(device)
        _palette_cache[key] = pal
    return pal, nc


def _mask_operand(masks, n, h, w):
    """masks -> (contiguous 16-byte aligned CUDA tensor, yb mask code): float32 -> 1, uint8 / bool -> 0, int32 -> 2 (packed bits
    [n,h,ceil(w/32)], the after_nms(mask_dtype='bits') layout)."""
    if masks.dtype == torch.int32:
        fmt, shape = 2, (n, h, (w + 31) // 32)
    elif masks.dtype == torch.float32:
        fmt, shape = 1, (n, h, w)
    elif masks.dtype in (torch.uint8, torch.bool):
        fmt, shape = 0, (n, h, w)
        masks = masks.view(torch.uint8)
    else:
        raise _lib.YolactB200Error(f'masks of dtype {masks.dtype}: expected float32, uint8, bool or int32 (packed bits)')
    if tuple(masks.shape) != shape:
        raise _lib.YolactB200Error(f'masks {tuple(masks.shape)} do not match {n} detections on a {h}x{w} image (expected {shape})')
    masks = masks.contiguous()
    return (masks if masks.data_ptr() % 16 == 0 else masks.clone()), fmt


def _draw_operands(img, ids, masks):
    _require_cuda(img, ids, masks)
    if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3:
        raise ValueError(f'img must be uint8 [h,w,3], got {img.dtype} {tuple(img.shape)}')
    if not (ids.device == masks.device == img.device):
        raise _lib.YolactB200Error('img, ids and masks must be on the same device')
    h, w = int(img.shape[0]), int(img.shape[1])
    m, fmt = _mask_operand(masks, int(ids.shape[0]), h, w)
    return img.contiguous(), ids.to(torch.int32).contiguous(), m, fmt, h, w


def blend_masks(img, ids, masks, num_classes):
    """draw_img's mask overlay on device-resident frames (utils/output_utils.py:322-326): every pixel becomes
    cv2.addWeighted(COLORS[semantic], 0.4, img, 0.6, 0) with semantic = (sum_i masks_i * (ids_i + 1)) % (num_classes - 1).
    img CUDA uint8 [h,w,3]; ids [n] integer class ids; masks [n,h,w] {0,1} float32 / uint8 / bool, or int32 packed bits
    [n,h,ceil(w/32)].  Returns a new CUDA uint8 [h,w,3].  One kernel launch."""
    img, ids32, m, fmt, h, w = _draw_operands(img, ids, masks)
    pal, nc = _palette(num_classes, img.device)
    out = torch.empty_like(img)
    L = _lib.lib()
    with torch.cuda.device(img.device):
        _lib.check(L.yb_draw_masks(img.data_ptr(), h, w, m.data_ptr(), fmt, int(ids32.shape[0]), ids32.data_ptr(), pal.data_ptr(), nc,
                                   out.data_ptr(), torch.cuda.current_stream().cuda_stream), 'yb_draw_masks')
    return out


def visible_count(det, visual_thre):
    """after_nms' visual_thre filter (utils/output_utils.py:204-212) for a detect_batched record, on the device and without a sync:
    the record is sorted by descending score, so `score >= visual_thre` keeps a prefix of each image's detections; returns its
    length per image (int32 [B]).  The comparison is after_nms' own (a float32 tensor against the Python float)."""
    count = det['count']
    if not visual_thre > 0:
        return count
    D = det['score'].shape[1]
    live = torch.arange(D, device=count.device)[None] < count[:, None].long()
    return (live & (det['score'] >= visual_thre)).sum(1, dtype=torch.int32)


def blend_masks_batched(src, items, det, masks, num_classes):
    """blend_masks for a batch of images of any sizes, in one yb_draw_masks_batch launch and without a host sync on the counts.
    src: CUDA uint8 buffer holding the BGR images back to back, `items` its numpy yb_val_aug_item table (pack_images); det: a
    record with 'count' [B] (DEVICE) and 'cls' [B,D]; masks: after_nms_batched's list of packed-mask views [D,h_b,ceil(w_b/32)].
    Returns a new CUDA buffer laid out as src: image b blended with its first count[b] masks, or unchanged when count[b] <= 0."""
    import numpy as np
    from .augmentations import VAL_ITEM_DTYPE
    count, cls = det['count'], det['cls']
    _require_cuda(src, count, cls, *masks)
    items = np.ascontiguousarray(items, dtype=VAL_ITEM_DTYPE)
    B, D = int(cls.shape[0]), int(cls.shape[1])
    if src.dtype != torch.uint8 or src.dim() != 1 or len(items) != B or len(masks) != B or tuple(count.shape) != (B,):
        raise ValueError(f'src {src.dtype} {tuple(src.shape)}, {len(items)} items, {len(masks)} mask views and count '
                         f'{tuple(count.shape)} do not describe {B} images')
    storage = masks[0].untyped_storage()
    for b, (m, (_, h, w)) in enumerate(zip(masks, items.tolist())):
        if m.dtype != torch.int32 or tuple(m.shape) != (D, h, (w + 31) // 32) or not m.is_contiguous() or \
                m.untyped_storage().data_ptr() != storage.data_ptr():
            raise ValueError(f'mask view {b}: {m.dtype} {tuple(m.shape)} is not a contiguous [{D},{h},{(w + 31) // 32}] int32 view of '
                             'the batch buffer')
    base = storage.data_ptr()
    off = np.asarray([m.storage_offset() for m in masks] + [masks[-1].storage_offset() + masks[-1].numel()], np.int64)
    pal, nc = _palette(num_classes, src.device)
    ids32, count32 = cls.to(torch.int32).contiguous(), count.to(torch.int32).contiguous()
    out = torch.empty_like(src)
    L = _lib.lib()
    with torch.cuda.device(src.device):
        ws = torch.empty(int(L.yb_draw_masks_batch_workspace_bytes(B)), dtype=torch.uint8, device=src.device)
        _lib.check(L.yb_draw_masks_batch(src.data_ptr(), src.numel(), items.ctypes.data, B, base, off.ctypes.data, storage.nbytes() // 4,
                                         D, ids32.data_ptr(), count32.data_ptr(), pal.data_ptr(), nc, ws.data_ptr(), ws.numel(),
                                         out.data_ptr(), torch.cuda.current_stream().cuda_stream), 'yb_draw_masks_batch')
    return out


def _winter_lut(device):
    key = ('winter', device.index)
    lut = _palette_cache.get(key)
    if lut is None:
        import cv2
        import numpy as np
        # for uint8 input applyColorMap is this table lookup
        table = cv2.applyColorMap(np.arange(256, dtype=np.uint8)[:, None], cv2.COLORMAP_WINTER)[:, 0]
        lut = _palette_cache[key] = torch.from_numpy(np.ascontiguousarray(table)).to(device)
    return lut


def lincomb_batched(proto, det):
    """draw_lincomb (utils/output_utils.py:276-305, cfg.save_lincomb) for detection 0 of each image, one yb_draw_lincomb launch.
    proto [B,P,P,32] (Yolact.forward's proto); det: a record with 'coef' [B,D,32] and optionally 'count' [B] (DEVICE): images
    with count <= 0 are left unwritten (zero).  Returns CUDA uint8 [B, 4P, 8P, 3], the BGR image cv2.imwrite writes.  Coefficients
    of equal magnitude are ordered lower channel first (the reference's order for them is numpy's unstable argsort)."""
    coef = det['coef']
    count = det.get('count')
    _require_cuda(proto, coef, *([] if count is None else [count]))
    proto = proto.detach().to(torch.float32).contiguous()
    coef = coef.detach().to(torch.float32).contiguous()
    B, P, _, K = proto.shape
    if tuple(proto.shape) != (B, P, P, K) or coef.dim() != 3 or coef.shape[0] != B or coef.shape[2] != K:
        raise ValueError(f'proto {tuple(proto.shape)} does not match coef {tuple(coef.shape)}')
    count32 = None if count is None else count.to(torch.int32).contiguous()
    out = torch.zeros(B, 4 * P, 8 * P, 3, dtype=torch.uint8, device=proto.device)
    L = _lib.lib()
    with torch.cuda.device(proto.device):
        _lib.check(L.yb_draw_lincomb(proto.data_ptr(), coef.data_ptr(), None if count32 is None else count32.data_ptr(), B,
                                     int(coef.shape[1]), P, K, _winter_lut(proto.device).data_ptr(), out.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream), 'yb_draw_lincomb')
    return out


def cutout_masks(img, ids, boxes, masks, num_classes):
    """draw_img's cfg.cutout images (utils/output_utils.py:328-341) on the device.  Returns (total_obj [h,w,3], [crop_i]) as host
    uint8 arrays: total_obj = img where the semantic index is non-zero, else 255; crop_i = (img where masks_i, else 255)[y1:y2,
    x1:x2] with numpy's slicing of the int box (x1, y1, x2, y2) = boxes[i] (a host array)."""
    total, crops, off, shapes = cutout_masks_device(img, ids, boxes, masks, num_classes)
    flat = crops.cpu().numpy()
    out = [flat[off[i]:off[i + 1]].reshape(*shapes[i], 3) for i in range(len(shapes))]
    return total.cpu().numpy(), out


def cutout_masks_device(img, ids, boxes, masks, num_classes):
    """cutout_masks without the copies to the host: (total_obj, crops, offsets, shapes) with total_obj a CUDA uint8 [h,w,3], crops
    a CUDA uint8 buffer holding crop_i at bytes offsets[i] .. offsets[i+1] (host int64), and shapes[i] its (height, width)."""
    import numpy as np
    img, ids32, m, fmt, h, w = _draw_operands(img, ids, masks)
    n = int(ids32.shape[0])
    yyxx = np.zeros((max(n, 1), 4), np.int32)
    off = np.zeros(n + 1, np.int64)
    for i in range(n):
        x1, y1, x2, y2 = (int(v) for v in boxes[i, :4])
        ya, yb, _ = slice(y1, y2).indices(h)
        xa, xb, _ = slice(x1, x2).indices(w)
        yyxx[i] = ya, max(ya, yb), xa, max(xa, xb)
        off[i + 1] = off[i] + 3 * (yyxx[i, 1] - ya) * (yyxx[i, 3] - xa)
    dev = img.device
    total = torch.empty_like(img)
    crops = torch.empty(max(int(off[-1]), 1), dtype=torch.uint8, device=dev)
    yyxx_d, off_d = torch.from_numpy(yyxx).to(dev), torch.from_numpy(off).to(dev)
    _, nc = _palette(num_classes, dev)
    L = _lib.lib()
    with torch.cuda.device(dev):
        _lib.check(L.yb_draw_cutout(img.data_ptr(), h, w, m.data_ptr(), fmt, n, ids32.data_ptr(), nc, yyxx_d.data_ptr(), off_d.data_ptr(),
                                    total.data_ptr(), crops.data_ptr(), torch.cuda.current_stream().cuda_stream), 'yb_draw_cutout')
    return total, crops, off, [(int(yyxx[i, 1] - yyxx[i, 0]), int(yyxx[i, 3] - yyxx[i, 2])) for i in range(n)]


def draw_img(ids_p, class_p, box_p, mask_p, img_origin, cfg, img_name=None, fps=None):
    """Reference signature (utils/output_utils.py:308).  Returns the drawn uint8 [h,w,3] image: `img_origin` itself when ids_p is
    None, and drawn in place when cfg.hide_mask (as the reference does; cfg.real_time then returns a new array).
    ids_p / class_p / box_p / mask_p: after_nms' CUDA tensors (masks float32, uint8, or int32 packed bits from
    mask_dtype='bits') or numpy arrays (after_nms_numpy: bool masks), which are uploaded.  img_origin: host uint8 BGR [h,w,3],
    uploaded once; the overlay (and the cfg.cutout matting) runs on the device, then one copy of the image comes back for the
    box / label / fps pass, which uses the reference's cv2 calls."""
    if ids_p is None:
        return img_origin
    import cv2
    import numpy as np
    args = (ids_p, class_p, box_p, mask_p)
    if any(isinstance(t, torch.Tensor) and not t.is_cuda for t in args):
        raise _lib.YolactB200Error('draw_img needs CUDA tensors or numpy arrays (no CPU fallback)')
    if not (isinstance(img_origin, np.ndarray) and img_origin.dtype == np.uint8 and img_origin.ndim == 3 and img_origin.shape[2] == 3):
        raise ValueError('img_origin must be a host uint8 [h,w,3] array')
    host = lambda t: t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    ids_np, scores_np, boxes_np = host(ids_p), host(class_p), host(box_p)
    img_fused = img_origin
    if not cfg.hide_mask:
        cuda_args = [t for t in args if isinstance(t, torch.Tensor)]
        dev = cuda_args[0].device if cuda_args else _np_dev()
        up = lambda t: t if isinstance(t, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(t)).to(dev)
        ids_d, masks_d = up(ids_p), up(mask_p)
        img_d = torch.from_numpy(np.ascontiguousarray(img_origin)).to(dev)
        fused_d = blend_masks(img_d, ids_d, masks_d, cfg.num_classes)
        if cfg.cutout:
            total, crops = cutout_masks(img_d, ids_d, boxes_np, masks_d, cfg.num_classes)
            cv2.imwrite(f'results/images/{img_name}_total_obj.jpg', total)
            for i, crop in enumerate(crops):
                cv2.imwrite(f'results/images/{img_name}_{i}.jpg', crop)
        img_fused = fused_d.cpu().numpy()
    return draw_labels(img_fused, ids_np, scores_np, boxes_np, cfg, fps)


def draw_labels(img_fused, ids_np, scores_np, boxes_np, cfg, fps=None):
    """draw_img's host pass (utils/output_utils.py:343-369) on the overlaid uint8 image: boxes and labels (drawn in place) unless
    cfg.hide_bbox, and with cfg.real_time the fps text on a darkened corner (a new array).  Returns the image."""
    import cv2
    import numpy as np
    from ..config import COLORS
    scale = 0.6
    thickness = 1
    font = cv2.FONT_HERSHEY_DUPLEX
    if not cfg.hide_bbox:
        for i in reversed(range(ids_np.shape[0])):
            x1, y1, x2, y2 = (int(v) for v in boxes_np[i, :])
            color = COLORS[ids_np[i] + 1].tolist()
            cv2.rectangle(img_fused, (x1, y1), (x2, y2), color, thickness)
            class_name = cfg.class_names[ids_np[i]]
            text_str = f'{class_name}: {scores_np[i]:.2f}' if not cfg.hide_score else class_name
            text_w, text_h = cv2.getTextSize(text_str, font, scale, thickness)[0]
            cv2.rectangle(img_fused, (x1, y1), (x1 + text_w, y1 + text_h + 5), color, -1)
            cv2.putText(img_fused, text_str, (x1, y1 + 15), font, scale, (255, 255, 255), thickness, cv2.LINE_AA)
    if cfg.real_time:
        fps_str = f'fps: {fps:.2f}'
        text_w, text_h = cv2.getTextSize(fps_str, font, scale, thickness)[0]
        img_fused = img_fused.astype(np.float32)        # a shadow behind the fps text
        img_fused[0:text_h + 8, 0:text_w + 8] *= 0.6
        img_fused = img_fused.astype(np.uint8)
        cv2.putText(img_fused, fps_str, (0, text_h + 2), font, scale, (255, 255, 255), thickness, cv2.LINE_AA)
    return img_fused


# ---- JPEG encoding on the device (yb_jpeg_encode_batch): the bytes cv2.imencode('.jpg', img, [IMWRITE_JPEG_QUALITY, q]) returns
def jpeg_bound(h, w):
    """Worst-case size in bytes of the JPEG file of an h x w image (yb_jpeg_encode_bound)."""
    b = int(_lib.lib().yb_jpeg_encode_bound(int(h), int(w)))
    if b < 0:
        raise ValueError(f'no JPEG of a {h}x{w} image (1 .. 65535 each)')
    return b


def imencode_batched(buffer, items, quality=95):
    """cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, quality]) for a batch of images on the device, in one
    yb_jpeg_encode_batch call queued on the current stream (no host synchronisation).  `buffer` is a CUDA uint8 tensor holding
    uint8 BGR HWC images, `items` their numpy table in yb_val_aug_item's layout (augmentations.pack_images).
    Returns (data, offsets, lengths): data a CUDA uint8 tensor, offsets a host int64 array [n + 1], lengths a CUDA int64 tensor
    [n]; file i is data[offsets[i]:offsets[i] + lengths[i]]."""
    import numpy as np
    _require_cuda(buffer)
    if buffer.dtype != torch.uint8 or buffer.dim() != 1 or not buffer.is_contiguous():
        raise ValueError('buffer must be a contiguous 1-D uint8 tensor')
    items = np.ascontiguousarray(items, dtype=np.dtype(_lib.ValAugItem))
    n = len(items)
    if n == 0:
        raise ValueError('no images to encode')
    offsets = np.zeros(n + 1, np.int64)
    offsets[1:] = np.cumsum([jpeg_bound(h, w) for h, w in zip(items['h'], items['w'])])
    L = _lib.lib()
    item_p = items.ctypes.data_as(ctypes.POINTER(_lib.ValAugItem))
    dev = buffer.device
    with torch.cuda.device(dev):
        ws_bytes = int(L.yb_jpeg_encode_workspace_bytes(item_p, n))
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
        data = torch.empty(int(offsets[-1]), dtype=torch.uint8, device=dev)
        lengths = torch.empty(n, dtype=torch.int64, device=dev)
        _lib.check(L.yb_jpeg_encode_batch(buffer.data_ptr(), buffer.numel(), item_p, n, int(quality), ws.data_ptr(), ws_bytes,
                                          data.data_ptr(), offsets.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), lengths.data_ptr(),
                                          torch.cuda.current_stream().cuda_stream), 'yb_jpeg_encode_batch')
    return data, offsets, lengths


def imencode_gpu(img, quality=95):
    """cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, quality])[1] for one uint8 BGR image [h, w, 3] (numpy, or a CUDA
    tensor), encoded on the device: a 1-D numpy uint8 array of the file's bytes."""
    import numpy as np
    if isinstance(img, torch.Tensor):
        t = img.detach()
        if not t.is_cuda:
            t = t.cuda()
    else:
        t = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3:
        raise ValueError(f'expected a uint8 HxWx3 BGR image, got {t.dtype} {tuple(t.shape)}')
    h, w = int(t.shape[0]), int(t.shape[1])
    items = np.array([(0, h, w)], dtype=np.dtype(_lib.ValAugItem))
    data, _, lengths = imencode_batched(t.contiguous().reshape(-1), items, quality)
    return data[:int(lengths[0])].cpu().numpy()
