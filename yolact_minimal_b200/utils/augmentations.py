"""Augmentation on the GPU.

`val_aug` kept from the reference's utils/augmentations.py:219-227, computed on the GPU by
yb_val_aug (one fused kernel: pad-to-square with the BGR mean, bilinear resize, normalise,
BGR->RGB, HWC->CHW).  Takes the uint8 BGR image (numpy HWC, as cv2.imread returns it, or a CUDA
uint8 tensor) and returns a CUDA float32 tensor [3, val_size, val_size].
`val_aug_batch` does the same for a batch of images of any sizes packed in one buffer
(`pack_images`, `PackedValBatch`), in one yb_val_aug_batch launch; image b of its output equals
`val_aug` on image b bit for bit.

`train_aug` (:230-252) is split in two.  Every random draw it makes depends only on shapes, boxes
and labels, never on pixel values, so `train_aug_plan` replays those draws on the host (the same
`random` calls in the same order, the same float64 box arithmetic) and returns a small plan without
touching a pixel; `train_aug_batch` then applies a batch of plans to the raw uint8 images and masks
in one yb_train_aug launch.  With the same `random` state the plan's boxes and labels are the
reference's bit for bit.
"""
import ctypes as C
import random
from dataclasses import dataclass

import numpy as np
import torch

from .. import _lib


def val_aug(img, val_size, device='cuda'):
    if isinstance(img, np.ndarray):
        if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
            raise ValueError(f'expected a uint8 HxWx3 BGR image, got {img.dtype} {img.shape}')
        img = torch.from_numpy(np.ascontiguousarray(img)).to(device)
    if not (img.is_cuda and img.dtype == torch.uint8):
        raise _lib.YolactB200Error('val_aug needs a uint8 image on a CUDA device (no CPU fallback)')
    img = img.contiguous()
    h, w = int(img.shape[0]), int(img.shape[1])
    out = torch.empty(3, int(val_size), int(val_size), dtype=torch.float32, device=img.device)
    with torch.cuda.device(img.device):
        _lib.check(_lib.lib().yb_val_aug(img.data_ptr(), h, w, int(val_size), out.data_ptr(),
                                         torch.cuda.current_stream().cuda_stream), 'yb_val_aug')
    return out


VAL_ITEM_DTYPE = np.dtype(_lib.ValAugItem)


def pack_images(images):
    """uint8 BGR images [h,w,3] of any sizes -> (torch uint8 buffer holding them back to back, numpy item table with
    yb_val_aug_item's layout)."""
    items = np.zeros(len(images), dtype=VAL_ITEM_DTYPE)
    buf = np.empty(sum(im.nbytes for im in images), dtype=np.uint8)
    off = 0
    for i, im in enumerate(images):
        if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
            raise ValueError(f'image {i}: expected a uint8 HxWx3 BGR image, got {im.dtype} {im.shape}')
        buf[off:off + im.nbytes] = im.reshape(-1)
        items[i] = (off, im.shape[0], im.shape[1])
        off += im.nbytes
    return torch.from_numpy(buf), items


# ----------------------------------------------------------------------------- JPEG decoding on the device
def jpeg_header(data):
    """(h, w) cv2.imread would return for the JPEG file bytes `data` (orientation applied) when yb_jpeg_decode_batch decodes it,
    None for a file it refuses (progressive, arithmetic, CMYK, 4:1:1, 4:4:0, not a JPEG ...; cv2.imread reads those)."""
    data = np.ascontiguousarray(data, dtype=np.uint8)
    h, w = C.c_int32(), C.c_int32()
    if _lib.lib().yb_jpeg_header(data.ctypes.data, data.size, C.byref(h), C.byref(w)) != 0:
        return None
    return int(h.value), int(w.value)


class EncodedImage:
    """A JPEG file's bytes (numpy uint8) and the (h, w) yb_jpeg_header read from them: what a DataLoader worker returns instead of
    the pixels when the batch is decoded on the device."""

    __slots__ = ('data', 'h', 'w')

    def __init__(self, data, h, w):
        self.data, self.h, self.w = data, int(h), int(w)

    @property
    def shape(self):
        return (self.h, self.w, 3)

    @property
    def nbytes(self):
        return self.h * self.w * 3


def read_image(path, decode_gpu=False):
    """cv2.imread(path); with decode_gpu, the file's bytes as an EncodedImage when yb_jpeg_header accepts them (cv2.imread
    otherwise).  None when cv2 cannot read the file either."""
    if decode_gpu:
        data = np.fromfile(path, np.uint8)
        hw = jpeg_header(data)
        if hw is not None:
            return EncodedImage(data, *hw)
    import cv2
    return cv2.imread(path)


def imdecode_batched(files_host, src_off, items, device='cuda', out=None):
    """Decodes JPEG files on the device: file i is files_host[src_off[i]:src_off[i+1]] (a torch uint8 CPU tensor, page-locked for
    an asynchronous copy) and lands as uint8 BGR [h,w,3] at byte items[i]['img_off'] of the device buffer (yb_val_aug_item
    table; `out`, or a new buffer just large enough).  One H2D copy of the file bytes and one yb_jpeg_decode_batch, no host sync.
    Returns (buffer, status): status a device int32 [n], nonzero where the entropy-coded data is corrupt."""
    device = torch.device(device)
    if device.type != 'cuda':
        raise _lib.YolactB200Error('imdecode_batched runs on a CUDA device (no CPU fallback)')
    if isinstance(files_host, np.ndarray):
        files_host = torch.from_numpy(np.ascontiguousarray(files_host, dtype=np.uint8))
    items = np.ascontiguousarray(items, dtype=VAL_ITEM_DTYPE)
    src_off = np.ascontiguousarray(src_off, dtype=np.int64)
    n = len(items)
    if len(src_off) != n + 1:
        raise ValueError(f'src_off must hold {n + 1} offsets, got {len(src_off)}')
    L = _lib.lib()
    host = files_host.numpy()
    off_p = src_off.ctypes.data_as(C.POINTER(C.c_int64))
    ws_bytes = int(L.yb_jpeg_decode_workspace_bytes(host.ctypes.data, off_p, n))
    if ws_bytes == 0:
        raise _lib.YolactB200Error('imdecode_batched: a file is not a JPEG yb_jpeg_decode_batch decodes (see yb_jpeg_header)')
    need = int(max((int(o) + int(h) * int(w) * 3 for o, h, w in items.tolist()), default=0))
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream()
        src = files_host.to(device, non_blocking=files_host.is_pinned())
        if out is None:
            out = torch.empty(max(need, 1), dtype=torch.uint8, device=device)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        status = torch.empty(n, dtype=torch.int32, device=device)
        _lib.check(L.yb_jpeg_decode_batch(host.ctypes.data, src.data_ptr(), off_p, n, items.ctypes.data_as(C.POINTER(_lib.ValAugItem)),
                                          out.data_ptr(), out.numel(), ws.data_ptr(), ws_bytes, status.data_ptr(), stream.cuda_stream),
                   'yb_jpeg_decode_batch')
    return out, status


def imread_gpu(path, device='cuda'):
    """cv2.imread(path) as a CUDA uint8 tensor [h,w,3]: decoded on the device by yb_jpeg_decode_batch, or by cv2 for a file it
    refuses.  Raises RuntimeError if the file cannot be read or its entropy-coded data is corrupt."""
    img = read_image(path, decode_gpu=True)
    if img is None:
        raise RuntimeError(f'cannot read image {path}')
    if not isinstance(img, EncodedImage):
        return torch.from_numpy(np.ascontiguousarray(img)).to(device)
    items = np.array([(0, img.h, img.w)], VAL_ITEM_DTYPE)
    out, status = imdecode_batched(torch.from_numpy(img.data), [0, img.data.size], items, device)
    if int(status[0]) != 0:
        raise RuntimeError(f'corrupt JPEG data in {path}')
    return out.view(img.h, img.w, 3)


class MixedImages:
    """A batch of images as JPEG file bytes (EncodedImage) and, for the files decoded by cv2, raw uint8 BGR pixels.  `items` is
    the yb_val_aug_item table of the device buffer to_device() fills, in pack_images' layout."""

    def __init__(self, images):
        self.items = np.zeros(len(images), dtype=VAL_ITEM_DTYPE)
        enc = [i for i, im in enumerate(images) if isinstance(im, EncodedImage)]
        raw = [i for i, im in enumerate(images) if not isinstance(im, EncodedImage)]
        off = 0
        for i, im in enumerate(images):
            if not isinstance(im, EncodedImage) and (im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3):
                raise ValueError(f'image {i}: expected a uint8 HxWx3 BGR image, got {im.dtype} {im.shape}')
            self.items[i] = (off, im.shape[0], im.shape[1])
            off += im.nbytes
        self.nbytes = off
        self.encoded = np.array(enc, np.int64)
        self.file_off = np.concatenate([[0], np.cumsum([images[i].data.size for i in enc])]).astype(np.int64)
        self.files = torch.from_numpy(np.concatenate([images[i].data for i in enc]) if enc else np.zeros(1, np.uint8))
        self.raw = [(int(self.items[i]['img_off']), images[i].nbytes) for i in raw]
        self.pixels = torch.from_numpy(np.concatenate([images[i].reshape(-1) for i in raw]) if raw else np.zeros(1, np.uint8))

    def pin_memory(self):
        self.files, self.pixels = self.files.pin_memory(), self.pixels.pin_memory()
        return self

    def to_device(self, device):
        """-> (CUDA uint8 buffer holding every image in `items`' layout, device int32 status of the decoded files (index
        self.encoded[k] for entry k), or None when no file is decoded on the device).  No host sync."""
        device = torch.device(device)
        out = torch.empty(max(self.nbytes, 1), dtype=torch.uint8, device=device)
        status = None
        if len(self.encoded):
            _, status = imdecode_batched(self.files, self.file_off, self.items[self.encoded], device, out=out)
        if self.raw:
            px = self.pixels.to(device, non_blocking=self.pixels.is_pinned())
            o = 0
            for dst, n in self.raw:
                out[dst:dst + n].copy_(px[o:o + n], non_blocking=True)
                o += n
        return out, status


def pack_any(images):
    """pack_images for a batch that may hold EncodedImages: (buffer, items, None) without any, (None, items, MixedImages) with."""
    if any(isinstance(im, EncodedImage) for im in images):
        mixed = MixedImages(images)
        return None, mixed.items, mixed
    buf, items = pack_images(images)
    return buf, items, None


def val_aug_batch(buffer, items, val_size, device='cuda'):
    """val_aug for a batch: `buffer` a torch uint8 tensor holding B BGR HWC images back to back, `items` their numpy table
    (pack_images).  One H2D copy of the buffer (asynchronous when it is pinned), one yb_val_aug_batch launch.
    Returns a CUDA float32 tensor [B, 3, val_size, val_size]."""
    device = torch.device(device)
    if device.type != 'cuda':
        raise _lib.YolactB200Error('val_aug_batch runs on a CUDA device (no CPU fallback)')
    if not (isinstance(buffer, torch.Tensor) and buffer.dtype == torch.uint8 and buffer.dim() == 1):
        raise ValueError('buffer must be a 1-D torch uint8 tensor')
    items = np.ascontiguousarray(items, dtype=VAL_ITEM_DTYPE)
    B, S = len(items), int(val_size)
    L = _lib.lib()
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream()
        src = buffer.to(device, non_blocking=buffer.is_pinned())
        ws_bytes = int(L.yb_val_aug_batch_workspace_bytes(B))
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=device)
        out = torch.empty(B, 3, S, S, dtype=torch.float32, device=device)
        _lib.check(L.yb_val_aug_batch(src.data_ptr(), src.numel(), items.ctypes.data, B, S, ws.data_ptr(), ws_bytes, out.data_ptr(),
                                      stream.cuda_stream), 'yb_val_aug_batch')
    return out


class PackedValBatch:
    """A batch of validation images ready for val_aug_batch, with what MapEvaluator.add needs of their annotations:
      buffer / items   the raw uint8 BGR images back to back and their yb_val_aug_item table (pack_images)
      gt               torch float32 [G,5]: x1,y1,x2,y2 in [0,1] and the class, all images back to back; gt_offset [B+1]
      gt_masks         torch int32: every image's packed gt masks [g_b, h_b, ceil(w_b/32)] back to back; gt_mask_off [B+1] (words)
      sizes, ids       (h, w) and the COCO image id of every image
    It is built in DataLoader workers (utils.coco.val_collate) and holds only picklable types; with DataLoader(pin_memory=True)
    the loader's pin thread calls pin_memory() and the copies to the device are asynchronous.
    Samples of COCOValDetection(..., coco_eval=True) also fill what CocoEvaluator.add needs, every annotation of every image:
      ann_cls int32 [N], ann_box float64 [N,4] (x,y,w,h), ann_area float64 [N], ann_crowd int32 [N]; ann_offset [B+1]
      ann_masks        torch int32: the annotations' packed masks back to back; ann_mask_off [B+1] (words)
    Otherwise these stay None."""

    ann_cls = ann_box = ann_area = ann_crowd = ann_offset = ann_masks = ann_mask_off = None

    mixed = None

    def __init__(self, samples):
        """samples: list of (img_u8 [h,w,3] or EncodedImage, gt float32 [g,5], gt_bits int32 [g,h,ceil(w/32)], (h, w), image
        id[, annotations]).  With EncodedImages `buffer` is None and `mixed` (MixedImages) holds the files; to_device decodes them."""
        self.buffer, self.items, self.mixed = pack_any([s[0] for s in samples])
        self.sizes = [(int(s[3][0]), int(s[3][1])) for s in samples]
        self.ids = [s[4] for s in samples]
        for i, (img, gt, bits, (h, w), _) in enumerate(s[:5] for s in samples):
            if img.shape[:2] != (h, w) or gt.dtype != np.float32 or gt.ndim != 2 or gt.shape[1] != 5 or bits.dtype != np.int32 or \
                    bits.shape != (gt.shape[0], h, (w + 31) // 32):
                raise ValueError(f'sample {i}: image {img.shape}, gt {gt.dtype} {gt.shape} and gt masks {bits.dtype} {bits.shape} do not '
                                 f'describe one {h}x{w} image')
        self.gt_offset = np.concatenate([[0], np.cumsum([s[1].shape[0] for s in samples])]).astype(int).tolist()
        self.gt_mask_off = np.concatenate([[0], np.cumsum([s[2].size for s in samples])]).astype(int).tolist()
        self.gt = torch.from_numpy(np.concatenate([s[1] for s in samples]).reshape(-1, 5))
        self.gt_masks = torch.from_numpy(np.concatenate([s[2].reshape(-1) for s in samples]))
        if samples and all(len(s) > 5 for s in samples):
            self._pack_annotations([s[5] for s in samples])

    def _pack_annotations(self, anns):
        for i, ((cls, box, area, crowd, bits), (h, w)) in enumerate(zip(anns, self.sizes)):
            m = len(cls)
            if cls.dtype != np.int32 or box.dtype != np.float64 or box.shape != (m, 4) or area.dtype != np.float64 or \
                    area.shape != (m,) or crowd.dtype != np.int32 or crowd.shape != (m,) or bits.dtype != np.int32 or \
                    bits.shape != (m, h, (w + 31) // 32):
                raise ValueError(f'sample {i}: annotation tables {cls.shape} {box.shape} {area.shape} {crowd.shape} {bits.shape} do not '
                                 f'describe {m} annotations of one {h}x{w} image')
        self.ann_offset = np.concatenate([[0], np.cumsum([len(a[0]) for a in anns])]).astype(int).tolist()
        self.ann_mask_off = np.concatenate([[0], np.cumsum([a[4].size for a in anns])]).astype(int).tolist()
        self.ann_cls, self.ann_box, self.ann_area, self.ann_crowd, self.ann_masks = (
            torch.from_numpy(np.concatenate([a[j].reshape((-1, 4) if j == 1 else -1) for a in anns])) for j in range(5))

    def __len__(self):
        return len(self.items)

    def pin_memory(self):
        """Called by DataLoader(pin_memory=True) in its pin thread: page-locks the images, the gts and the gt masks (and the
        annotation tables when there are any)."""
        if self.mixed is not None:
            self.mixed.pin_memory()
        else:
            self.buffer = self.buffer.pin_memory()
        self.gt, self.gt_masks = self.gt.pin_memory(), self.gt_masks.pin_memory()
        if self.ann_cls is not None:
            self.ann_cls, self.ann_box, self.ann_area, self.ann_crowd, self.ann_masks = (
                t.pin_memory() for t in (self.ann_cls, self.ann_box, self.ann_area, self.ann_crowd, self.ann_masks))
        return self

    def to_device(self, device):
        """-> (CUDA uint8 buffer of the images in `items`' layout, device int32 status of the files decoded there or None); the
        files are decoded by yb_jpeg_decode_batch, no host sync."""
        if self.mixed is not None:
            return self.mixed.to_device(device)
        return self.buffer.to(device, non_blocking=self.buffer.is_pinned()), None

    def gt_to(self, device):
        """-> (gt [G,5], list of B packed gt masks [g_b, h_b, ceil(w_b/32)]) on `device`: views of one copy of each buffer."""
        gt = self.gt.to(device, non_blocking=self.gt.is_pinned())
        words = self.gt_masks.to(device, non_blocking=self.gt_masks.is_pinned())
        o, g = self.gt_mask_off, self.gt_offset
        masks = [words[o[b]:o[b + 1]].view(g[b + 1] - g[b], h, (w + 31) // 32) for b, (h, w) in enumerate(self.sizes)]
        return gt, masks


# ----------------------------------------------------------------------------- train_aug: host planner
@dataclass
class TrainAugPlan:
    """What train_aug does to one image, minus the pixels.  Coordinates follow the reference's stages:
    `crop` = (x, y, w, h) in the mirrored image, `pad` = (x, y) offset of the crop in the `square`,
    `train_off` = (x, y) pad offset (resize < train_size) or crop offset (resize > train_size)."""
    h: int
    w: int
    brightness: object          # float delta, or None when the draw skipped it
    contrast: object            # float alpha, or None
    saturation: float
    hue: float
    mirror: bool
    crop: tuple
    square: int
    pad: tuple
    resize: int
    train_size: int
    train_off: tuple
    mask_u8: bool               # the masks stay uint8 through the resize (no pad to square happened)
    keep: np.ndarray            # int64 indices of the source masks that survive, in output order
    boxes: np.ndarray           # float64 [n,4] in [0,1]
    labels: np.ndarray          # float64 [n]


def _crop_window(ori_h, crop_h, ori_w, crop_w, boxes, keep_ratio=0.3):
    """utils/augmentations.py:80-124 `crop` without pixels: up to 1000 tries of (x, then y); a box is kept when
    its intersection with the window covers more than keep_ratio of its area.  The window corners are float32 in
    the reference and the boxes float64, so the test runs in float64 (a zero-area box gives NaN and never passes).
    Returns (x1, y1, keep mask, kept intersection boxes relative to the window) or None."""
    area = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1])
    for _ in range(1000):
        x1 = random.randint(0, ori_w - crop_w)
        y1 = random.randint(0, ori_h - crop_h)
        lo_x = np.maximum(np.float64(np.float32(x1)), boxes[:, 0])
        lo_y = np.maximum(np.float64(np.float32(y1)), boxes[:, 1])
        hi_x = np.minimum(np.float64(np.float32(x1 + crop_w)), boxes[:, 2])
        hi_y = np.minimum(np.float64(np.float32(y1 + crop_h)), boxes[:, 3])
        inter = np.clip(hi_x - lo_x, 0, 10000) * np.clip(hi_y - lo_y, 0, 10000)
        with np.errstate(divide='ignore', invalid='ignore'):
            keep = inter / area > keep_ratio
        if keep.any():
            kept = np.stack([lo_x, lo_y, hi_x, hi_y], axis=1)[keep]
            kept[:, [0, 2]] -= x1
            kept[:, [1, 3]] -= y1
            return x1, y1, keep, kept
    return None


def train_aug_plan(h, w, boxes, labels, train_size):
    """Draw one image's train_aug plan (utils/augmentations.py:230-252) from Python's `random`, in the reference's
    order.  boxes: [n,4] x1y1x2y2 pixels (float64), labels: [n].  Returns a TrainAugPlan, or None where the
    reference returns (None,)*4 (the crop found no window in 1000 tries, or no box survived)."""
    h, w, S = int(h), int(w), int(train_size)
    boxes = np.array(boxes, dtype=np.float64).reshape(-1, 4)
    labels = np.asarray(labels).astype(np.float64).reshape(-1)
    idx = np.arange(boxes.shape[0])
    # photometric_distort (:62-77): brightness and contrast each behind a coin, then saturation and hue
    brightness = random.uniform(-32, 32) if random.randint(0, 1) else None
    contrast = random.uniform(0.7, 1.3) if random.randint(0, 1) else None
    saturation = random.uniform(0.7, 1.3)
    hue = random.uniform(-15., 15.)
    # random_mirror (:10-17)
    mirror = bool(random.randint(0, 1))
    if mirror:
        boxes[:, [0, 2]] = w - boxes[:, [2, 0]]
    # random_crop (:127-135): a coin of 1 leaves the image whole
    crop = (0, 0, w, h)
    if not random.randint(0, 1):
        crop_h = int(random.uniform(0.6, 1) * h)
        crop_w = int(random.uniform(0.6, 1) * w)
        r = _crop_window(h, crop_h, w, crop_w, boxes)
        if r is None:
            return None
        x1, y1, keep, boxes = r
        idx, labels = idx[keep], labels[keep]
        crop = (x1, y1, crop_w, crop_h)
    # pad_to_square (:138-165): a random offset along the short side; a square crop is left alone (masks stay uint8)
    cw, ch = crop[2], crop[3]
    square, pad = max(cw, ch), (0, 0)
    if ch < cw:
        pad = (0, random.randint(0, cw - ch))
        boxes[:, [1, 3]] += pad[1]
    elif ch > cw:
        pad = (random.randint(0, ch - cw), 0)
        boxes[:, [0, 2]] += pad[0]
    # multi_scale_resize (:168-189)
    resize = random.randint(8, 24) * 32
    boxes *= resize / square
    # to_train_size (:192-209): pad (y, then x) or crop (the crop loop again, x then y)
    train_off = (0, 0)
    if resize < S:
        ty = random.randint(0, S - resize)
        tx = random.randint(0, S - resize)
        boxes[:, [1, 3]] += ty
        boxes[:, [0, 2]] += tx
        train_off = (tx, ty)
    elif resize > S:
        r = _crop_window(resize, S, resize, S, boxes)
        if r is None:
            return None
        tx, ty, keep, boxes = r
        idx, labels = idx[keep], labels[keep]
        train_off = (tx, ty)
    # clip_box, remove_small_box (area > 20), to_01_box (:20-35)
    boxes[:, [0, 2]] = np.clip(boxes[:, [0, 2]], 0, S - 1)
    boxes[:, [1, 3]] = np.clip(boxes[:, [1, 3]], 0, S - 1)
    big = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1]) > 20
    boxes, labels, idx = boxes[big], labels[big], idx[big]
    if boxes.shape[0] == 0:
        return None
    boxes[:, [0, 2]] /= S
    boxes[:, [1, 3]] /= S
    return TrainAugPlan(h=h, w=w, brightness=brightness, contrast=contrast, saturation=saturation, hue=hue, mirror=mirror,
                        crop=tuple(int(v) for v in crop), square=square, pad=pad, resize=resize, train_size=S, train_off=train_off,
                        mask_u8=(cw == ch), keep=idx.astype(np.int64), boxes=boxes, labels=labels)


# ----------------------------------------------------------------------------- train_aug: batch packing + GPU executor
class PackedTrainBatch:
    """A batch ready for yb_train_aug: one contiguous uint8 buffer (each image [h,w,3] BGR then its masks [n,h,w]),
    the item table, the `keep` table and the targets ([n_i,5] float32: boxes in [0,1] then the label).

    It is built in DataLoader workers and sent to the main process, so it holds only picklable types: the buffer is a
    torch uint8 tensor (it travels through shared memory), the item table a numpy array with yb_train_aug_item's
    layout, `keep` an int32 numpy array.  With DataLoader(pin_memory=True) the loader's pin thread calls pin_memory()
    and train_aug_batch copies the buffer to the device asynchronously."""

    ITEM_DTYPE = np.dtype(_lib.TrainAugItem)

    def __init__(self, samples):
        """samples: list of (img_u8 [h,w,3], masks_u8 [n,h,w], TrainAugPlan)."""
        sizes = [s[0].nbytes + s[1].nbytes for s in samples]
        buf = np.empty(sum(sizes), dtype=np.uint8)
        self.items = np.zeros(len(samples), dtype=self.ITEM_DTYPE)
        keeps, self.targets, self.num_keep = [], [], []
        off = rows = 0
        for i, ((img, masks, plan), size) in enumerate(zip(samples, sizes)):
            h, w = img.shape[:2]
            if img.dtype != np.uint8 or img.shape != (plan.h, plan.w, 3) or masks.dtype != np.uint8 or masks.shape[1:] != (h, w):
                raise ValueError(f'sample {i}: expected uint8 image [{plan.h},{plan.w},3] and uint8 masks [n,{plan.h},{plan.w}], '
                                 f'got {img.dtype} {img.shape} and {masks.dtype} {masks.shape}')
            buf[off:off + img.nbytes] = img.reshape(-1)
            buf[off + img.nbytes:off + size] = masks.reshape(-1)
            fields = dict(img_off=off, mask_off=off + img.nbytes, h=h, w=w, num_masks=masks.shape[0],
                          brightness_on=plan.brightness is not None, brightness_delta=np.float32(plan.brightness or 0.0),
                          contrast_on=plan.contrast is not None, contrast_alpha=np.float32(plan.contrast or 1.0),
                          saturation_scale=np.float32(plan.saturation), hue_delta=np.float32(plan.hue), mirror=plan.mirror,
                          crop_x=plan.crop[0], crop_y=plan.crop[1], crop_w=plan.crop[2], crop_h=plan.crop[3], square=plan.square,
                          pad_x=plan.pad[0], pad_y=plan.pad[1], resize=plan.resize, train_x=plan.train_off[0],
                          train_y=plan.train_off[1], mask_u8=plan.mask_u8, out_mask=rows, keep_begin=rows, num_keep=len(plan.keep))
            for k, v in fields.items():
                self.items[k][i] = v
            keeps.append(plan.keep)
            self.targets.append(torch.from_numpy(np.hstack((plan.boxes, plan.labels[:, None])).astype(np.float32)))
            self.num_keep.append(len(plan.keep))
            off += size
            rows += len(plan.keep)
        self.buffer = torch.from_numpy(buf)
        self.keep = np.ascontiguousarray(np.concatenate(keeps).astype(np.int32))
        self.train_size = samples[0][2].train_size
        if any(s[2].train_size != self.train_size for s in samples):
            raise ValueError('every plan of a batch must have the same train_size')

    def __len__(self):
        return len(self.items)

    def pin_memory(self):
        """Called by DataLoader(pin_memory=True) in its pin thread: page-locks the buffer and the targets."""
        self.buffer = self.buffer.pin_memory()
        self.targets = [t.pin_memory() for t in self.targets]
        return self

    def items_ptr(self):
        return self.items.ctypes.data_as(C.POINTER(_lib.TrainAugItem))

    def keep_ptr(self):
        return self.keep.ctypes.data_as(C.c_void_p)


def train_aug_batch(packed, train_size, device='cuda'):
    """Apply a packed batch of plans on the GPU: one H2D copy of the uint8 buffer (asynchronous when the batch was
    pinned by the DataLoader; no extra host copy is made here), one yb_train_aug launch.
    Returns (images [B,3,S,S], targets: list of [n_i,5], masks: list of [n_i,S,S]), CUDA float32, the inputs
    Yolact.forward(img, targets, masks) takes in train mode."""
    S = int(train_size)
    if S != packed.train_size:
        raise ValueError(f'the plans were drawn for train_size {packed.train_size}, not {S}')
    device = torch.device(device)
    if device.type != 'cuda':
        raise _lib.YolactB200Error('train_aug_batch runs on a CUDA device (no CPU fallback)')
    B, G = len(packed), int(packed.keep.shape[0])
    L = _lib.lib()
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream()
        src = packed.buffer.to(device, non_blocking=packed.buffer.is_pinned())
        ws_bytes = int(L.yb_train_aug_workspace_bytes(B, G))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        images = torch.empty(B, 3, S, S, dtype=torch.float32, device=device)
        masks = torch.empty(G, S, S, dtype=torch.float32, device=device)
        _lib.check(L.yb_train_aug(src.data_ptr(), src.numel(), packed.items_ptr(), B, packed.keep_ptr(), S,
                                  ws.data_ptr(), ws_bytes, images.data_ptr(), masks.data_ptr() if G else None, stream.cuda_stream),
                   'yb_train_aug')
        targets = [t.to(device, non_blocking=t.is_pinned()) for t in packed.targets]
    return images, targets, list(masks.split(packed.num_keep, 0))


class TrainAugLoader:
    """Wraps a DataLoader whose collate is utils.coco.train_collate and yields what the reference's train loop
    feeds the network (train.py:112-117), augmented on `device`:

        for images, targets, masks in TrainAugLoader(data_loader, cfg.img_size):
            loss_c, loss_b, loss_m, loss_s = net(images, targets, masks)
    """

    def __init__(self, loader, train_size, device=None):
        self.loader, self.train_size = loader, int(train_size)
        self.device = device if device is not None else torch.device('cuda', torch.cuda.current_device())

    def __len__(self):
        return len(self.loader)

    def __iter__(self):
        for packed in self.loader:
            yield train_aug_batch(packed, self.train_size, self.device)
