"""Mask output stage on the GPU (SURVEY.md 8(f) rank 2): bit-packed masks, pairwise mask IoU and COCO run-length encoding -- the
work the reference's evaluation loop does on 100 x H x W float32 masks per image (utils/common_utils.py:88-96,:174-183,
utils/box_utils.py:189-200) -- behind yb_pack_mask_bits / yb_mask_iou_bits / yb_mask_rle (include/yolact_b200.h).

    bits = after_nms(..., mask_dtype='bits')[3]          # [d, h, ceil(w/32)] uint32, 1 bit / pixel
    iou  = mask_iou_bits(bits_pred, bits_gt)             # [d, g] float32 on the device
    rles = encode_rle(bits, h, w)                        # [{'size': [h, w], 'counts': '...'}]  == pycocotools.mask.encode(...)

CUDA tensors only; nothing falls back to the CPU (the ASCII compression of the run lengths is host work by definition: it
produces a Python string per mask)."""
import numpy as np
import torch

from .. import _lib


def _cuda(t, what):
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise _lib.YolactB200Error(f'{what} needs CUDA tensors (no CPU fallback)')


def pack_masks(masks):
    """{0,1} masks [n,h,w] (uint8 / bool / float32, CUDA) -> packed uint32 words [n,h,ceil(w/32)] (stored as int32)."""
    _cuda(masks, 'pack_masks')
    if masks.dtype == torch.bool:
        masks = masks.to(torch.uint8)
    if masks.dtype not in (torch.uint8, torch.float32):
        masks = masks.to(torch.float32)
    m = masks.contiguous()
    n, h, w = m.shape
    out = torch.empty(n, h, (w + 31) // 32, dtype=torch.int32, device=m.device)
    with torch.cuda.device(m.device):
        _lib.check(_lib.lib().yb_pack_mask_bits(m.data_ptr(), 1 if m.dtype == torch.float32 else 0, n, h, w, out.data_ptr(),
                                                torch.cuda.current_stream().cuda_stream), 'yb_pack_mask_bits')
    return out


def pack_masks_host(masks):
    """pack_masks on the host: {0,1} masks [n,h,w] (numpy) -> numpy int32 words [n,h,ceil(w/32)] in the same layout
    (np.packbits with little bit order over rows padded to 32 pixels; 8x less to pickle and copy than the uint8 masks)."""
    m = np.asarray(masks)
    n, h, w = m.shape
    rows = np.zeros((n, h, (w + 31) // 32 * 32), np.uint8)
    rows[..., :w] = m
    return np.ascontiguousarray(np.packbits(rows, axis=-1, bitorder='little')).view('<i4')


def unpack_masks(bits, w):
    """Packed words [n,h,words] -> uint8 masks [n,h,w] (plain torch bit arithmetic; for tests and visualisation)."""
    n, h, words = bits.shape
    b = bits.to(torch.int64) & 0xffffffff
    sh = torch.arange(32, device=bits.device, dtype=torch.int64)
    return ((b[..., None] >> sh) & 1).reshape(n, h, words * 32)[..., :w].to(torch.uint8)


def mask_iou_bits(a, b):
    """Pairwise IoU of two sets of packed masks with equal geometry: [n,...] x [m,...] -> float32 [n,m] on the device
    (0/0 = NaN, like the reference's float division)."""
    _cuda(a, 'mask_iou_bits'); _cuda(b, 'mask_iou_bits')
    a, b = a.contiguous(), b.contiguous()
    n, m = a.shape[0], b.shape[0]
    words = a[0].numel() if n else (b[0].numel() if m else 1)
    if n and m and a[0].numel() != b[0].numel():
        raise ValueError(f'mask geometries differ: {tuple(a.shape)} vs {tuple(b.shape)}')
    out = torch.empty(n, m, dtype=torch.float32, device=a.device)
    with torch.cuda.device(a.device):
        _lib.check(_lib.lib().yb_mask_iou_bits(a.data_ptr(), n, b.data_ptr(), m, words, out.data_ptr(), torch.cuda.current_stream().cuda_stream),
                   'yb_mask_iou_bits')
    return out


def rle_counts(bits, h, w, max_runs=4096):
    """Run lengths of every packed mask in COCO order (column-major, first run = zeros).  Returns a list of numpy uint32 arrays."""
    _cuda(bits, 'rle_counts')
    bits = bits.contiguous()
    n = bits.shape[0]
    L = _lib.lib()
    while True:
        counts = torch.empty(n, max_runs, dtype=torch.int32, device=bits.device)
        nruns = torch.empty(n, dtype=torch.int32, device=bits.device)
        with torch.cuda.device(bits.device):
            _lib.check(L.yb_mask_rle(bits.data_ptr(), n, h, w, counts.data_ptr(), max_runs, nruns.data_ptr(), torch.cuda.current_stream().cuda_stream),
                       'yb_mask_rle')
        nr = nruns.cpu().numpy()
        if n == 0 or nr.min() >= 0:
            break
        max_runs = int(-nr.min())                                  # a mask needed more runs than the buffer holds: retry once, exactly sized
    c = counts.cpu().numpy().view(np.uint32)
    return [c[i, :nr[i]].copy() for i in range(n)]


def rle_counts_to_string(counts):
    """pycocotools' rleToString: counts[i] (difference to counts[i-2] for i > 2) in 5-bit groups with a continuation bit, + 48."""
    out = []
    c = [int(v) for v in counts]
    for i, x in enumerate(c):
        if i > 2:
            x -= c[i - 2]
        more = True
        while more:
            ch = x & 0x1f
            x >>= 5                                                # arithmetic shift: Python ints behave like the C long here
            more = (x != -1) if (ch & 0x10) else (x != 0)
            if more:
                ch |= 0x20
            out.append(chr(ch + 48))
    return ''.join(out)


def rle_string_to_counts(s):
    """Inverse of rle_counts_to_string (pycocotools' rleFrString)."""
    counts, p, m = [], 0, 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            ch = ord(s[p]) - 48
            x |= (ch & 0x1f) << (5 * k)
            more = bool(ch & 0x20)
            p += 1; k += 1
            if not more and (ch & 0x10):
                x |= -1 << (5 * k)
        if m > 2:
            x += counts[m - 2]
        counts.append(x); m += 1
    return counts


def encode_rle(bits, h, w):
    """Packed masks -> [{'size': [h, w], 'counts': str}] -- the objects pycocotools.mask.encode(np.asfortranarray(mask)) returns
    (with counts already decoded to str, as utils/common_utils.py:91 does for json.dump)."""
    return [{'size': [int(h), int(w)], 'counts': rle_counts_to_string(c)} for c in rle_counts(bits, h, w)]
