"""GPU: yb_jpeg_encode_batch writes the file cv2.imencode('.jpg') writes, byte for byte.
  * one call over the whole corpus (tests/jpeg_corpus.py), images packed back to back with sentinel gaps: each file equals the
    oracle (oracle/jpeg_np.py), the golden (tests/golden/jpeg.npz) and cv2 on this host; no byte past out_len[i] changes;
  * bad offsets, sizes and qualities are refused before anything is launched;
  * a call is five launches and never synchronises (set_sync_debug_mode('error'));
  * imencode_gpu equals cv2.imencode on one image."""
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch

import jpeg_corpus
from oracle import jpeg_np

pytestmark = pytest.mark.gpu

SENT = 0xA5
GAP = 13


@pytest.fixture(scope='module')
def golden():
    with np.load(os.path.join(jpeg_corpus.GOLDEN_DIR, 'jpeg.npz')) as z:
        return {k: z[k] for k in z.files}


def _pack(images, gap=GAP):
    from yolact_minimal_b200 import _lib
    items = np.zeros(len(images), np.dtype(_lib.ValAugItem))
    src = np.full(sum(im.nbytes + gap for im in images) + gap, SENT, np.uint8)
    o = gap
    for i, im in enumerate(images):
        items[i] = (o, *im.shape[:2])
        src[o:o + im.nbytes] = im.reshape(-1)
        o += im.nbytes + gap
    return src, items


def _encode(dev, src, items, q, out_off, out_bytes, ws_extra=0):
    from yolact_minimal_b200 import _lib
    L = _lib.lib()
    ip = items.ctypes.data_as(ctypes.POINTER(_lib.ValAugItem))
    ws_bytes = int(L.yb_jpeg_encode_workspace_bytes(ip, len(items)))
    ws = torch.empty(ws_bytes + ws_extra, dtype=torch.uint8, device=dev)
    src_d = torch.from_numpy(src).to(dev)
    out = torch.full((out_bytes,), SENT, dtype=torch.uint8, device=dev)
    out_len = torch.full((len(items),), -1, dtype=torch.int64, device=dev)
    before = _lib.launch_count()
    status = L.yb_jpeg_encode_batch(src_d.data_ptr(), src_d.numel(), ip, len(items), q, ws.data_ptr(), ws_bytes, out.data_ptr(),
                                    out_off.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), out_len.data_ptr(),
                                    torch.cuda.current_stream().cuda_stream)
    return status, out, out_len, _lib.launch_count() - before


def _offsets(items, gap=GAP):
    from yolact_minimal_b200.utils.output_utils import jpeg_bound
    off = np.zeros(len(items) + 1, np.int64)
    o = gap
    for i, (h, w) in enumerate(zip(items['h'], items['w'])):
        off[i] = o
        o += jpeg_bound(h, w) + gap
    off[-1] = o - gap
    return off, o


@pytest.mark.parametrize('q', jpeg_corpus.QUALITIES)
def test_batch_equals_golden_oracle_and_cv2(cuda, q, golden):
    import cv2
    cases = jpeg_corpus.corpus()
    src, items = _pack([img for _, img in cases])
    out_off, total = _offsets(items)
    status, out, out_len, launches = _encode(cuda, src, items, q, out_off, total)
    assert status == 0
    assert launches == 5
    got, lens = out.cpu().numpy(), out_len.cpu().numpy()
    touched = np.zeros(total, bool)
    for i, (name, img) in enumerate(cases):
        data = got[out_off[i]:out_off[i] + lens[i]].tobytes()
        key = f'{name}@{q}'
        assert hashlib.sha256(data).digest() == golden[f'sha256/{key}'].tobytes(), key
        assert data == cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes(), key
        if img.shape[0] * img.shape[1] <= 128 * 128 or name.startswith('photo'):
            assert data == jpeg_np.encode(img, q), key
        touched[out_off[i]:out_off[i] + lens[i]] = True
    assert np.all(got[~touched] == SENT), 'a byte outside the written files changed'


def test_refused_before_launch(cuda):
    from yolact_minimal_b200 import _lib
    img = jpeg_corpus.synth(37, 53, 'noise')
    src, items = _pack([img, img])
    out_off, total = _offsets(items)
    L = _lib.lib()

    def call(items=items, q=95, off=out_off, src_bytes=len(src)):
        ip = items.ctypes.data_as(ctypes.POINTER(_lib.ValAugItem))
        ws = torch.empty(1 << 20, dtype=torch.uint8, device=cuda)
        out = torch.empty(total, dtype=torch.uint8, device=cuda)
        ln = torch.empty(2, dtype=torch.int64, device=cuda)
        before = _lib.launch_count()
        s = L.yb_jpeg_encode_batch(ws.data_ptr(), src_bytes, ip, len(items), q, ws.data_ptr() + (1 << 19), 1 << 19, out.data_ptr(),
                                   off.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), ln.data_ptr(), None)
        return s, _lib.launch_count() - before

    for q in (0, 101, -5):
        assert call(q=q) == (-1, 0)
    bad = items.copy()
    bad[1]['h'] = 0
    assert call(items=bad) == (-1, 0)
    bad = items.copy()
    bad[0]['w'] = 70000
    assert call(items=bad) == (-1, 0)
    bad = items.copy()
    bad[1]['img_off'] = len(src) - 10
    assert call(items=bad) == (-1, 0)
    off = out_off.copy()
    off[1] = off[0] + 100                        # image 0's bound does not fit
    assert call(off=off) == (-1, 0)
    off = out_off.copy()
    off[0] = -1
    assert call(off=off) == (-1, 0)
    off = out_off.copy()
    off[2] -= 1
    assert call(off=off) == (-1, 0)
    assert call(src_bytes=len(src) - GAP - 1) == (-1, 0)
    assert L.yb_jpeg_encode_bound(0, 5) == -1 and L.yb_jpeg_encode_bound(65536, 5) == -1
    ip = items.ctypes.data_as(ctypes.POINTER(_lib.ValAugItem))
    ws_bytes = int(L.yb_jpeg_encode_workspace_bytes(ip, 2))
    status, _, _, launches = _encode(cuda, src, items, 95, out_off, total, ws_extra=0)
    assert status == 0 and launches == 5
    # a workspace one byte short is refused
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=cuda)
    out = torch.empty(total, dtype=torch.uint8, device=cuda)
    ln = torch.empty(2, dtype=torch.int64, device=cuda)
    src_d = torch.from_numpy(src).to(cuda)
    assert L.yb_jpeg_encode_batch(src_d.data_ptr(), len(src), ip, 2, 95, ws.data_ptr(), ws_bytes - 1, out.data_ptr(),
                                  out_off.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), ln.data_ptr(), None) == -1


def test_queues_without_sync(cuda):
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils.output_utils import imencode_batched
    imgs = [jpeg_corpus.synth(h, w, 'noise', seed=3) for h, w in ((480, 640), (1, 1), (37, 53))]
    src, items = _pack(imgs, gap=0)
    buf = torch.from_numpy(src).to(cuda)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for _ in range(3):
            data, off, lens = imencode_batched(buf, items, 95)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert _lib.launch_count() - before == 15
    lens = lens.cpu().numpy()
    got = data.cpu().numpy()
    for i, img in enumerate(imgs):
        assert got[off[i]:off[i] + lens[i]].tobytes() == jpeg_np.encode(img, 95)


@pytest.mark.parametrize('q', [95, 75, 1])
def test_imencode_gpu_equals_cv2(cuda, q):
    import cv2
    from yolact_minimal_b200.utils.output_utils import imencode_gpu
    for name, img in jpeg_corpus.photos():
        want = cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, q])[1]
        got = imencode_gpu(img, q)
        assert got.dtype == want.dtype and got.shape == want.shape and np.array_equal(got, want), name
        got_t = imencode_gpu(torch.from_numpy(img).to(cuda), q)
        assert np.array_equal(got_t, want), name
