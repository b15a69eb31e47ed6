"""GPU: yb_jpeg_decode_batch returns the pixels cv2.imread returns, bit for bit.
  * the whole corpus (tests/jpeg_decode_corpus.py: layouts, restart intervals, qualities, sizes, orientations) in batches of 64, 7
    and 1 mixing all of them, each image placed in an output slot with sentinel gaps: every image equals cv2.imread and the golden
    (tests/golden/jpeg_decode.npz), the small ones the oracle (oracle/jpeg_decode_np.py), and no byte outside the slots changes;
  * batches that mix decoded files with files the header refuses (read by cv2, copied into their slots on the device);
  * one call queues without a host synchronisation (set_sync_debug_mode('error')) in five launches;
  * corrupt entropy-coded data (a file cut mid-scan, flipped scan bytes, a missing restart marker) gives a nonzero status,
    leaves the sentinels and every other image of the batch intact."""
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch

import jpeg_corpus
import jpeg_decode_corpus
from oracle import jpeg_decode_np

pytestmark = pytest.mark.gpu

SENT = 0x5A
GAP = 11


@pytest.fixture(scope='module')
def golden():
    with np.load(os.path.join(jpeg_corpus.GOLDEN_DIR, 'jpeg_decode.npz')) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope='module')
def corpus():
    return jpeg_decode_corpus.corpus()


def _decode(dev, files, gap=GAP):
    """One yb_jpeg_decode_batch over `files` into slots separated by sentinel gaps -> (status, out numpy, items, launches)."""
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils.augmentations import VAL_ITEM_DTYPE, jpeg_header
    L = _lib.lib()
    src = np.concatenate([np.frombuffer(f, np.uint8) for f in files])
    src_off = np.concatenate([[0], np.cumsum([len(f) for f in files])]).astype(np.int64)
    items = np.zeros(len(files), VAL_ITEM_DTYPE)
    o = gap
    for i, f in enumerate(files):
        h, w = jpeg_header(np.frombuffer(f, np.uint8))
        items[i] = (o, h, w)
        o += h * w * 3 + gap
    off_p = src_off.ctypes.data_as(ctypes.POINTER(ctypes.c_int64))
    ws_bytes = int(L.yb_jpeg_decode_workspace_bytes(src.ctypes.data, off_p, len(files)))
    assert ws_bytes > 0
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    src_d = torch.from_numpy(src).to(dev)
    out = torch.full((o,), SENT, dtype=torch.uint8, device=dev)
    status = torch.full((len(files),), -1, dtype=torch.int32, device=dev)
    before = _lib.launch_count()
    s = L.yb_jpeg_decode_batch(src.ctypes.data, src_d.data_ptr(), off_p, len(files), items.ctypes.data_as(ctypes.POINTER(_lib.ValAugItem)),
                               out.data_ptr(), out.numel(), ws.data_ptr(), ws_bytes, status.data_ptr(),
                               torch.cuda.current_stream().cuda_stream)
    launches = _lib.launch_count() - before
    rounds = ws[:4 * len(files)].view(torch.int32).cpu().numpy()
    return s, out.cpu().numpy(), items, status.cpu().numpy(), launches, rounds


def _slot(out, item):
    off, h, w = (int(v) for v in item)
    return out[off:off + h * w * 3].reshape(h, w, 3)


def _check_sentinels(out, items):
    touched = np.zeros(len(out), bool)
    for off, h, w in items.tolist():
        touched[off:off + h * w * 3] = True
    assert np.all(out[~touched] == SENT), 'a byte outside the output slots changed'


@pytest.mark.parametrize('B', [64, 7, 1])
def test_corpus_equals_cv2_golden_and_oracle(cuda, corpus, golden, tmp_path, B):
    rng = np.random.default_rng(B)
    order = rng.permutation(len(corpus))
    for a in range(0, len(order), B):
        batch = [corpus[k] for k in order[a:a + B]]
        s, out, items, status, launches, rounds = _decode(cuda, [d for _, d in batch])
        assert s == 0 and launches == 5
        assert np.all(status == 0), [batch[k][0] for k in np.flatnonzero(status)]
        assert np.all(rounds >= 1)
        _check_sentinels(out, items)
        for i, (name, data) in enumerate(batch):
            got = _slot(out, items[i])
            assert hashlib.sha256(got.tobytes()).digest() == golden[f'pixels_sha256/{name}'].tobytes(), name
            assert np.array_equal(got, jpeg_decode_corpus.cv2_decode(data, tmp_path)), name
            if got.size <= 64 * 64 * 3:
                assert np.array_equal(got, jpeg_decode_np.decode(data)), name


def test_mixed_with_fallback_files(cuda, corpus, tmp_path):
    """MixedImages: decoded files and cv2-read pixels in one device buffer in pack_images' layout."""
    from yolact_minimal_b200.utils.augmentations import MixedImages, read_image
    files = [corpus[3][1], jpeg_decode_corpus.refused()[0][1], corpus[40][1], jpeg_decode_corpus.refused()[1][1], corpus[-1][1]]
    images, want = [], []
    for i, data in enumerate(files):
        p = tmp_path / f'{i}.jpg'
        p.write_bytes(data)
        images.append(read_image(str(p), decode_gpu=True))
        want.append(jpeg_decode_corpus.cv2_decode(data, tmp_path))
    m = MixedImages(images).pin_memory()
    assert m.encoded.tolist() == [0, 2, 4]
    buf, status = m.to_device(cuda)
    got = buf.cpu().numpy()
    assert status.cpu().numpy().tolist() == [0, 0, 0]
    for i, w in enumerate(want):
        assert np.array_equal(_slot(got, m.items[i]), w), i


def test_queues_without_sync(cuda, corpus):
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils.augmentations import VAL_ITEM_DTYPE, imdecode_batched, jpeg_header
    files = [d for _, d in corpus[:12]]
    src = torch.from_numpy(np.concatenate([np.frombuffer(f, np.uint8) for f in files])).pin_memory()
    src_off = np.concatenate([[0], np.cumsum([len(f) for f in files])])
    items = np.zeros(len(files), VAL_ITEM_DTYPE)
    o = 0
    for i, f in enumerate(files):
        h, w = jpeg_header(np.frombuffer(f, np.uint8))
        items[i] = (o, h, w)
        o += h * w * 3
    torch.cuda.synchronize()
    before = _lib.launch_count()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for _ in range(3):
            out, status = imdecode_batched(src, src_off, items, cuda)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert _lib.launch_count() - before == 15
    got = out.cpu().numpy()
    assert np.all(status.cpu().numpy() == 0)
    for i, f in enumerate(files):
        assert np.array_equal(_slot(got, items[i]), jpeg_decode_np.decode(f))


def _corrupt_files():
    img = jpeg_corpus.synth(45, 70, 'noise', seed=9)
    base = jpeg_decode_corpus.encode(img, 95, '420')
    sos = base.index(b'\xff\xda')
    cut = base[:sos + (len(base) - sos) // 2]                           # ends mid-scan, no EOI
    k = next(k for k in range(sos + 60, len(base)) if 0xFF not in base[k - 1:k + 41])
    flipped = base[:k] + b'\xff\x00' * 20 + base[k + 40:]                # 40 scan bytes overwritten by 160 one-bits
    rst = jpeg_decode_corpus.encode(img, 95, '420', rst=1)
    k = rst.index(b'\xff\xd3', rst.index(b'\xff\xda'))
    missing = rst[:k] + rst[k + 2:]                                     # one restart marker taken out
    return [('cut', cut), ('flipped', bytes(flipped)), ('missing_rst', missing)]


@pytest.mark.parametrize('which', [0, 1, 2])
def test_corrupt_data_sets_status(cuda, corpus, tmp_path, which):
    name, bad = _corrupt_files()[which]
    good = [corpus[5][1], corpus[60][1]]
    s, out, items, status, launches, _ = _decode(cuda, [good[0], bad, good[1]])
    assert s == 0 and launches == 5
    assert status[0] == 0 and status[2] == 0 and status[1] != 0, (name, status)
    _check_sentinels(out, items)
    for i, data in ((0, good[0]), (2, good[1])):
        assert np.array_equal(_slot(out, items[i]), jpeg_decode_corpus.cv2_decode(data, tmp_path)), name


def test_imread_gpu(cuda, tmp_path):
    from yolact_minimal_b200.utils.augmentations import imread_gpu
    for name, img in jpeg_corpus.photos():
        p = os.path.join(jpeg_corpus.GOLDEN_DIR, name + '.jpg')
        got = imread_gpu(p, cuda)
        assert got.is_cuda and np.array_equal(got.cpu().numpy(), img), name
    prog = tmp_path / 'prog.jpg'
    prog.write_bytes(jpeg_decode_corpus.refused()[0][1])
    assert np.array_equal(imread_gpu(str(prog), cuda).cpu().numpy(), jpeg_decode_corpus.cv2_decode(prog.read_bytes(), tmp_path))


def test_large_dequantized_coefficients_equal_oracle(cuda):
    """Dequantized coefficients far outside the DCT range (a 16-bit quantization table): the kernels' 64-bit IDCT sums equal the
    oracle's, which restate jidctint.c's C arithmetic.  (cv2's SIMD IDCT works in 16-bit lanes there, so cv2 is not compared.)"""
    from test_jpeg_decode_cpu import large_dequant_file
    data = large_dequant_file()
    s, out, items, status, launches, _ = _decode(cuda, [data, data])
    assert s == 0 and launches == 5 and status.tolist() == [0, 0]
    want = jpeg_decode_np.decode(data)
    for i in range(2):
        assert np.array_equal(_slot(out, items[i]), want)
