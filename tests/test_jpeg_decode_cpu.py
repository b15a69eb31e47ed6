"""CPU: the numpy restatement of cv2's baseline JPEG decode (oracle/jpeg_decode_np.py) equals cv2.imread pixel for pixel on the
corpus of tests/jpeg_decode_corpus.py (4:4:4, 4:2:2, 4:2:0 and grayscale; restart intervals, optimized Huffman tables, qualities
50 to 100; sizes 1x1 to 1080x1920 across every MCU edge; the three photos; EXIF orientations 1 to 8 in both byte orders) and the
pixels minted into tests/golden/jpeg_decode.npz.  yb_jpeg_header reads the same (h, w) and refuses progressive, 4:1:1, 4:4:0, PNG
and truncated files with the right codes."""
import hashlib
import os

import numpy as np
import pytest

import jpeg_corpus
import jpeg_decode_corpus
from oracle import jpeg_decode_np

CASES = jpeg_decode_corpus.corpus()


@pytest.fixture(scope='module')
def golden():
    with np.load(os.path.join(jpeg_corpus.GOLDEN_DIR, 'jpeg_decode.npz')) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize('name,data', CASES, ids=[c[0] for c in CASES])
def test_oracle_equals_cv2_and_golden(name, data, golden, tmp_path):
    got = jpeg_decode_np.decode(data)
    assert hashlib.sha256(data).digest() == golden[f'file_sha256/{name}'].tobytes(), f'{name}: cv2 wrote another file'
    assert got.shape == tuple(golden[f'shape/{name}'])
    assert hashlib.sha256(got.tobytes()).digest() == golden[f'pixels_sha256/{name}'].tobytes(), name
    if f'pixels/{name}' in golden:
        assert np.array_equal(got, golden[f'pixels/{name}'])
        assert np.array_equal(jpeg_decode_np.decode(golden[f'file/{name}'].tobytes()), golden[f'pixels/{name}'])
    assert np.array_equal(got, jpeg_decode_corpus.cv2_decode(data, tmp_path))


def test_corpus_covers_the_supported_set():
    layouts = set()
    for name, data in CASES:
        hd = jpeg_decode_np.parse(data)
        layouts.add((len(hd.comps), hd.comps[0][1], hd.comps[0][2], bool(hd.ri), hd.orientation))
    for comps, hs, vs in ((3, 1, 1), (3, 2, 1), (3, 2, 2), (1, 1, 1)):
        assert (comps, hs, vs, True, 1) in layouts and (comps, hs, vs, False, 1) in layouts
    assert {o for *_, o in layouts} == set(range(1, 9))


@pytest.mark.parametrize('name,data', CASES[::7], ids=[c[0] for c in CASES[::7]])
def test_header_size(name, data):
    from yolact_minimal_b200.utils.augmentations import jpeg_header
    assert jpeg_header(np.frombuffer(data, np.uint8)) == jpeg_decode_np.decode(data).shape[:2]


def test_header_refuses():
    import ctypes
    from yolact_minimal_b200 import _lib
    for name, data, code in jpeg_decode_corpus.refused():
        buf = np.frombuffer(data + b'\x00', np.uint8)        # a valid pointer for the empty file too
        h, w = ctypes.c_int32(-7), ctypes.c_int32(-7)
        assert _lib.lib().yb_jpeg_header(buf.ctypes.data, len(data), ctypes.byref(h), ctypes.byref(w)) == code, name
        assert (h.value, w.value) == (-7, -7), name
        with pytest.raises(jpeg_decode_np.Unsupported if code == -3 else jpeg_decode_np.Invalid):
            jpeg_decode_np.parse(data)


def test_read_image_falls_back_to_cv2(tmp_path):
    """read_image(decode_gpu=True) returns the file's bytes for a supported file and cv2.imread's pixels for a refused one."""
    from yolact_minimal_b200.utils.augmentations import EncodedImage, read_image
    img = jpeg_corpus.synth(37, 53, 'gradient')
    for name, data in (('ok', jpeg_decode_corpus.encode(img)), ('prog', jpeg_decode_corpus.encode(img, progressive=True))):
        p = tmp_path / f'{name}.jpg'
        p.write_bytes(data)
        got = read_image(str(p), decode_gpu=True)
        if name == 'ok':
            assert isinstance(got, EncodedImage) and got.data.tobytes() == data and got.shape == (37, 53, 3)
        else:
            assert np.array_equal(got, jpeg_decode_corpus.cv2_decode(data, tmp_path))
        assert np.array_equal(read_image(str(p)), jpeg_decode_corpus.cv2_decode(data, tmp_path))


def test_mixed_batch_layout():
    """A batch of files and pixels gets pack_images' item table."""
    from yolact_minimal_b200.utils.augmentations import EncodedImage, MixedImages, pack_images
    a, b = jpeg_corpus.synth(5, 7, 'noise'), jpeg_corpus.synth(9, 3, 'noise')
    enc = EncodedImage(np.frombuffer(jpeg_decode_corpus.encode(a), np.uint8), 5, 7)
    m = MixedImages([enc, b, enc])
    _, items = pack_images([a, b, a])
    assert np.array_equal(m.items, items)
    assert m.encoded.tolist() == [0, 2] and m.raw == [(int(items[1]['img_off']), b.nbytes)]
    assert m.file_off.tolist() == [0, enc.data.size, 2 * enc.data.size]


def _dht_segments(data):
    """[(offset of the segment's class/id byte, class/id)] of the DHT segments before SOS (one table per segment, as cv2 writes)."""
    out, o = [], 2
    while data[o + 1] != 0xDA:
        n = int.from_bytes(data[o + 2:o + 4], 'big')
        if data[o + 1] == 0xC4:
            out.append((o + 4, data[o + 4]))
        o += 2 + n
    return out


def bad_huffman_files():
    """A cv2 file whose AC luma table claims 162 codes of length 1 (an over-subscribed code space), and one whose DC luma table
    holds the symbol 16 (DC categories stop at 15)."""
    data = jpeg_decode_corpus.encode(jpeg_corpus.synth(16, 16, 'noise'), 95, '420')
    segs = dict((tc, o) for o, tc in _dht_segments(data))
    ac = bytearray(data)
    counts = ac[segs[0x10] + 1:segs[0x10] + 17]
    ac[segs[0x10] + 1:segs[0x10] + 17] = bytes([sum(counts)] + [0] * 15)
    dc = bytearray(data)
    dc[segs[0x00] + 17] = 16
    return [('ac_oversubscribed', bytes(ac)), ('dc_symbol_16', bytes(dc))]


@pytest.mark.parametrize('which', [0, 1])
def test_invalid_huffman_tables_refused(which, tmp_path):
    """jdhuff.c's table checks: yb_jpeg_header, the workspace sizing and the oracle refuse the file as malformed, as libjpeg does."""
    import ctypes
    from yolact_minimal_b200 import _lib
    name, data = bad_huffman_files()[which]
    buf = np.frombuffer(data, np.uint8)
    h, w = ctypes.c_int32(-7), ctypes.c_int32(-7)
    assert _lib.lib().yb_jpeg_header(buf.ctypes.data, len(data), ctypes.byref(h), ctypes.byref(w)) == -1, name
    off = np.array([0, len(data)], np.int64)
    assert _lib.lib().yb_jpeg_decode_workspace_bytes(buf.ctypes.data, off.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), 1) == 0
    with pytest.raises(jpeg_decode_np.Invalid):
        jpeg_decode_np.parse(data)
    assert jpeg_decode_corpus.cv2_decode(data, tmp_path) is None, name


def test_idct_64bit_workspace():
    """Dequantized coefficients far outside the DCT range (a 16-bit quantization table of 30000s over q100 noise): the oracle's IDCT
    keeps jidctint.c's 64-bit sums, which 32-bit sums would not."""
    data = large_dequant_file()
    hd = jpeg_decode_np.parse(data)
    cf = jpeg_decode_np.coefficients(data, hd)[0]
    assert int(np.abs(cf * hd.qt[hd.comps[0][3]]).max()) > 1 << 22
    img = jpeg_decode_np.decode(data)
    assert img.shape == (45, 70, 3) and len(np.unique(img)) > 2


def large_dequant_file():
    """A grayscale q100 noise file whose 8-bit DQT is replaced by a 16-bit one with every entry 30000."""
    data = jpeg_decode_corpus.encode(jpeg_corpus.synth(45, 70, 'noise', 11)[..., 0], 100)
    o = data.index(b'\xff\xdb')
    n = int.from_bytes(data[o + 2:o + 4], 'big')
    assert n == 67
    dqt = b'\xff\xdb' + (131).to_bytes(2, 'big') + bytes([0x10 | (data[o + 4] & 15)]) + (30000).to_bytes(2, "big") * 64
    return data[:o] + dqt + data[o + 2 + n:]
