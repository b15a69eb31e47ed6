"""CPU: the numpy restatement of cv2's baseline JPEG encoder (oracle/jpeg_np.py) equals cv2.imencode('.jpg') byte for byte on the
seeded corpus (tests/jpeg_corpus.py: every MCU edge rule, noise for the longest codes and 0xFF stuffing, gradients, constants,
checkerboards, three photos) at q 95, 100 and 50, and equals the bytes minted into tests/golden/jpeg.npz."""
import hashlib
import os

import numpy as np
import pytest

import jpeg_corpus
from oracle import jpeg_np

GOLDEN = os.path.join(jpeg_corpus.GOLDEN_DIR, 'jpeg.npz')
CASES = jpeg_corpus.corpus()


def _cv2(img, q):
    cv2 = pytest.importorskip('cv2')
    return cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()


@pytest.fixture(scope='module')
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize('q', jpeg_corpus.QUALITIES)
@pytest.mark.parametrize('name,img', CASES, ids=[c[0] for c in CASES])
def test_oracle_equals_cv2_and_golden(name, img, q, golden):
    got = jpeg_np.encode(img, q)
    key = f'{name}@{q}'
    assert len(got) == int(golden[f'len/{key}']), key
    assert hashlib.sha256(got).digest() == golden[f'sha256/{key}'].tobytes(), key
    if f'bytes/{key}' in golden:
        assert got == golden[f'bytes/{key}'].tobytes()
    assert got == _cv2(img, q)


@pytest.mark.parametrize('q', [1, 10, 49, 51, 75, 99])
def test_oracle_other_qualities(q):
    img = jpeg_corpus.synth(37, 53, 'noise', seed=q)
    assert jpeg_np.encode(img, q) == _cv2(img, q)


def test_header_layout():
    """SOF0's height and width are the only image-dependent header bytes, at the offsets the CUDA stuff kernel patches."""
    a, b = jpeg_np.header(1, 1, 95), jpeg_np.header(0x1234, 0x5678, 95)
    assert len(a) == 623 and a[158:160] == b'\xff\xc0'
    assert [i for i in range(len(a)) if a[i] != b[i]] == [163, 164, 165, 166]
    assert b[163:167] == bytes([0x12, 0x34, 0x56, 0x78])


def _decode_coefficients(data):
    """Baseline Huffman decoder of a file with cv2's layout: the quantized coefficients in scan order, zigzag within a block."""
    hdr = 623
    h, w = int.from_bytes(data[163:165], 'big'), int.from_bytes(data[165:167], 'big')
    scan = data[hdr:-2].replace(b'\xff\x00', b'\xff')
    bits = np.unpackbits(np.frombuffer(scan, np.uint8))
    tables = []
    for spec in jpeg_np.HUFF_SPECS:
        tables.append({(l, c): s for s, (c, l) in jpeg_np.huff_codes(*spec).items()})
    pos = 0

    def read(n):
        nonlocal pos
        v = 0
        for _ in range(n):
            v = (v << 1) | int(bits[pos])
            pos += 1
        return v

    def sym(t):
        c = l = 0
        while True:
            c, l = (c << 1) | read(1), l + 1
            if (l, c) in tables[t]:
                return tables[t][(l, c)]

    def extend(v, s):
        return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v

    mx, my, _, _ = jpeg_np.geometry(h, w)
    out = np.zeros((mx * my * 6, 64), np.int64)
    pred = [0, 0, 0]
    for blk in range(len(out)):
        comp = [0, 0, 0, 0, 1, 2][blk % 6]
        t = 2 * (comp > 0)
        s = sym(t)
        pred[comp] += extend(read(s), s)
        out[blk, 0] = pred[comp]
        k = 1
        while k < 64:
            rs = sym(t + 1)
            r, s = rs >> 4, rs & 15
            if s == 0:
                if r == 15:
                    k += 16
                    continue
                break
            k += r
            out[blk, k] = extend(read(s), s)
            k += 1
    return out


@pytest.mark.parametrize('h,w', [(15, 17), (37, 53)])
def test_coefficients_decode_back(h, w):
    """cv2's own file decodes to the oracle's quantized coefficients, dummy blocks included."""
    img = jpeg_corpus.synth(h, w, 'gradient')
    np.testing.assert_array_equal(_decode_coefficients(_cv2(img, 95)), jpeg_np.coefficients(img, 95))
