"""Plain-numpy restatement of the baseline JPEG encoder `cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, q])` runs
(libjpeg-turbo with cv2's defaults: 4:2:0, ISLOW DCT, standard Annex K Huffman tables, no restart markers, JFIF header).

    encode(img_bgr_uint8_hw3, quality=95) -> bytes           (the file cv2 writes)

Every step is integer arithmetic as libjpeg-turbo does it, so the bytes equal cv2's:
  header       jpeg_set_quality's scaling of the Annex K tables; SOI, APP0 JFIF 1.01, DQT x2, SOF0, DHT x4, SOS ... EOI
  colour       jccolor.c's 16-bit fixed-point RGB -> YCbCr
  downsample   jcsample.c h2v2 with the alternating 1, 2 rounding bias; right columns replicated to the padded width,
               the bottom row replicated to an even row count, then the last chroma row to the MCU height (jcprepct.c)
  dummy blocks jccoefct.c: a partial last MCU holds blocks with zero AC and the quantized DC of the block to the left
               (right edge) or of the MCU's last block of the block row above (bottom edge)
  transform    jfdctint.c's ISLOW forward DCT, then jcdctmgr.c's quantization by reciprocal multiply of divisor q << 3
  entropy      jchuff.c: per-component DC prediction, ZRL and EOB, 0xFF00 stuffing, 1-bit padding
"""
import numpy as np

BASE_LUMA = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)
BASE_CHROMA = np.array([
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
    47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32, np.int64)

# Annex K.3 - K.6 as (16 code-length counts, symbols): DC luma, AC luma, DC chroma, AC chroma
_AC_LUMA_VALS = (
    '01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a3435363738393a4344'
    '45464748494a535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4'
    'b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa')
_AC_CHROMA_VALS = (
    '000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a35363738393a43'
    '4445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2'
    'b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa')
HUFF_SPECS = (
    ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12))),
    ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], list(bytes.fromhex(_AC_LUMA_VALS))),
    ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12))),
    ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], list(bytes.fromhex(_AC_CHROMA_VALS))),
)


def _zigzag():
    """ZIGZAG[k] = natural (row-major) index of the k-th coefficient in zigzag order."""
    order = sorted(((r, c) for r in range(8) for c in range(8)),
                   key=lambda rc: (rc[0] + rc[1], rc[1] if (rc[0] + rc[1]) % 2 == 0 else rc[0]))
    return np.array([r * 8 + c for r, c in order], np.int64)


ZIGZAG = _zigzag()


def quant_tables(quality):
    """jpeg_set_quality(cinfo, quality, force_baseline=TRUE): the luma and chroma tables in natural order."""
    q = min(max(int(quality), 1), 100)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return [np.clip((base * scale + 50) // 100, 1, 255) for base in (BASE_LUMA, BASE_CHROMA)]


def huff_codes(bits, vals):
    """Canonical Huffman code of each symbol (jchuff.c jpeg_make_c_derived_tbl): {symbol: (code, length)}."""
    codes, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            codes[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return codes


def header(h, w, quality):
    """Every byte before the entropy-coded segment; only SOF0's height and width depend on the image."""
    tables = quant_tables(quality)
    out = bytearray(b'\xff\xd8')
    out += b'\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00'
    for i, t in enumerate(tables):
        out += bytes([0xff, 0xdb, 0x00, 0x43, i]) + bytes(t[ZIGZAG].astype(np.uint8))
    out += bytes([0xff, 0xc0, 0x00, 0x11, 8, h >> 8, h & 255, w >> 8, w & 255, 3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1])
    for cls_id, (bits, vals) in zip((0x00, 0x10, 0x01, 0x11), HUFF_SPECS):
        n = 2 + 1 + 16 + len(vals)
        out += bytes([0xff, 0xc4, n >> 8, n & 255, cls_id]) + bytes(bits) + bytes(vals)
    out += bytes([0xff, 0xda, 0x00, 0x0c, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0])
    return bytes(out)


# ---- colour conversion and downsampling -------------------------------------------------------------------------------
SCALEBITS = 16
ONE_HALF = 1 << (SCALEBITS - 1)
CBCR_OFFSET = 128 << SCALEBITS


def _fix(x):
    return int(x * (1 << SCALEBITS) + 0.5)


def rgb_to_ycc(img_bgr):
    """jccolor.c rgb_ycc_convert on a BGR image: int64 Y, Cb, Cr planes."""
    b, g, r = (img_bgr[..., i].astype(np.int64) for i in range(3))
    y = (_fix(0.29900) * r + _fix(0.58700) * g + _fix(0.11400) * b + ONE_HALF) >> SCALEBITS
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + CBCR_OFFSET + ONE_HALF - 1) >> SCALEBITS
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + CBCR_OFFSET + ONE_HALF - 1) >> SCALEBITS
    return y, cb, cr


def geometry(h, w):
    """(MCU columns, MCU rows, Y blocks across, Y blocks down): Y is 2x2 blocks per 16x16 MCU, Cb and Cr one each."""
    return -(-w // 16), -(-h // 16), -(-w // 8), -(-h // 8)


def planes(img_bgr):
    """The padded sample planes the DCT reads: Y [16 my, 16 mx] and Cb, Cr [8 my, 8 mx] (Y beyond its real blocks unused)."""
    h, w = img_bgr.shape[:2]
    mx, my, _, _ = geometry(h, w)
    y, cb, cr = rgb_to_ycc(img_bgr)
    rows = np.minimum(np.arange(16 * my), h - 1)
    cols = np.minimum(np.arange(16 * mx), w - 1)
    yp = y[rows][:, cols]
    # chroma: the colour buffer is padded to an even row count, then the last downsampled row fills the MCU height
    ch = -(-h // 2)
    r2 = np.minimum(np.arange(8 * my), ch - 1)
    top, bot = np.minimum(2 * r2, h - 1), np.minimum(2 * r2 + 1, h - 1)
    bias = np.tile(np.array([1, 2], np.int64), 4 * mx)
    out = []
    for c in (cb, cr):
        c = c[:, cols]
        s = c[top][:, 0::2] + c[top][:, 1::2] + c[bot][:, 0::2] + c[bot][:, 1::2]
        out.append((s + bias) >> 2)
    return yp, out[0], out[1]


# ---- ISLOW forward DCT and quantization -------------------------------------------------------------------------------
CONST_BITS, PASS1_BITS = 13, 2
F0298, F0390, F0541, F0765, F0899, F1175 = 2446, 3196, 4433, 6270, 7373, 9633
F1501, F1847, F1961, F2053, F2562, F3072 = 12299, 15137, 16069, 16819, 20995, 25172


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_pass(d, first):
    """One 1-D pass of jpeg_fdct_islow along the last axis of d [..., 8]."""
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    n = CONST_BITS - PASS1_BITS if first else CONST_BITS + PASS1_BITS
    o = np.empty_like(d)
    if first:
        o[..., 0], o[..., 4] = (t10 + t11) << PASS1_BITS, (t10 - t11) << PASS1_BITS
    else:
        o[..., 0], o[..., 4] = _descale(t10 + t11, PASS1_BITS), _descale(t10 - t11, PASS1_BITS)
    z1 = (t12 + t13) * F0541
    o[..., 2] = _descale(z1 + t13 * F0765, n)
    o[..., 6] = _descale(z1 - t12 * F1847, n)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * F1175
    t4, t5, t6, t7 = t4 * F0298, t5 * F2053, t6 * F3072, t7 * F1501
    z1, z2, z3, z4 = -z1 * F0899, -z2 * F2562, -z3 * F1961 + z5, -z4 * F0390 + z5
    o[..., 7] = _descale(t4 + z1 + z3, n)
    o[..., 5] = _descale(t5 + z2 + z4, n)
    o[..., 3] = _descale(t6 + z2 + z3, n)
    o[..., 1] = _descale(t7 + z1 + z4, n)
    return o


def fdct_islow(blocks):
    """jpeg_fdct_islow on level-shifted samples [..., 8, 8] (int64): coefficients scaled up by 8, natural order."""
    d = _fdct_pass(blocks, True)
    return np.swapaxes(_fdct_pass(np.swapaxes(d, -1, -2), False), -1, -2)


def divisors(table):
    """jcdctmgr.c compute_reciprocal for each divisor q << 3 with 16-bit DCTELEM: (reciprocal, correction, shift)."""
    recip, corr, shift = (np.empty(64, np.int64) for _ in range(3))
    for i, q in enumerate(table):
        d = int(q) << 3
        b = d.bit_length() - 1
        r = 16 + b
        fq, fr = (1 << r) // d, (1 << r) % d
        c = d // 2
        if fr == 0:
            fq >>= 1
            r -= 1
        elif fr <= d // 2:
            c += 1
        else:
            fq += 1
        recip[i], corr[i], shift[i] = fq, c, r
    return recip, corr, shift


def quantize(coef, table):
    """jcdctmgr.c quantize: |x| + correction times the reciprocal, shifted, sign restored."""
    recip, corr, shift = divisors(table)
    mag = ((np.abs(coef) + corr) * recip) >> shift
    return np.where(coef < 0, -mag, mag)


def _blocks(plane, nby, nbx):
    return plane.reshape(nby, 8, nbx, 8).transpose(0, 2, 1, 3)


def coefficients(img_bgr, quality=95):
    """Quantized coefficients in scan order, zigzag within a block: int64 [MCUs * 6, 64], dummy blocks included."""
    h, w = img_bgr.shape[:2]
    mx, my, bx, by = geometry(h, w)
    yq, cq = quant_tables(quality)
    yp, cb, cr = planes(img_bgr)
    q = []
    for p, t, n in ((yp, yq, (2 * my, 2 * mx)), (cb, cq, (my, mx)), (cr, cq, (my, mx))):
        blk = _blocks(p - 128, *n)
        q.append(quantize(fdct_islow(blk).reshape(*n, 64), t))
    yb = q[0]
    # dummy blocks of a partial last MCU (jccoefct.c): zero AC, DC of the neighbouring real block
    if bx % 2:
        yb[:, bx] = 0
        yb[:, bx, 0] = yb[:, bx - 1, 0]
    if by % 2:
        yb[by] = 0
        yb[by, :, 0] = yb[by - 1, 1::2, 0].repeat(2)
    y4 = yb.reshape(my, 2, mx, 2, 64).transpose(0, 2, 1, 3, 4).reshape(my, mx, 4, 64)
    scan = np.concatenate([y4, q[1][:, :, None], q[2][:, :, None]], axis=2).reshape(-1, 64)
    return scan[:, ZIGZAG]


# ---- entropy coding ---------------------------------------------------------------------------------------------------
def _nbits(v):
    """Magnitude category: bits needed for |v| (0 for 0)."""
    a = np.abs(v)
    n = np.zeros(a.shape, np.int64)
    while np.any(a >> n):
        n += (a >> n) > 0
    return n


def _lut(codes):
    code, size = np.zeros(256, np.int64), np.zeros(256, np.int64)
    for s, (c, l) in codes.items():
        code[s], size[s] = c, l
    return code, size


_LUTS = [_lut(huff_codes(*spec)) for spec in HUFF_SPECS]


def symbols(zz):
    """The entropy-coded segment of scan-order coefficients zz [N, 64] as (value, length) per Huffman code, in stream order.
    Each value is the Huffman code followed by the coefficient's extra bits."""
    n = zz.shape[0]
    comp = np.tile(np.array([0, 0, 0, 0, 1, 2]), n // 6)
    chroma = (comp > 0).astype(np.int64)
    dc = zz[:, 0]
    diff = np.empty_like(dc)
    for c in range(3):
        sel = np.nonzero(comp == c)[0]
        diff[sel] = np.diff(dc[sel], prepend=0)
    # (block, order key, symbol, extra-bit value, extra-bit count, table): DC at key 0, ZRLs and the coefficient at key 4k..4k+3,
    # EOB at key 256
    blk, key, sym, val, nb, tab = [], [], [], [], [], []
    s = _nbits(diff)
    blk.append(np.arange(n)); key.append(np.zeros(n, np.int64)); sym.append(s)
    val.append(diff); nb.append(s); tab.append(2 * chroma)
    bi, k = np.nonzero(zz[:, 1:])
    k = k + 1
    first = np.ones(len(bi), bool)
    first[1:] = bi[1:] != bi[:-1]
    prev = np.where(first, 0, np.concatenate([[0], k[:-1]]))
    run = k - prev - 1
    v = zz[bi, k]
    s = _nbits(v)
    blk.append(bi); key.append(4 * k + 3); sym.append(((run & 15) << 4) | s)
    val.append(v); nb.append(s); tab.append(2 * chroma[bi] + 1)
    nz = run >> 4
    zb, zk = np.repeat(bi, nz), np.repeat(4 * k, nz)
    zj = np.arange(len(zb)) - np.repeat(np.cumsum(nz) - nz, nz)
    blk.append(zb); key.append(zk + zj); sym.append(np.full(len(zb), 0xF0))
    val.append(np.zeros(len(zb), np.int64)); nb.append(np.zeros(len(zb), np.int64)); tab.append(2 * chroma[zb] + 1)
    last = np.zeros(n, np.int64)
    np.maximum.at(last, bi, k)
    eb = np.nonzero(last < 63)[0]
    blk.append(eb); key.append(np.full(len(eb), 256)); sym.append(np.zeros(len(eb), np.int64))
    val.append(np.zeros(len(eb), np.int64)); nb.append(np.zeros(len(eb), np.int64)); tab.append(2 * chroma[eb] + 1)
    blk, key, sym, val, nb, tab = (np.concatenate(a) for a in (blk, key, sym, val, nb, tab))
    order = np.lexsort((key, blk))
    sym, val, nb, tab = sym[order], val[order], nb[order], tab[order]
    code, size = np.zeros(len(sym), np.int64), np.zeros(len(sym), np.int64)
    for t in range(4):
        sel = tab == t
        code[sel], size[sel] = _LUTS[t][0][sym[sel]], _LUTS[t][1][sym[sel]]
    assert np.all(size > 0), 'symbol without a Huffman code'
    extra = np.where(val < 0, val - 1, val) & ((1 << nb) - 1)
    return (code << nb) | extra, size + nb


def pack_bits(value, length, chunk=1 << 20):
    """MSB-first concatenation of the codes, padded with 1-bits to a whole byte, 0xFF bytes followed by 0x00."""
    bits = []
    for a in range(0, len(value), chunk):
        v, l = value[a:a + chunk], length[a:a + chunk]
        start = np.cumsum(l) - l
        idx = np.arange(int(l.sum())) - np.repeat(start, l)
        bits.append(((np.repeat(v, l) >> (np.repeat(l, l) - 1 - idx)) & 1).astype(np.uint8))
    bits = np.concatenate(bits) if bits else np.zeros(0, np.uint8)
    bits = np.concatenate([bits, np.ones(-len(bits) % 8, np.uint8)])
    data = np.packbits(bits)
    ff = np.nonzero(data == 0xFF)[0]
    return np.insert(data, ff + 1, 0).tobytes()


def encode(img_bgr, quality=95):
    """The bytes of cv2.imencode('.jpg', img_bgr, [cv2.IMWRITE_JPEG_QUALITY, quality])[1] for uint8 [h, w, 3]."""
    img = np.asarray(img_bgr)
    assert img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3, 'uint8 [h, w, 3] BGR'
    h, w = img.shape[:2]
    assert 1 <= h <= 65535 and 1 <= w <= 65535 and 1 <= quality <= 100
    value, length = symbols(coefficients(img, quality))
    return header(h, w, quality) + pack_bits(value, length) + b'\xff\xd9'
