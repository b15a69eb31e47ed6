"""Plain-numpy restatement of the baseline JPEG decode `cv2.imread(path)` runs (libjpeg-turbo: ISLOW IDCT, fancy upsampling,
BGR output, then the EXIF orientation applied as OpenCV applies it).

    parse(data) -> Header                     (raises Unsupported for a valid file outside the supported set, Invalid otherwise)
    decode(data) -> uint8 [h, w, 3] BGR       (what cv2.imread returns for the file)

Supported files: baseline or extended-sequential Huffman, 8-bit samples, one scan holding every component, with or without restart
intervals, and one of: grayscale; YCbCr with chroma 1x1 and luma 1x1, 2x1 or 2x2 (4:4:4, 4:2:2, 4:2:0).
Every step is integer arithmetic as libjpeg-turbo does it:
  entropy      jdhuff.c: DC prediction per component, reset at every restart marker; ZRL and EOB; 0xFF00 destuffing
  transform    jidctint.c's ISLOW IDCT (pass 1 on columns with PASS1_BITS = 2, pass 2 on rows), the output through the
               range-limit table indexed & 1023 (jdmaster.c prepare_range_limit_table)
  upsampling   jdsample.c h2v1 / h2v2 fancy upsampling (plain replication when the downsampled width is at most 2); the
               context row above the first row and below the last real chroma row repeat that row (jdmainct.c)
  colour       jdcolor.c's 16-bit fixed-point YCbCr -> RGB tables; grayscale replicates Y
  orientation  OpenCV's ExifTransform for EXIF Orientation 1 .. 8 in the first APP1 'Exif' segment
"""
from dataclasses import dataclass, field

import numpy as np

from .jpeg_np import ZIGZAG


class Unsupported(ValueError):
    """A valid JPEG outside the supported set (progressive, arithmetic, 12-bit, CMYK / Adobe, 4:1:1, 4:4:0, multi-scan ...)."""


class Invalid(ValueError):
    """Not a JPEG, or a malformed or truncated header."""


@dataclass
class Header:
    h: int = 0                   # frame height and width (before the orientation)
    w: int = 0
    comps: list = field(default_factory=list)      # [(id, hs, vs, tq)] in frame order
    qt: dict = field(default_factory=dict)         # tq -> int64 [64] natural order
    huff: dict = field(default_factory=dict)       # (class, id) -> (16 counts, symbols)
    ri: int = 0                  # restart interval in MCUs (0: none)
    scan: list = field(default_factory=list)       # [(td, ta)] per component, frame order
    scan_off: int = 0            # first byte of the entropy-coded data
    orientation: int = 1

    @property
    def out_hw(self):
        return (self.w, self.h) if self.orientation >= 5 else (self.h, self.w)


def _u16(d, o):
    if o + 2 > len(d):
        raise Invalid('truncated header')
    return (d[o] << 8) | d[o + 1]


def _exif_orientation(seg):
    """Orientation (tag 0x0112) of IFD0 in an APP1 payload starting 'Exif\\0\\0'; 1 when absent or out of 1 .. 8."""
    t = seg[6:]
    if len(t) < 8 or t[:2] not in (b'II', b'MM'):
        return 1
    order = 'little' if t[:2] == b'II' else 'big'
    rd = lambda o, n: int.from_bytes(t[o:o + n], order)
    ifd = rd(4, 4)
    if ifd + 2 > len(t):
        return 1
    for e in range(rd(ifd, 2)):
        o = ifd + 2 + 12 * e
        if o + 12 > len(t):
            break
        if rd(o, 2) == 0x0112 and rd(o + 2, 2) == 3:
            v = rd(o + 8, 2)
            return v if 1 <= v <= 8 else 1
    return 1


def parse(data):
    d = bytes(data)
    if len(d) < 4 or d[0] != 0xFF or d[1] != 0xD8:
        raise Invalid('no SOI')
    hd = Header()
    seen_exif = seen_sof = False
    o = 2
    while True:
        if o >= len(d) or d[o] != 0xFF:
            raise Invalid(f'no marker at byte {o}')
        while o < len(d) and d[o] == 0xFF:
            o += 1
        if o >= len(d):
            raise Invalid('truncated header')
        m = d[o]
        o += 1
        if m == 0x01 or 0xD0 <= m <= 0xD9:
            raise Invalid(f'marker 0x{m:02x} before SOS')
        n = _u16(d, o)
        if n < 2 or o + n > len(d):
            raise Invalid('segment past the end of the file')
        seg = d[o + 2:o + n]
        if m == 0xE1 and not seen_exif and seg[:6] == b'Exif\x00\x00':
            seen_exif = True
            hd.orientation = _exif_orientation(seg)
        elif m == 0xEE and seg[:5] == b'Adobe':
            raise Unsupported('Adobe APP14 (colour transform)')
        elif m == 0xDB:
            p = 0
            while p < len(seg):
                pq, tq = seg[p] >> 4, seg[p] & 15
                size = 128 if pq else 64
                if pq > 1 or tq > 3 or p + 1 + size > len(seg):
                    raise Invalid('bad DQT')
                v = np.frombuffer(seg[p + 1:p + 1 + size], '>u2' if pq else np.uint8).astype(np.int64)
                q = np.zeros(64, np.int64)
                q[ZIGZAG] = v
                hd.qt[tq] = q
                p += 1 + size
        elif m == 0xC4:
            p = 0
            while p < len(seg):
                if p + 17 > len(seg):
                    raise Invalid('bad DHT')
                tc, th = seg[p] >> 4, seg[p] & 15
                counts = list(seg[p + 1:p + 17])
                nv = sum(counts)
                if tc > 1 or th > 3 or nv > 256 or p + 17 + nv > len(seg):
                    raise Invalid('bad DHT')
                hd.huff[(tc, th)] = (counts, list(seg[p + 17:p + 17 + nv]))
                p += 17 + nv
        elif m == 0xDD:
            if n != 4:
                raise Invalid('bad DRI')
            hd.ri = _u16(d, o + 2)
        elif m in (0xC0, 0xC1):
            if seen_sof or len(seg) < 6:
                raise Invalid('bad SOF')
            seen_sof = True
            prec, hd.h, hd.w, nf = seg[0], _u16(seg, 1), _u16(seg, 3), seg[5]
            if len(seg) != 6 + 3 * nf or nf == 0:
                raise Invalid('bad SOF')
            if prec != 8:
                raise Unsupported(f'{prec}-bit samples')
            if hd.h == 0 or hd.w == 0:
                raise Unsupported('height or width 0 (DNL)')
            hd.comps = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nf)]
        elif 0xC2 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            raise Unsupported(f'SOF 0x{m:02x} (progressive, lossless or arithmetic)')
        elif m == 0xCC:
            raise Unsupported('arithmetic coding')
        elif m == 0xDA:
            if not seen_sof:
                raise Invalid('SOS before SOF')
            ns = seg[0] if seg else 0
            if len(seg) != 4 + 2 * ns:
                raise Invalid('bad SOS')
            ids = [seg[1 + 2 * i] for i in range(ns)]
            if ids != [c[0] for c in hd.comps]:
                raise Unsupported('a scan without every component in frame order (multi-scan)')
            if (seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]) != (0, 63, 0):
                raise Unsupported('spectral selection or successive approximation')
            hd.scan = [(seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15) for i in range(ns)]
            hd.scan_off = o + n
            _check_layout(hd)
            return hd
        o += n


def _check_layout(hd):
    nf = len(hd.comps)
    if nf == 3:
        if [(c[1], c[2]) for c in hd.comps[1:]] != [(1, 1), (1, 1)] or (hd.comps[0][1], hd.comps[0][2]) not in ((1, 1), (2, 1), (2, 2)):
            raise Unsupported(f'sampling {[(c[1], c[2]) for c in hd.comps]}')
        if [c[0] for c in hd.comps] == [82, 71, 66]:
            raise Unsupported('RGB components')
    elif nf != 1:
        raise Unsupported(f'{nf} components')
    for (cid, hs, vs, tq), (td, ta) in zip(hd.comps, hd.scan):
        if not (1 <= hs <= 4 and 1 <= vs <= 4):
            raise Invalid('bad sampling factor')
        if tq not in hd.qt or (0, td) not in hd.huff or (1, ta) not in hd.huff:
            raise Invalid('a table the scan uses is not defined')
        for cls, tid in ((0, td), (1, ta)):
            if not valid_table(*hd.huff[(cls, tid)], dc=cls == 0):
                raise Invalid('a Huffman table the scan uses is invalid')


def valid_table(counts, vals, dc):
    """jdhuff.c jpeg_make_d_derived_tbl's checks: the codes of every length fit in that many bits with the all-ones code left
    free, and DC symbols are at most 15."""
    last = max((l for l in range(1, 17) if counts[l - 1]), default=0)
    code = 0
    for l in range(1, last + 1):
        code += counts[l - 1]
        if code >= 1 << l:
            return False
        code <<= 1
    return not dc or all(v <= 15 for v in vals)


def geometry(hd):
    """(hmax, vmax, mcus_x, mcus_y, [(blocks wide, blocks high) per component in the MCU grid]).  A grayscale scan is
    non-interleaved: one block per MCU over ceil(w/8) x ceil(h/8)."""
    if len(hd.comps) == 1:
        bx, by = -(-hd.w // 8), -(-hd.h // 8)
        return 1, 1, bx, by, [(bx, by)]
    hmax, vmax = max(c[1] for c in hd.comps), max(c[2] for c in hd.comps)
    mx, my = -(-hd.w // (8 * hmax)), -(-hd.h // (8 * vmax))
    return hmax, vmax, mx, my, [(mx * c[1], my * c[2]) for c in hd.comps]


def _huff_lut(counts, vals):
    """16-bit lookahead -> (symbol, code length); length 0 where no code matches."""
    sym, ln = np.zeros(1 << 16, np.int64), np.zeros(1 << 16, np.int64)
    code, k = 0, 0
    for l in range(1, 17):
        for _ in range(counts[l - 1]):
            lo = code << (16 - l)
            sym[lo:lo + (1 << (16 - l))] = vals[k]
            ln[lo:lo + (1 << (16 - l))] = l
            code += 1
            k += 1
        code <<= 1
    return sym.tolist(), ln.tolist()


def intervals(data, start):
    """Destuffed entropy-coded bytes from `start` to the first marker other than RSTn, split at the restart markers."""
    d = bytes(data)
    out, cur, o = [], bytearray(), start
    while True:
        f = d.find(b'\xff', o)
        if f < 0 or f + 1 >= len(d):
            cur += d[o:]
            out.append(bytes(cur))
            return out
        cur += d[o:f]
        m = d[f + 1]
        if m == 0x00:
            cur.append(0xFF)
            o = f + 2
        elif 0xD0 <= m <= 0xD7:
            out.append(bytes(cur))
            cur = bytearray()
            o = f + 2
        elif m == 0xFF:
            o = f + 1                  # fill byte before a marker
        else:
            out.append(bytes(cur))
            return out


def coefficients(data, hd=None):
    """Quantized coefficients per component, int64 [blocks high, blocks wide, 64] natural order (DC prediction applied)."""
    hd = hd or parse(data)
    hmax, vmax, mx, my, grids = geometry(hd)
    coef = [np.zeros((gy, gx, 64), np.int64) for gx, gy in grids]
    if len(hd.comps) == 1:
        mcu_blocks = [(0, 0, 0)]
    else:
        mcu_blocks = [(ci, bx, by) for ci, c in enumerate(hd.comps) for by in range(c[2]) for bx in range(c[1])]
    luts = {k: _huff_lut(*v) for k, v in hd.huff.items()}
    n_mcu = mx * my
    ri = hd.ri or n_mcu
    segs = intervals(data, hd.scan_off)
    n_int = -(-n_mcu // ri)
    if len(segs) < n_int:
        raise Invalid(f'{len(segs)} restart intervals, {n_int} expected')
    zz = ZIGZAG.tolist()
    for it in range(n_int):
        s = segs[it] + b'\x00' * 8
        nbits = 8 * len(segs[it])
        pos = 0

        def bits(n):
            nonlocal pos
            b = pos >> 3
            v = ((s[b] << 24) | (s[b + 1] << 16) | (s[b + 2] << 8) | s[b + 3]) >> (32 - n - (pos & 7)) & ((1 << n) - 1)
            pos += n
            return v

        def huff(lut):
            nonlocal pos
            b = pos >> 3
            v = ((s[b] << 16) | (s[b + 1] << 8) | s[b + 2]) >> (8 - (pos & 7)) & 0xFFFF
            l = lut[1][v]
            if l == 0:
                raise Invalid('invalid Huffman code')
            pos += l
            return lut[0][v]

        def extend(v, t):
            return v - (1 << t) + 1 if t and v < (1 << (t - 1)) else v

        pred = [0] * len(hd.comps)
        for m in range(it * ri, min(n_mcu, (it + 1) * ri)):
            my_, mx_ = divmod(m, mx)
            for ci, bx, by in mcu_blocks:
                c = hd.comps[ci]
                dc, ac = luts[(0, hd.scan[ci][0])], luts[(1, hd.scan[ci][1])]
                blk = coef[ci][my_ * (c[2] if len(hd.comps) > 1 else 1) + by, mx_ * (c[1] if len(hd.comps) > 1 else 1) + bx]
                t = huff(dc)
                pred[ci] += extend(bits(t) if t else 0, t)
                blk[0] = pred[ci]
                k = 1
                while k < 64:
                    rs = huff(ac)
                    r, t = rs >> 4, rs & 15
                    if t == 0:
                        if r != 15:
                            break
                        k += 16
                        continue
                    k += r
                    if k > 63:
                        raise Invalid('run past coefficient 63')
                    blk[zz[k]] = extend(bits(t), t)
                    k += 1
                if k > 64:
                    raise Invalid('run past coefficient 63')
        if pos > nbits:
            raise Invalid('entropy-coded data ends early')
    return coef


# ---- ISLOW IDCT ----------------------------------------------------------------------------------------------------------------
CONST_BITS, PASS1_BITS = 13, 2
F0298, F0390, F0541, F0765, F0899, F1175 = 2446, 3196, 4433, 6270, 7373, 9633
F1501, F1847, F1961, F2053, F2562, F3072 = 12299, 15137, 16069, 16819, 20995, 25172


def _idct_1d(d0, d1, d2, d3, d4, d5, d6, d7):
    """The even and odd parts of jpeg_idct_islow; returns the 8 sums before the descale."""
    z1 = (d2 + d6) * F0541
    tmp2 = z1 - d6 * F1847
    tmp3 = z1 + d2 * F0765
    tmp0 = (d0 + d4) << CONST_BITS
    tmp1 = (d0 - d4) << CONST_BITS
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    o0, o1, o2, o3 = d7, d5, d3, d1
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * F1175
    o0, o1, o2, o3 = o0 * F0298, o1 * F2053, o2 * F3072, o3 * F1501
    z1, z2, z3, z4 = -z1 * F0899, -z2 * F2562, -z3 * F1961 + z5, -z4 * F0390 + z5
    o0 += z1 + z3
    o1 += z2 + z4
    o2 += z2 + z3
    o3 += z1 + z4
    return [t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3]


def range_limit(x):
    """IDCT output x (before the +128) -> sample: the post-IDCT range-limit table indexed x & 1023."""
    y = ((x + 512) & 1023) - 512
    return np.clip(y + 128, 0, 255)


def idct_islow(coef, q):
    """coef int64 [..., 64] natural order, q [64] -> uint8 [..., 8, 8].  jidctint.c's C arithmetic: 64-bit sums (JLONG), the pass-1
    results stored in an int workspace."""
    c = (coef * q).reshape(coef.shape[:-1] + (8, 8))
    n1 = CONST_BITS - PASS1_BITS
    ws = _idct_1d(*[c[..., k, :] for k in range(8)])              # columns: rows k of the block
    ws = np.stack([(v + (1 << (n1 - 1))) >> n1 for v in ws], -2).astype(np.int32).astype(np.int64)    # the int workspace
    n2 = CONST_BITS + PASS1_BITS + 3
    out = _idct_1d(*[ws[..., :, k] for k in range(8)])           # rows
    out = np.stack([(v + (1 << (n2 - 1))) >> n2 for v in out], -1)
    return range_limit(out).astype(np.uint8)


def planes(data, hd=None):
    """Component planes at their own resolution, cropped to libjpeg's downsampled size ceil(w * hs / hmax) x ceil(h * vs / vmax)."""
    hd = hd or parse(data)
    hmax, vmax, _, _, _ = geometry(hd)
    out = []
    for (cid, hs, vs, tq), cf in zip(hd.comps, coefficients(data, hd)):
        px = idct_islow(cf, hd.qt[tq])                               # [by, bx, 8, 8]
        px = px.transpose(0, 2, 1, 3).reshape(px.shape[0] * 8, px.shape[1] * 8)
        if len(hd.comps) == 1:
            hs = vs = hmax = vmax = 1
        out.append(px[:-(-hd.h * vs // vmax), :-(-hd.w * hs // hmax)].astype(np.int64))
    return out


# ---- upsampling, colour, orientation -------------------------------------------------------------------------------------------
def _h2v1_fancy(p):
    """jdsample.c h2v1_fancy_upsample on every row of p [rows, W] (W > 2) -> [rows, 2W]."""
    left = np.concatenate([p[:, :1], p[:, :-1]], 1)
    right = np.concatenate([p[:, 1:], p[:, -1:]], 1)
    out = np.empty((p.shape[0], 2 * p.shape[1]), np.int64)
    out[:, 0::2] = (3 * p + left + 1) >> 2
    out[:, 1::2] = (3 * p + right + 2) >> 2
    out[:, 0], out[:, -1] = p[:, 0], p[:, -1]
    return out


def _h2v2_fancy(p):
    """jdsample.c h2v2_fancy_upsample over p [R, W] (W > 2) -> [2R, 2W]; rows beyond the edges repeat the edge row."""
    above = np.concatenate([p[:1], p[:-1]], 0)
    below = np.concatenate([p[1:], p[-1:]], 0)
    out = np.empty((2 * p.shape[0], 2 * p.shape[1]), np.int64)
    for v, other in ((0, above), (1, below)):
        s = 3 * p + other
        left = np.concatenate([s[:, :1], s[:, :-1]], 1)
        right = np.concatenate([s[:, 1:], s[:, -1:]], 1)
        o = out[v::2]
        o[:, 0::2] = (3 * s + left + 8) >> 4
        o[:, 1::2] = (3 * s + right + 7) >> 4
        o[:, 0] = (4 * s[:, 0] + 8) >> 4
        o[:, -1] = (4 * s[:, -1] + 7) >> 4
    return out


def upsample(p, fh, fv):
    """A chroma plane to luma resolution: factor fh x fv in {1x1, 2x1, 2x2}."""
    if fh == 1 and fv == 1:
        return p
    if p.shape[1] <= 2:
        return np.repeat(np.repeat(p, fh, 1), fv, 0)
    return _h2v1_fancy(p) if fv == 1 else _h2v2_fancy(p)


def _fix(x):
    return int(x * 65536 + 0.5)


_X = np.arange(256, dtype=np.int64) - 128
CR_R = (_fix(1.40200) * _X + (1 << 15)) >> 16
CB_B = (_fix(1.77200) * _X + (1 << 15)) >> 16
CR_G = -_fix(0.71414) * _X
CB_G = -_fix(0.34414) * _X + (1 << 15)


def ycc_to_bgr(y, cb, cr):
    r = np.clip(y + CR_R[cr], 0, 255)
    g = np.clip(y + ((CB_G[cb] + CR_G[cr]) >> 16), 0, 255)
    b = np.clip(y + CB_B[cb], 0, 255)
    return np.stack([b, g, r], -1).astype(np.uint8)


def orient(img, o):
    """OpenCV's ExifTransform for orientation o."""
    if o >= 5:
        img = img.transpose(1, 0, 2)
    flips = {2: (False, True), 3: (True, True), 4: (True, False), 6: (False, True), 7: (True, True), 8: (True, False)}
    fv, fh = flips.get(o, (False, False))
    if fv:
        img = img[::-1]
    if fh:
        img = img[:, ::-1]
    return np.ascontiguousarray(img)


def decode(data):
    hd = parse(data)
    ps = planes(data, hd)
    if len(ps) == 1:
        img = np.repeat(ps[0][..., None], 3, -1).astype(np.uint8)
    else:
        fh, fv = hd.comps[0][1], hd.comps[0][2]
        y = ps[0]
        cb, cr = (upsample(p, fh, fv)[:hd.h, :hd.w] for p in ps[1:])
        img = ycc_to_bgr(y, cb, cr)
    return orient(img, hd.orientation)
