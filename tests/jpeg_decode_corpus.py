"""The seeded file corpus of the JPEG decode tests: files cv2 writes from tests/jpeg_corpus.py's images and the committed photos,
covering every layout, coding option, MCU edge and EXIF orientation the decoder supports, and files it must refuse."""
import struct

import numpy as np

import jpeg_corpus

SIZES = [(1, 1), (1, 17), (17, 1), (8, 8), (9, 9), (15, 16), (16, 15), (37, 53), (2, 3), (3, 5)]
LAYOUTS = {'444': 'SAMPLING_FACTOR_444', '422': 'SAMPLING_FACTOR_422', '420': 'SAMPLING_FACTOR_420'}


def _cv2():
    import cv2
    return cv2


def encode(img, q=95, layout='420', rst=0, optimize=False, progressive=False):
    """cv2.imencode('.jpg') bytes: a 1-channel image writes a grayscale file."""
    cv2 = _cv2()
    p = [cv2.IMWRITE_JPEG_QUALITY, q]
    if img.ndim == 3:
        p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, getattr(cv2, 'IMWRITE_JPEG_' + LAYOUTS.get(layout, 'SAMPLING_FACTOR_' + layout))]
    if rst:
        p += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    if optimize:
        p += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    if progressive:
        p += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    ok, buf = cv2.imencode('.jpg', img, p)
    assert ok
    return buf.tobytes()


def exif_app1(orientation, little=False):
    """An APP1 segment holding an EXIF IFD0 with one Orientation entry."""
    e = '<' if little else '>'
    tiff = (b'II*\x00' if little else b'MM\x00*') + struct.pack(e + 'I', 8) + struct.pack(e + 'H', 1) + \
        struct.pack(e + 'HHI', 0x0112, 3, 1) + struct.pack(e + 'H', orientation) + b'\x00\x00' + struct.pack(e + 'I', 0)
    payload = b'Exif\x00\x00' + tiff
    return b'\xff\xe1' + struct.pack('>H', len(payload) + 2) + payload


def with_orientation(data, orientation, little=False):
    """Splices the EXIF APP1 in right after SOI."""
    return data[:2] + exif_app1(orientation, little) + data[2:]


def corpus():
    """[(name, file bytes)] in a fixed order, every file inside the supported set."""
    out = []
    for lay in LAYOUTS:
        for h, w in SIZES:
            for kind in ('noise', 'gradient'):
                out.append((f'{kind}_{h}x{w}_{lay}', encode(jpeg_corpus.synth(h, w, kind), 95, lay)))
        out.append((f'noise_61x67_{lay}_q100', encode(jpeg_corpus.synth(61, 67, 'noise', 1), 100, lay)))
        out.append((f'noise_61x67_{lay}_q50', encode(jpeg_corpus.synth(61, 67, 'noise', 2), 50, lay)))
        out.append((f'noise_45x70_{lay}_rst1', encode(jpeg_corpus.synth(45, 70, 'noise', 3), 95, lay, rst=1)))
        out.append((f'gradient_45x70_{lay}_rst3', encode(jpeg_corpus.synth(45, 70, 'gradient'), 95, lay, rst=3)))
        out.append((f'noise_45x70_{lay}_opt', encode(jpeg_corpus.synth(45, 70, 'noise', 4), 90, lay, optimize=True)))
        out.append((f'checker_40x40_{lay}_q100', encode(jpeg_corpus.synth(40, 40, 'checker'), 100, lay)))
        out.append((f'gradient_1080x1920_{lay}', encode(jpeg_corpus.synth(1080, 1920, 'gradient'), 95, lay)))
    for h, w in SIZES + [(61, 67)]:
        out.append((f'gray_{h}x{w}', encode(jpeg_corpus.synth(h, w, 'noise', 5)[..., 1], 95)))
    out.append(('gray_45x70_rst2', encode(jpeg_corpus.synth(45, 70, 'noise', 6)[..., 0], 95, rst=2)))
    out.append(('gray_45x70_q100_opt', encode(jpeg_corpus.synth(45, 70, 'noise', 7)[..., 2], 100, optimize=True)))
    for name, img in jpeg_corpus.photos():
        out.append((f'photo_{name}', open(f'{jpeg_corpus.GOLDEN_DIR}/{name}.jpg', 'rb').read()))
        out.append((f'photo_{name}_420_rst5', encode(img, 95, '420', rst=5)))
    base = encode(jpeg_corpus.synth(19, 29, 'gradient'), 95, '422')
    gray = encode(jpeg_corpus.synth(19, 29, 'noise', 8)[..., 0], 95)
    for o in range(1, 9):
        out.append((f'orient{o}_19x29_422', with_orientation(base, o)))
        out.append((f'orient{o}_19x29_gray_le', with_orientation(gray, o, little=True)))
    return out


def refused():
    """[(name, file bytes, expected status)]: -3 unsupported, -1 invalid."""
    img = jpeg_corpus.synth(37, 53, 'gradient')
    cv2 = _cv2()
    good = encode(img, 95, '420')
    return [('progressive', encode(img, 95, '420', progressive=True), -3),
            ('411', encode(img, 95, '411'), -3),
            ('440', encode(img, 95, '440'), -3),
            ('png', cv2.imencode('.png', img)[1].tobytes(), -1),
            ('empty', b'', -1),
            ('soi_only', good[:2], -1),
            ('header_cut', good[:100], -1),
            ('sos_cut', good[:good.index(b'\xff\xda') + 5], -1)]


def photo_files(sizes=((480, 640), (640, 480), (427, 640)), layouts=('420', '444'), q=95):
    """The committed photos resized to each size and re-encoded by cv2: [(name, bytes)]."""
    cv2 = _cv2()
    out = []
    for name, img in jpeg_corpus.photos():
        for h, w in sizes:
            r = cv2.resize(img, (w, h), interpolation=cv2.INTER_AREA)
            for lay in layouts:
                out.append((f'{name}_{h}x{w}_{lay}', encode(r, q, lay)))
    return out


def cv2_decode(data, tmp_dir, name='f.jpg'):
    """cv2.imread of the bytes written to a file."""
    cv2 = _cv2()
    p = f'{tmp_dir}/{name}'
    with open(p, 'wb') as f:
        f.write(data)
    return cv2.imread(p)


def as_array(data):
    return np.frombuffer(data, np.uint8)
