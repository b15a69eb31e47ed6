"""The seeded image corpus of the JPEG tests: every size and content the encoder's edge rules and longest codes depend on, and
three photos (tests/golden/*.jpg, from the reference's custom_dataset/)."""
import glob
import os

import numpy as np

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
SIZES = [(1, 1), (1, 17), (8, 8), (15, 17), (16, 16), (37, 53), (427, 640), (480, 640), (544, 1088), (1080, 1920)]
CONTENTS = ['noise', 'gradient', 'constant', 'checker']
QUALITIES = [95, 100, 50]


def synth(h, w, kind, seed=0):
    """uint8 BGR [h, w, 3]: uniform noise (long codes, 0xFF bytes), smooth gradients, a constant, a 0/255 checkerboard."""
    yy, xx = np.mgrid[:h, :w]
    if kind == 'noise':
        return np.random.default_rng(seed + 7 * h + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == 'gradient':
        return np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), (xx + 2 * yy) * 3 % 256], -1).astype(np.uint8)
    if kind == 'constant':
        return np.full((h, w, 3), (201, 37, 118), np.uint8)
    if kind == 'checker':
        return np.repeat(((yy + xx) % 2 * 255).astype(np.uint8)[..., None], 3, -1)
    raise ValueError(kind)


def photos():
    import cv2
    return [(os.path.basename(p)[:-4], cv2.imread(p)) for p in sorted(glob.glob(os.path.join(GOLDEN_DIR, '0*.jpg')))]


def corpus():
    """[(name, image)] in a fixed order."""
    out = [(f'{kind}_{h}x{w}', synth(h, w, kind)) for h, w in SIZES for kind in CONTENTS]
    return out + [(f'photo_{name}', img) for name, img in photos()]
