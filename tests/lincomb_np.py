"""numpy restatement of draw_lincomb (the reference's utils/output_utils.py:276-305, cfg.save_lincomb) as yb_draw_lincomb computes
it, and the cases its golden (tests/golden/lincomb.npz: the colour-table index of every pixel) and the GPU tests use.

For detection 0: the 32 prototype channels ordered by |coef| descending -- ties to the lower channel (a stable sort; the
reference's np.argsort is unstable there) -- cell i = 8r + c of a 4 x 8 grid shows channel ch = order[i] as
x = fp32(fp32(proto[..., ch] / max(proto[..., ch])) * coef[ch]), byte = ((double)x + 1) * 127.5 cast to uint8 as numpy does on
x86-64 (truncation to int32, low byte; NaN gives 0), and the pixel is COLORMAP_WINTER[byte]."""
import numpy as np

K = 32


def winter_lut():
    """uint8 [256,3]: cv2.applyColorMap on uint8 input is this table lookup."""
    import cv2
    return np.ascontiguousarray(cv2.applyColorMap(np.arange(256, dtype=np.uint8)[:, None], cv2.COLORMAP_WINTER)[:, 0])


def lincomb(proto, coef, lut):
    """proto float32 [P,P,32], coef float32 [D,32] (detection 0 is drawn), lut [256,3] -> uint8 [4P, 8P, 3]."""
    return lut[lincomb_bytes(proto, coef)]


def lincomb_bytes(proto, coef):
    """The colour-table index of every pixel: uint8 [4P, 8P]."""
    P = proto.shape[0]
    c0 = coef[0].astype(np.float32)
    order = np.argsort(-np.abs(c0), kind='stable')
    out = np.zeros((4 * P, 8 * P), np.uint8)
    for i, ch in enumerate(order):
        r, c = divmod(i, 8)
        plane = proto[:, :, ch].astype(np.float32)
        with np.errstate(all='ignore'):
            x = (plane / plane.max()) * c0[ch]
            u = (x.astype(np.float64) + 1.0) * 127.5
            ok = (u > -2147483649.0) & (u < 2147483648.0)
            t = np.where(ok, np.trunc(np.where(ok, u, 0.0)), -2.0 ** 31).astype(np.int64) & 255
        out[r * P:(r + 1) * P, c * P:(c + 1) * P] = t
    return out


def lut_index(img, lut):
    """Inverse of lut[...] on an image whose every pixel is a table entry (COLORMAP_WINTER's 256 entries are distinct)."""
    key = lambda a: (a[..., 0].astype(np.int64) << 16) | (a[..., 1].astype(np.int64) << 8) | a[..., 2]
    inv = np.full(1 << 24, -1, np.int64)
    inv[key(lut)] = np.arange(256)
    idx = inv[key(img)]
    assert (idx >= 0).all(), 'a pixel outside the colour table'
    return idx.astype(np.uint8)


# name -> (P, seed, kind).  kind: 'mixed' signed coefficients, 'neg' all negative, 'zero' one all-zero proto channel (0 / 0),
# 'tie' several coefficients of |coef| = 1.0 (saturated tanh): oracle and GPU only, the reference's order there is unstable.
CASES = {'p138_mixed': (138, 1, 'mixed'), 'p136_zero': (136, 2, 'zero'), 'p69_neg': (69, 3, 'neg'), 'p16_mixed': (16, 4, 'mixed'),
         'p16_tie': (16, 5, 'tie')}
ZERO_CHANNEL = 7


def case_inputs(name, D=3):
    """-> (proto float32 [P,P,32], coef float32 [D,32]) of a case: proto >= 0 as after the ProtoNet's ReLU -- smooth planes, as
    prototypes are, with a little noise so that every rounding step is exercised -- and coefficients in [-1, 1] as after tanh,
    with distinct magnitudes except in 'tie'.  Smooth planes keep the golden small."""
    P, seed, kind = CASES[name]
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:P, 0:P] / P
    f = rng.uniform(0.25, 1.0, size=(4, K))
    ph = rng.uniform(0, 2 * np.pi, size=(2, K))
    smooth = np.sin(2 * np.pi * (f[0] * xx[..., None] + f[1] * yy[..., None]) + ph[0]) + \
        np.cos(2 * np.pi * (f[2] * xx[..., None] - f[3] * yy[..., None]) + ph[1])
    proto = np.maximum(smooth + rng.normal(0, 0.004, size=(P, P, K)), 0).astype(np.float32)
    coef = np.tanh(rng.normal(0, 1.5, size=(D, K))).astype(np.float32)
    if kind == 'neg':
        coef = -np.abs(coef)
    elif kind == 'zero':
        proto[:, :, ZERO_CHANNEL] = 0
    elif kind == 'tie':
        coef[0, [3, 9, 10, 20, 31]] = [1.0, -1.0, 1.0, -1.0, 1.0]
        coef[0, [0, 1]] = [0.5, -0.5]
    return np.ascontiguousarray(proto), np.ascontiguousarray(coef)


def has_tie(coef):
    a = np.abs(coef[0])
    return len(np.unique(a)) != len(a)


GOLDEN_CASES = [n for n, (_, _, kind) in CASES.items() if kind != 'tie']
