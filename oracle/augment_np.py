"""numpy restatement of train_aug's pixel path (utils/augmentations.py:230-252) given a host plan
(yolact_minimal_b200.utils.augmentations.TrainAugPlan) -- the oracle of yb_train_aug (TEST INFRASTRUCTURE).

Stage by stage as the reference runs them: photometric_distort on the whole float32 image (cv2's float
BGR<->HSV formulas), mirror, crop, pad_to_square, cv2.resize INTER_LINEAR, to_train_size, normalise.
The resize follows OpenCV's resizeGeneric_: x taps clamped at the borders with weight 0 outside, y rows
clipped with the weights kept; float32 arithmetic for images and padded masks, and for masks that stay uint8
the 11-bit fixed-point weights with the rounding of OpenCV's vectorised vertical pass."""
import numpy as np

F32 = np.float32
FLT_EPSILON = F32(np.finfo(np.float32).eps)
NORM_MEAN = np.array([103.94, 116.78, 123.68], dtype=F32)     # BGR, config.py:66
NORM_STD = np.array([57.38, 57.12, 58.40], dtype=F32)         # config.py:67


def bgr2hsv(img):
    """cv2.cvtColor(float32 BGR, COLOR_BGR2HSV): H in [0,360), S = (V-min)/(V+eps), V = max."""
    b, g, r = (img[..., k].astype(F32) for k in range(3))
    v = np.maximum(np.maximum(r, g), b)
    vmin = np.minimum(np.minimum(r, g), b)
    diff = (v - vmin).astype(F32)
    s = (diff / (np.abs(v) + FLT_EPSILON)).astype(F32)
    rdiff = (F32(60) / (diff + FLT_EPSILON)).astype(F32)
    h = np.where(v == r, (g - b) * rdiff, np.where(v == g, (b - r) * rdiff + F32(120), (r - g) * rdiff + F32(240))).astype(F32)
    h = np.where(h < 0, h + F32(360), h).astype(F32)
    return np.stack([h, s, v], axis=-1)


def hsv2bgr(hsv):
    """cv2.cvtColor(float32 HSV, COLOR_HSV2BGR) for H in [0,360]; S > 1 gives negative channels (not clipped here)."""
    h, s, v = (hsv[..., k].astype(F32) for k in range(3))
    h = (h * F32(6.0 / 360.0)).astype(F32)
    h = np.where(h >= 6, h - F32(6), h).astype(F32)
    sector = np.floor(h).astype(np.int64)
    h = (h - sector.astype(F32)).astype(F32)
    bad = (sector < 0) | (sector >= 6)
    sector[bad] = 0
    h[bad] = 0
    one = F32(1)
    tab = np.stack([v, v * (one - s), v * (one - s * h), v * (one - s * (one - h))], axis=-1).astype(F32)
    sel = np.array([[1, 3, 0], [1, 0, 2], [3, 0, 1], [0, 2, 1], [0, 1, 3], [2, 1, 0]])[sector]
    out = np.take_along_axis(tab, sel, axis=-1)
    return np.where((s == 0)[..., None], v[..., None], out).astype(F32)


def photometric(img_u8, plan):
    img = img_u8.astype(F32)
    if plan.brightness is not None:
        img = np.clip(img + F32(plan.brightness), 0, 255).astype(F32)
    if plan.contrast is not None:
        img = np.clip(img * F32(plan.contrast), 0, 255).astype(F32)
    hsv = bgr2hsv(img)
    hsv[..., 1] *= F32(plan.saturation)
    hsv[..., 0] += F32(plan.hue)
    hsv[..., 0][hsv[..., 0] > 360] -= F32(360)
    hsv[..., 0][hsv[..., 0] < 0] += F32(360)
    return np.clip(hsv2bgr(hsv), 0, 255).astype(F32)


def _axis(src, dst, y_rule):
    scale = 1.0 / (float(dst) / float(src))
    d = np.arange(dst, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(F32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(F32)).astype(F32)
    if y_rule:
        s0, s1 = np.clip(s, 0, src - 1), np.clip(s + 1, 0, src - 1)
    else:
        lo = s < 0
        s[lo] = 0; f[lo] = 0
        hi = s >= src - 1
        s[hi] = src - 1; f[hi] = 0
        s0, s1 = s, np.minimum(s + 1, src - 1)
    a0, a1 = (F32(1) - f).astype(F32), f
    return s0, s1, a0, a1


def resize_f32(x, dst):
    """cv2.resize(x [P,P,C] float32, (dst,dst)) INTER_LINEAR: horizontal pass, then vertical."""
    P = x.shape[0]
    x0, x1, ax0, ax1 = _axis(P, dst, False)
    y0, y1, ay0, ay1 = _axis(P, dst, True)
    rows0 = (x[y0][:, x0] * ax0[None, :, None] + x[y0][:, x1] * ax1[None, :, None]).astype(F32)
    rows1 = (x[y1][:, x0] * ax0[None, :, None] + x[y1][:, x1] * ax1[None, :, None]).astype(F32)
    return (rows0 * ay0[:, None, None] + rows1 * ay1[:, None, None]).astype(F32)


def resize_u8(x, dst):
    """cv2.resize(x [P,P,C] uint8, (dst,dst)) INTER_LINEAR: 11-bit weights rounded to nearest; exact int horizontal pass;
    vertical pass as VResizeLinearVec_32s8u rounds it: (((h0>>4)*b0>>16) + ((h1>>4)*b1>>16) + 2) >> 2."""
    P = x.shape[0]
    fx = lambda a: np.rint(a * F32(2048)).astype(np.int64)
    x0, x1, ax0, ax1 = _axis(P, dst, False)
    y0, y1, ay0, ay1 = _axis(P, dst, True)
    ax0, ax1, ay0, ay1 = fx(ax0), fx(ax1), fx(ay0), fx(ay1)
    xi = x.astype(np.int64)
    h0 = xi[y0][:, x0] * ax0[None, :, None] + xi[y0][:, x1] * ax1[None, :, None]
    h1 = xi[y1][:, x0] * ax0[None, :, None] + xi[y1][:, x1] * ax1[None, :, None]
    t = (((h0 >> 4) * ay0[:, None, None]) >> 16) + (((h1 >> 4) * ay1[:, None, None]) >> 16)
    return np.clip((t + 2) >> 2, 0, 255).astype(np.uint8)


def train_aug_pixels(img_u8, masks_u8, plan):
    """img_u8 [h,w,3] BGR, masks_u8 [n,h,w] -> (img float32 [3,S,S] RGB normalised, masks float32 [len(keep),S,S])."""
    img = photometric(img_u8, plan)
    masks = masks_u8[plan.keep]
    if plan.mirror:
        img, masks = img[:, ::-1], masks[:, :, ::-1]
    cx, cy, cw, ch = plan.crop
    img, masks = img[cy:cy + ch, cx:cx + cw], masks[:, cy:cy + ch, cx:cx + cw]
    P = plan.square
    if ch != cw:
        px, py = plan.pad
        pimg = np.empty((P, P, 3), F32)
        pimg[:] = NORM_MEAN
        pimg[py:py + ch, px:px + cw] = img
        pm = np.zeros((masks.shape[0], P, P), F32)
        pm[:, py:py + ch, px:px + cw] = masks
        img, masks = pimg, pm
    rs, S = plan.resize, plan.train_size
    img = resize_f32(np.ascontiguousarray(img), rs)
    mt = np.ascontiguousarray(masks.transpose(1, 2, 0))
    masks = (resize_u8(mt, rs) if plan.mask_u8 else resize_f32(mt, rs)).transpose(2, 0, 1).astype(F32)
    tx, ty = plan.train_off
    if rs < S:
        pimg = np.empty((S, S, 3), F32)
        pimg[:] = NORM_MEAN
        pimg[ty:ty + rs, tx:tx + rs] = img
        pm = np.zeros((masks.shape[0], S, S), F32)
        pm[:, ty:ty + rs, tx:tx + rs] = masks
        img, masks = pimg, pm
    elif rs > S:
        img, masks = img[ty:ty + S, tx:tx + S], masks[:, ty:ty + S, tx:tx + S]
    img = ((img - NORM_MEAN) / NORM_STD).astype(F32)
    return np.ascontiguousarray(img[:, :, ::-1].transpose(2, 0, 1)), np.ascontiguousarray(masks)


# ----------------------------------------------------------------------------- synthetic COCO-like samples
def synthetic_sample(seed, h, w, n, kind='normal'):
    """A deterministic uint8 BGR image [h,w,3], n elliptical uint8 masks [n,h,w], their float64 x1y1x2y2 boxes and
    int64 labels.  kind 'tiny' makes every other box 3-5 px wide (removed by remove_small_box after the resize);
    'zero' makes every box zero-width (no crop window can keep one)."""
    from oracle import synth
    img = (synth.uniform(seed, 41, (h, w, 3)) * 256).astype(np.uint8)
    # smooth regions so that the photometric transform sees greys, saturated and dark pixels
    yy, xx = np.mgrid[0:h, 0:w]
    img[(yy // 37 + xx // 53) % 5 == 0] = (synth.uniform(seed, 42, (1,)) * 256).astype(np.uint8)[0]
    img[(yy // 41 + xx // 29) % 7 == 0] = 0
    u = synth.uniform(seed, 43, (n, 4))
    bw = np.maximum(4.0, u[:, 2] * w * 0.6)
    bh = np.maximum(4.0, u[:, 3] * h * 0.6)
    if kind == 'tiny':
        bw[::2] = 3 + np.floor(u[::2, 2] * 3)
        bh[::2] = 3 + np.floor(u[::2, 3] * 3)
    x1 = np.floor(u[:, 0] * (w - bw) * 4) / 4
    y1 = np.floor(u[:, 1] * (h - bh) * 4) / 4
    boxes = np.stack([x1, y1, x1 + bw, y1 + bh], axis=1).astype(np.float64)
    if kind == 'zero':
        boxes[:, 2] = boxes[:, 0]
    masks = np.zeros((n, h, w), np.uint8)
    for j in range(n):
        cx, cy = (boxes[j, 0] + boxes[j, 2]) / 2, (boxes[j, 1] + boxes[j, 3]) / 2
        rx, ry = max((boxes[j, 2] - boxes[j, 0]) / 2, 0.5), max((boxes[j, 3] - boxes[j, 1]) / 2, 0.5)
        masks[j] = (((xx + 0.5 - cx) / rx) ** 2 + ((yy + 0.5 - cy) / ry) ** 2 <= 1).astype(np.uint8)
    labels = np.floor(synth.uniform(seed, 44, (n,)) * 80).astype(np.int64)
    return img, masks, boxes, labels


def hsv_triples(seed, n):
    """float32 BGR triples in [0,255] (a quarter grey, some with v = 0) with per-triple saturation scales in
    [0.7,1.3] and hue shifts in [-15,15] (float32), for the cvtColor round trip."""
    from oracle import synth
    bgr = (synth.uniform(seed, 51, (n, 3)) * 255).astype(F32)
    grey = synth.uniform(seed, 52, (n,)) < 0.25
    bgr[grey] = bgr[grey, :1]
    bgr[synth.uniform(seed, 53, (n,)) < 0.02] = 0
    sat = (0.7 + 0.6 * synth.uniform(seed, 54, (n,))).astype(F32)
    hue = (-15 + 30 * synth.uniform(seed, 55, (n,))).astype(F32)
    return bgr, sat, hue


def hsv_round_trip(bgr, sat, hue):
    hsv = bgr2hsv(bgr)
    hsv[:, 1] *= sat
    hsv[:, 0] += hue
    hsv[:, 0][hsv[:, 0] > 360] -= F32(360)
    hsv[:, 0][hsv[:, 0] < 0] += F32(360)
    return hsv2bgr(hsv)
