"""numpy restatement of the reference's draw_img (utils/output_utils.py:308-369) (TEST INFRASTRUCTURE -- never imported by the
product package).

The mask overlay and the cutout matting are numpy; the box, label and fps pass is the reference's cv2 calls in the reference's
order.  The per-pixel class sum is accumulated one detection at a time, so 1080p inputs with 100 masks fit in memory.
`golden_cases()` builds the deterministic inputs of tests/golden/draw.npz from synthetic head outputs passed through
oracle/postprocess_np.nms / after_nms, plus hand-made rectangles for the modulo quirks.
"""
import types

import numpy as np

from . import postprocess_np as pp
from . import synth

F32 = np.float32


def semantic(ids, masks, num_colors):
    """(sum_i masks_i * (ids_i + 1)) % num_colors in int64 (output_utils.py:322-324); masks [n,h,w] with values {0,1}."""
    sem = np.zeros(masks.shape[1:], np.int64)
    for i in range(len(ids)):
        sem += (masks[i] != 0).astype(np.int64) * (int(ids[i]) + 1)
    return sem % num_colors


def blend(color, img):
    """cv2.addWeighted(color, 0.4, img, 0.6, 0) on uint8: fp32 products and sum, rounded to nearest even."""
    return np.rint(F32(0.4) * color.astype(F32) + F32(0.6) * img.astype(F32)).astype(np.uint8)


def overlay(img, ids, masks, num_classes, palette):
    return blend(palette[semantic(ids, masks, num_classes - 1)], img)


def cutout(img, ids, boxes, masks, num_classes):
    """total_obj and the per-detection crops (output_utils.py:328-341), as uint8 (the values the reference hands to imwrite)."""
    sem = semantic(ids, masks, num_classes - 1)
    total = np.where((sem != 0)[:, :, None], img, 255).astype(np.uint8)
    crops = []
    for i in range(len(ids)):
        x1, y1, x2, y2 = boxes[i, :]
        crops.append(np.where((masks[i] != 0)[:, :, None], img, 255).astype(np.uint8)[y1:y2, x1:x2, :])
    return total, crops


def draw(ids, scores, boxes, masks, img, cfg, palette, img_name=None, fps=None):
    """Returns (image, [(path, array) written by the cutout]).  The image is a new array unless hide_mask (then `img` itself,
    drawn in place, as the reference does) or ids is None (`img`)."""
    import cv2
    if ids is None:
        return img, []
    writes = []
    fused = img
    if not cfg.hide_mask:
        fused = overlay(img, ids, masks, cfg.num_classes, palette)
        if cfg.cutout:
            total, crops = cutout(img, ids, boxes, masks, cfg.num_classes)
            writes.append((f'results/images/{img_name}_total_obj.jpg', total))
            writes += [(f'results/images/{img_name}_{i}.jpg', c) for i, c in enumerate(crops)]
    scale, thickness, font = 0.6, 1, cv2.FONT_HERSHEY_DUPLEX
    if not cfg.hide_bbox:
        for i in reversed(range(ids.shape[0])):
            x1, y1, x2, y2 = (int(v) for v in boxes[i, :])
            color = palette[ids[i] + 1].tolist()
            cv2.rectangle(fused, (x1, y1), (x2, y2), color, thickness)
            class_name = cfg.class_names[ids[i]]
            text_str = f'{class_name}: {scores[i]:.2f}' if not cfg.hide_score else class_name
            text_w, text_h = cv2.getTextSize(text_str, font, scale, thickness)[0]
            cv2.rectangle(fused, (x1, y1), (x1 + text_w, y1 + text_h + 5), color, -1)
            cv2.putText(fused, text_str, (x1, y1 + 15), font, scale, (255, 255, 255), thickness, cv2.LINE_AA)
    if cfg.real_time:
        fps_str = f'fps: {fps:.2f}'
        text_w, text_h = cv2.getTextSize(fps_str, font, scale, thickness)[0]
        fused = fused.astype(np.float32)
        fused[0:text_h + 8, 0:text_w + 8] *= 0.6
        fused = fused.astype(np.uint8)
        cv2.putText(fused, fps_str, (0, text_h + 2), font, scale, (255, 255, 255), thickness, cv2.LINE_AA)
    return fused, writes


# ----------------------------------------------------------------------------- golden inputs
SIZES = ((96, 128), (128, 96), (37, 70))


def draw_cfg(num_classes=81, **opts):
    from yolact_minimal_b200.config import COCO_CLASSES, PASCAL_CLASSES
    names = COCO_CLASSES if num_classes == 81 else PASCAL_CLASSES
    assert len(names) == num_classes - 1
    c = dict(num_classes=num_classes, class_names=names, hide_mask=False, hide_bbox=False, hide_score=False, cutout=False,
             real_time=False)
    c.update(opts)
    return types.SimpleNamespace(**c)


def test_image(seed, h, w):
    """A smooth BGR uint8 image (compresses well, every channel value occurs)."""
    y, x = np.mgrid[0:h, 0:w]
    v = x[..., None] * (3 + seed) + y[..., None] * 5 + np.arange(3) * 77 + ((x * y) % 13)[..., None]
    return (v % 256).astype(np.uint8)


def rect_masks(rects, h, w):
    m = np.zeros((len(rects), h, w), F32)
    for i, (x1, y1, x2, y2) in enumerate(rects):
        m[i, max(y1, 0):max(y2, 0), max(x1, 0):max(x2, 0)] = 1
    return m


def detections(seed, h, w, many, num_classes):
    """after_nms outputs (ids int64, scores float32, boxes int32 [d,4], masks float32 [d,h,w]): the top 1 or 30 detections of
    synthetic head outputs, and with `many` three hand-made rectangles -- class num_classes-2 (which the modulo paints with
    colour 0), a repeated class, and a box past the right edge of the image."""
    S, P = 64, 16
    anchors = pp.make_anchors(S)
    cls, box, coef = synth.head_outputs(seed, len(anchors), num_classes=81)
    ids, scores, boxes, aidx = pp.nms(cls, box, anchors)
    k = 30 if many else 1
    # no_crop: the synthetic boxes are small, the uncropped masks cover large, overlapping areas
    ids, scores, boxes_px, masks = pp.after_nms(ids[:k], scores[:k], boxes[:k], coef[aidx[:k]], synth.proto(seed, P), h, w,
                                                no_crop=True)
    ids = ids % (num_classes - 1)
    if many:
        rects = [(2, 3, w // 2, h // 2), (w // 3, h // 4, w - 2, h - 5), (w // 2, h // 3, w + 17, h - 1)]
        ids = np.concatenate([ids, [num_classes - 2, ids[0], num_classes - 2]]).astype(np.int64)
        scores = np.concatenate([scores, F32([0.91, 0.42, 0.07])]).astype(F32)
        boxes_px = np.concatenate([boxes_px, np.asarray(rects, np.int32)]).astype(np.int32)
        masks = np.concatenate([masks, rect_masks(rects, h, w)])
    return ids.astype(np.int64), scores.astype(F32), boxes_px.astype(np.int32), masks.astype(F32)


def golden_cases():
    """[(name, seed, size index, many, num_classes, options, fps)]"""
    cases = []
    for s in range(len(SIZES)):
        cases.append((f's{s}_one', 10 + s, s, False, 81, {}, None))
        cases.append((f's{s}_many', 20 + s, s, True, 81, {}, None))
    cases += [('s0_many_nc21', 30, 0, True, 21, {}, None),
              ('s2_many_nc21', 31, 2, True, 21, {}, None),
              ('s0_many_hide_mask', 32, 0, True, 81, {'hide_mask': True}, None),
              ('s1_many_hide_bbox', 33, 1, True, 81, {'hide_bbox': True}, None),
              ('s2_many_hide_score', 34, 2, True, 81, {'hide_score': True}, None),
              ('s1_many_cutout', 35, 1, True, 81, {'cutout': True}, None),
              ('s2_one_cutout', 36, 2, False, 21, {'cutout': True}, None),
              ('s0_many_real_time', 37, 0, True, 81, {'real_time': True}, 23.456),
              ('s1_one_hide_mask_real_time', 38, 1, False, 81, {'hide_mask': True, 'real_time': True}, 7.0),
              ('s2_none', 39, 2, False, 81, {}, None)]
    return cases


def case_inputs(case):
    """(ids or None, scores, boxes, masks, img, cfg, img_name, fps) of a golden case."""
    name, seed, s, many, nc, opts, fps = case
    h, w = SIZES[s]
    img = test_image(seed, h, w)
    cfg = draw_cfg(nc, **opts)
    if name.endswith('_none'):
        return None, None, None, None, img, cfg, name, fps
    ids, scores, boxes, masks = detections(seed, h, w, many, nc)
    return ids, scores, boxes, masks, img, cfg, name, fps
