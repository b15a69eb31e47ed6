#!/usr/bin/env python
"""train_aug golden generator (TEST INFRASTRUCTURE).  Runs only where a read-only checkout of the reference is
named by $YOLACT_REFERENCE and cv2 is installed; the fixture it writes next to this file (train_aug.npz) is
committed, and the tests need nothing else.

  YOLACT_REFERENCE=... python tests/golden/make_golden_train_aug.py

Each case runs the UNMODIFIED reference utils/augmentations.py train_aug on a synthetic sample from
oracle/augment_np.synthetic_sample under random.seed(seed), and stores its boxes, labels, surviving mask indices (from a second run on index-tagged masks), subsampled pixels,
per-mask and per-channel sums and the `random` state after the call.  The oracle (oracle/augment_np.py, fed the
host planner's plan) is compared with it here, and the max errors are printed and stored as the bounds.
A cvtColor section stores cv2's float BGR->HSV->(scale S, shift H)->BGR round trip on 2^18 triples.
"""
import os
import random
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ['YOLACT_REFERENCE']
sys.path.insert(0, ROOT)

from oracle import augment_np as an  # noqa: E402
from yolact_minimal_b200.utils.augmentations import train_aug_plan  # noqa: E402

# (name, h, w, n instances, kind, S, seeds)
CASES = [
    ('wide', 480, 640, 7, 'normal', 550, range(0, 12)),
    ('tall', 640, 427, 5, 'normal', 550, range(100, 112)),
    ('square', 640, 640, 3, 'normal', 550, range(200, 212)),
    ('s544', 427, 640, 4, 'normal', 544, range(300, 316)),
    ('one', 480, 640, 1, 'normal', 550, range(400, 406)),
    ('many', 480, 640, 60, 'normal', 550, range(500, 503)),
    ('tiny', 480, 640, 12, 'tiny', 550, range(600, 606)),
    ('zero', 300, 400, 2, 'zero', 550, range(700, 706)),
]
SUB = 23


def sample_seed(name):
    return 1 + [c[0] for c in CASES].index(name)


def import_reference():
    scratch = '/tmp/yolact_ref_cwd'
    os.makedirs(scratch, exist_ok=True)
    os.chdir(scratch)                      # config.py mkdirs in CWD on import
    sys.path.insert(0, REF)
    from utils.augmentations import train_aug
    return train_aug


def main():
    import cv2
    ref_train_aug = import_reference()
    out, img_err, mask_err = {}, 0.0, 0.0
    seen = set()
    for name, h, w, n, kind, S, seeds in CASES:
        img, masks, boxes, labels = an.synthetic_sample(sample_seed(name), h, w, n, kind)
        for seed in seeds:
            key = f'{name}/{seed}'
            random.seed(seed)
            r_img, r_masks, r_boxes, r_labels = ref_train_aug(img.copy(), masks.copy(), boxes.copy(), labels.copy(), S)
            state = np.asarray(random.getstate()[1], dtype=np.int64)
            random.seed(seed)
            plan = train_aug_plan(h, w, boxes, labels, S)
            assert np.array_equal(np.asarray(random.getstate()[1], dtype=np.int64), state), key
            out[key + '/state'] = state
            if r_img is None:
                assert plan is None, key
                out[key + '/none'] = np.int64(1)
                seen.add('none')
                continue
            assert plan is not None, key
            r_img = r_img.astype(np.float32)
            r_masks = np.asarray(r_masks).astype(np.float32)
            assert np.array_equal(plan.boxes, r_boxes) and np.array_equal(plan.labels, r_labels.astype(np.float64)), key
            # which source masks survive, in output order: the same draws on masks tagged with their index + 1 (the draws
            # never look at pixels, so the run repeats the geometry); each output mask's peak is its tag
            random.seed(seed)
            tagged = np.broadcast_to(np.arange(1, n + 1, dtype=np.uint8)[:, None, None], masks.shape).copy()
            t_out = ref_train_aug(img.copy(), tagged, boxes.copy(), labels.copy(), S)
            assert np.array_equal(np.asarray(random.getstate()[1], dtype=np.int64), state), key
            ref_keep = np.rint(np.asarray(t_out[1]).reshape(len(r_boxes), -1).max(axis=1)).astype(np.int64) - 1
            assert np.array_equal(plan.keep, ref_keep), (key, plan.keep, ref_keep)
            out[key + '/keep'] = ref_keep
            o_img, o_masks = an.train_aug_pixels(img, masks, plan)
            ei, em = float(np.abs(o_img - r_img).max()), float(np.abs(o_masks - r_masks).max())
            img_err, mask_err = max(img_err, ei), max(mask_err, em)
            if plan.mask_u8:
                assert em == 0, (key, em)
            seen.update({'crop' if plan.crop[2:] != (w, h) else 'nocrop', 'mirror' if plan.mirror else 'nomirror',
                         'u8' if plan.mask_u8 else 'f32', 'ttspad' if plan.resize < S else ('ttscrop' if plan.resize > S else 'ttseq'),
                         'tinydrop' if kind == 'tiny' and len(plan.keep) < n else 'x'})
            out[key + '/none'] = np.int64(0)
            out[key + '/boxes'] = r_boxes.astype(np.float64)
            out[key + '/labels'] = r_labels.astype(np.float64)
            out[key + '/img_sub'] = r_img[:, ::SUB, ::SUB]
            out[key + '/img_sum'] = r_img.astype(np.float64).sum(axis=(1, 2))
            out[key + '/mask_sum'] = r_masks.astype(np.float64).sum(axis=(1, 2))
            out[key + '/mask_sub'] = r_masks[:, ::SUB, ::SUB]
            print(f'  train_aug {key}: n={len(plan.keep)} crop={plan.crop} P={plan.square} rs={plan.resize} u8={plan.mask_u8} '
                  f'oracle-vs-reference max err img {ei:.2e} masks {em:.2e}')
    for must in ('none', 'crop', 'nocrop', 'mirror', 'nomirror', 'u8', 'f32', 'ttspad', 'ttscrop', 'ttseq', 'tinydrop'):
        assert must in seen, must
    out['cases'] = np.array([f'{c[0]}:{c[1]}:{c[2]}:{c[3]}:{c[4]}:{c[5]}:{c[6].start}:{c[6].stop}' for c in CASES])
    out['img_err'] = np.float64(img_err)
    out['mask_err'] = np.float64(mask_err)
    print(f'  train_aug: oracle-vs-reference max err img {img_err:.2e} (normalised) masks {mask_err:.2e}')

    # cvtColor round trip: cv2 on 2^18 triples
    bgr, sat, hue = an.hsv_triples(7, 1 << 18)
    hsv = cv2.cvtColor(bgr.reshape(-1, 1, 3), cv2.COLOR_BGR2HSV).reshape(-1, 3)
    hsv[:, 1] *= sat
    hsv[:, 0] += hue
    hsv[:, 0][hsv[:, 0] > 360.0] -= 360.0
    hsv[:, 0][hsv[:, 0] < 0.0] += 360.0
    ref = cv2.cvtColor(hsv.reshape(-1, 1, 3), cv2.COLOR_HSV2BGR).reshape(-1, 3)
    mine = an.hsv_round_trip(bgr, sat, hue)
    err = float(np.abs(ref - mine).max())
    out['hsv/sub'] = ref[::8]
    out['hsv/err'] = np.float64(err)
    print(f'  cvtColor round trip: {len(bgr)} triples, {int((ref < 0).any(axis=1).sum())} with a negative channel, '
          f'oracle-vs-reference max err {err:.2e}')
    np.savez_compressed(os.path.join(HERE, 'train_aug.npz'), **out)


if __name__ == '__main__':
    main()
