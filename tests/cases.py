"""Shared synthetic post-process cases: the same construction as tests/golden/make_golden.py
(kept in sync by test_oracle_golden.py, which replays every golden through the oracle)."""
import numpy as np

from oracle import synth, postprocess_np as pp


def nms_cases():
    cases = []
    for S in (128, 256):
        for regime in ('stress', 'realistic', 'sparse'):
            for seed in (1, 2):
                cases.append((f'{regime}_S{S}_s{seed}', S, regime, seed, None))
    cases.append(('stress_S544_s1', 544, 'stress', 1, None))
    cases.append(('realistic_S544_s1', 544, 'realistic', 1, None))
    cases.append(('realistic_S550_s3', 550, 'realistic', 3, None))
    for mut in ('dup_boxes', 'zero_area', 'few', 'none', 'one'):
        cases.append((f'adv_{mut}', 128, 'stress', 7, mut))
    return cases


def build_nms_inputs(S, regime, seed, mut, num_classes=81):
    anchors = pp.make_anchors(S)
    A = anchors.shape[0]
    cls, box, coef = synth.head_outputs(seed, A, num_classes, regime)
    if mut == 'dup_boxes':
        box[1::2] = box[0::2][:box[1::2].shape[0]]
        anchors = anchors.copy(); anchors[1::2] = anchors[0::2][:anchors[1::2].shape[0]]
    elif mut == 'zero_area':
        box[:, :2] += 40.0
    elif mut in ('few', 'none', 'one'):
        keep_n = {'few': 37, 'none': 0, 'one': 1}[mut]
        cls[:] = 0.0; cls[:, 0] = 1.0
        src, _, _ = synth.head_outputs(seed + 1, A, num_classes, 'stress')
        rows = (np.arange(keep_n) * 23 + 5) % A
        cls[rows] = src[rows]
    return anchors, cls, box, coef


def tie_case(seed=3, S=128):
    """Deliberate exact score ties (quantised scores) and duplicate boxes: exercises the
    tie-break rules (score desc, then anchor asc within a class, class-major across classes)."""
    anchors, cls, box, coef = build_nms_inputs(S, 'stress', seed, None)
    cls = (np.round(cls * 16) / 16).astype(np.float32)
    return anchors, cls, box, coef
