"""GPU: traditional NMS (`cfg.traditional_nms`: k_filter_decode<false> -> k_class_hard_nms -> k_final_topk) against the oracle
(oracle/postprocess_np.traditional_nms + hard_nms), bit for bit: count, class, anchor, score, box bits and coefficient rows of every
image, with `_check_image` of test_postprocess_gpu.

  * the full head sizes, batched: S = 550 (A = 19 248) and 544 (A = 18 525), B = 4 (stress, realistic, sparse and an image with no
    candidates), max_det in {1, 5, 100, 256} x iou_thr in {0, 0.5, 1}.  This is where the transposed score matrix, the A-float
    shared-memory score array and the batched grid are large;
  * score ties at the max_det cut.  The greedy loop visits tied scores larger anchor first (the reversed stable argsort of
    cython_nms), while the cross-class ranking (output_utils.py:115-117) keeps the SMALLER anchors of a tied group: a class with more
    than max_det survivors must keep its smallest tied anchors, however many ties there are;
  * tied boxes that overlap, where the greedy tie rule decides which box suppresses which;
  * the largest supported head (A = 49 152) runs, and A = 49 153 is refused before anything is launched or written.
"""
import ctypes

import numpy as np
import pytest
import torch

from cases import build_nms_inputs
from oracle import synth, postprocess_np as pp
from test_postprocess_gpu import _cfg, _run, _check_image

pytestmark = pytest.mark.gpu

MAX_DETS = (1, 5, 100, 256)
IOU_THRS = (0.0, 0.5, 1.0)


def _oracle(cls, box, anchors, S, iou_thr, max_det):
    return pp.nms(cls, box, anchors, iou_thre=iou_thr, max_det=max_det, traditional=True, img_size=S)


def _cut(o, max_det):
    """traditional_nms ranks ALL survivors and then takes [:max_det] (output_utils.py:115-117): one oracle run with an unbounded
    max_det serves every max_det."""
    return None if o is None else tuple(a[:max_det] for a in o)


def _check_batch(cuda, cls, box, coef, anchors, S, iou_thr, max_dets):
    oracle = [_oracle(cls[b], box[b], anchors, S, iou_thr, 10 ** 9) for b in range(cls.shape[0])]
    for md in max_dets:
        r = _run(cuda, cls, box, coef, anchors, _cfg(True, S=S, max_detections=md, nms_iou_thre=iou_thr))
        for b in range(cls.shape[0]):
            _check_image(r, b, _cut(oracle[b], md), coef[b])
    return oracle


@pytest.mark.parametrize('S', [550, 544])
@pytest.mark.parametrize('iou_thr', IOU_THRS)
def test_full_head_batched(cuda, S, iou_thr):
    anchors = pp.make_anchors(S)
    assert anchors.shape[0] == {550: 19248, 544: 18525}[S]
    items = [build_nms_inputs(S, reg, seed, None)[1:] for reg, seed in (('stress', 11), ('realistic', 12), ('sparse', 13), ('sparse', 14))]
    cls = np.stack([i[0] for i in items]); box = np.stack([i[1] for i in items]); coef = np.stack([i[2] for i in items])
    cls[3, :, 1:] = 0; cls[3, :, 0] = 1                     # no candidates in this image
    oracle = _check_batch(cuda, cls, box, coef, anchors, S, iou_thr, MAX_DETS)
    assert oracle[3] is None and all(o is not None for o in oracle[:3])
    if iou_thr == 0.5:
        assert len(oracle[0][0]) > 256                      # the stress image has more survivors than the largest max_det


def _background(A, C=81):
    cls = np.zeros((A, C), np.float32); cls[:, 0] = 1
    return cls


def test_tie_at_max_det_minimal(cuda):
    """Two far-apart boxes of class 5 tie at 0.9: with max_det = 1 the reference keeps the smaller anchor (10), not the one the
    greedy loop visits first (1013)."""
    S = 128
    anchors = pp.make_anchors(S)
    A = anchors.shape[0]
    cls = _background(A)
    cls[[10, 1013], 6] = 0.9; cls[[10, 1013], 0] = 0.1
    box = np.zeros((A, 4), np.float32)
    coef = synth.normal(41, 1, (A, 32)).astype(np.float32)
    o = _oracle(cls, box, anchors, S, 0.5, 10)
    assert list(o[3]) == [10, 1013] and list(o[0]) == [5, 5]
    for md in (1, 2):
        r = _run(cuda, cls[None], box[None], coef[None], anchors, _cfg(True, S=S, max_detections=md))
        _check_image(r, 0, _cut(o, md), coef)


def _far_apart_case(A=1024, seed=42):
    """Anchors on a 32 x 32 grid of small boxes that never overlap (pixel IoU 0 at S = 550, boxes 11 px apart).  Class 3: 7 boxes
    at 0.9, 300 at 0.75 (tied), 50 at 0.6; class 9: 40 boxes at 0.75 and 260 at 0.7 (tied).  The tied anchors are scattered over
    the index range, so which of them are the smallest is not their position in the greedy order."""
    g = (np.arange(A) % 32, np.arange(A) // 32)
    anchors = np.stack([(g[0] + 0.5) / 32, (g[1] + 0.5) / 32, np.full(A, 0.01), np.full(A, 0.01)], 1).astype(np.float32)
    perm = np.argsort(synth.uniform(seed, 1, (A,)))
    cls = _background(A)
    def put(idx, c, s):
        cls[idx, c] = s; cls[idx, 0] = 1 - s
    put(perm[:7], 4, 0.9); put(perm[7:307], 4, 0.75); put(perm[307:357], 4, 0.6)
    put(perm[400:440], 10, 0.75); put(perm[440:700], 10, 0.7)
    box = np.zeros((A, 4), np.float32)
    coef = synth.normal(seed, 2, (A, 32)).astype(np.float32)
    return anchors, cls, box, coef


def test_many_ties_beyond_max_det(cuda):
    """More tied survivors than max_det (and than the per-class storage): exactly the smallest tied anchors are kept."""
    S = 550
    anchors, cls, box, coef = _far_apart_case()
    o = _oracle(cls, box, anchors, S, 0.5, 10 ** 9)
    assert len(o[0]) == 657                                 # nothing overlaps: every candidate survives
    o100 = _cut(o, 100)                                     # the 7 boxes at 0.9, then the 93 smallest of class 3's tied anchors
    assert np.array_equal(o100[3][:7], np.nonzero(cls[:, 4] == np.float32(0.9))[0])
    assert np.array_equal(o100[3][7:], np.nonzero(cls[:, 4] == np.float32(0.75))[0][:93]) and (o100[0] == 3).all()
    for md in (1, 7, 8, 100, 256):
        for thr in (0.5, 1.0):
            r = _run(cuda, cls[None], box[None], coef[None], anchors, _cfg(True, S=S, max_detections=md, nms_iou_thre=thr))
            _check_image(r, 0, _cut(_oracle(cls, box, anchors, S, thr, 10 ** 9), md), coef)


def test_quantised_scores_full_head(cuda):
    """Scores quantised to 1/16 at the full head size: large tied groups in every class, at every cut."""
    S = 550
    anchors = pp.make_anchors(S)
    items = [build_nms_inputs(S, reg, seed, None)[1:] for reg, seed in (('stress', 21), ('realistic', 22))]
    cls = np.stack([(np.round(i[0] * 16) / 16).astype(np.float32) for i in items])
    box = np.stack([i[1] for i in items]); coef = np.stack([i[2] for i in items])
    _check_batch(cuda, cls, box, coef, anchors, S, 0.5, (1, 5, 100))


def _overlap_ties_case():
    """Clusters of equal-score boxes that overlap, in one class.  Pairs (a < b, pixel IoU 0.82): the greedy loop keeps b and
    suppresses a.  Triples (a < b < c): c's box lies between a's and b's, IoU(c, a) = IoU(c, b) = 0.6 and IoU(a, b) = 0.33, so c
    suppresses both (visiting a first would keep a and b).  Every cluster has its own score."""
    S, A = 550, 2048
    rng = np.random.default_rng(7)
    anchors = np.zeros((A, 4), np.float32)
    anchors[:] = [0.5, 0.5, 0.001, 0.001]
    cls = _background(A)
    free = rng.permutation(A)
    k = 0
    for cl in range(24):
        cx, cy = 0.06 + 0.08 * (cl % 12), 0.2 + 0.5 * (cl // 12)
        sc = np.float32(0.9 - 0.02 * cl)
        if cl % 2 == 0:
            ids = np.sort(free[k:k + 2]); k += 2
            anchors[ids[0]] = [cx, cy, 0.05, 0.05]
            anchors[ids[1]] = [cx + 0.005, cy, 0.05, 0.05]
        else:
            ids = np.sort(free[k:k + 3]); k += 3
            anchors[ids[0]] = [cx - 0.008, cy, 0.03, 0.03]
            anchors[ids[1]] = [cx + 0.008, cy, 0.03, 0.03]
            anchors[ids[2]] = [cx, cy, 0.03, 0.03]
        cls[ids, 8] = sc; cls[ids, 0] = 1 - sc
    box = np.zeros((A, 4), np.float32)
    coef = synth.normal(8, 1, (A, 32)).astype(np.float32)
    return S, anchors, cls, box, coef


def test_tied_overlapping_boxes(cuda):
    S, anchors, cls, box, coef = _overlap_ties_case()
    o = _oracle(cls, box, anchors, S, 0.5, 10 ** 9)
    assert len(o[0]) == 12 * 1 + 12 * 1                     # one box per pair, and only the middle box of each triple
    for md in (1, 5, 12, 100):
        r = _run(cuda, cls[None], box[None], coef[None], anchors, _cfg(True, S=S, max_detections=md))
        _check_image(r, 0, _cut(o, md), coef)


def _raw_detect(cuda, cls, box, coef, anchors, S, fill, max_det=100, traditional=1):
    """yb_detect with output and workspace buffers the caller owns, pre-filled with `fill` bytes."""
    from yolact_minimal_b200 import _lib
    B, A, C = cls.shape
    K, D = coef.shape[-1], max_det
    p = _lib.DetectParams(0.05, 0.5, 200, D, C, K, traditional, float(S), 0)
    L = _lib.lib()
    nbytes = int(L.yb_detect_workspace_bytes(B, A, ctypes.byref(p)))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    dcls, dbox, dcoef, danc = t(cls), t(box), t(coef), t(anchors)
    ws = torch.full((nbytes,), fill, dtype=torch.uint8, device=cuda)
    out = {k: torch.full((n,), fill, dtype=torch.uint8, device=cuda)
           for k, n in (('count', B * 4), ('cls', B * D * 4), ('anchor', B * D * 4), ('score', B * D * 4), ('box', B * D * 16),
                        ('coef', B * D * K * 4))}
    st = L.yb_detect(dcls.data_ptr(), dbox.data_ptr(), dcoef.data_ptr(), danc.data_ptr(), B, A, ctypes.byref(p), ws.data_ptr(), nbytes,
                     *(out[k].data_ptr() for k in ('count', 'cls', 'anchor', 'score', 'box', 'coef')), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return st, ws, out


def test_largest_head_and_refusal(cuda):
    """A = 49 152 (the A-float score array fills 192 KiB of shared memory) equals the oracle; A = 49 153 returns
    YB_ERR_UNSUPPORTED and writes nothing, neither the outputs nor the workspace."""
    from yolact_minimal_b200 import _lib
    S = 550
    for A in (49152, 49153):
        u = synth.uniform(51, 1, (A, 4))
        anchors = np.stack([u[:, 0], u[:, 1], 0.02 + 0.2 * u[:, 2], 0.02 + 0.2 * u[:, 3]], 1).astype(np.float32)
        cls, box, coef = synth.head_outputs(51, A, 81, 'sparse')
        if A == 49152:
            r = _run(cuda, cls[None], box[None], coef[None], anchors, _cfg(True, S=S))
            o = _oracle(cls, box, anchors, S, 0.5, 100)
            assert o is not None and len(o[0]) > 20
            _check_image(r, 0, o, coef)
        else:
            st, ws, out = _raw_detect(cuda, cls[None], box[None], coef[None], anchors, S, 0xA5)
            assert st == -3 and b'num_anchors' in _lib.lib().yb_last_error()
            assert bool((ws == 0xA5).all())
            for k, v in out.items():
                assert bool((v == 0xA5).all()), k
