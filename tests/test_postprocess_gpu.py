"""GPU parity: CUDA post-process (through the C ABI, via the ctypes shims) vs the oracle and
the golden vectors minted from the reference.  Index/class/score/coef comparisons are
bit-exact; boxes are bit-exact vs the oracle (same correctly-rounded exp) and within 1 ulp of
the reference goldens (SLEEF expf)."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden
from cases import nms_cases, build_nms_inputs, tie_case
from oracle import synth, postprocess_np as pp

pytestmark = pytest.mark.gpu


def _cfg(traditional=False, S=544, classes='res101_coco', **kw):
    """classes: a config name, or a class count (background included) for res101_coco's settings at that count."""
    from yolact_minimal_b200.config import make_config
    cfg = make_config('res101_coco' if isinstance(classes, int) else classes, S, traditional_nms=traditional)
    if isinstance(classes, int):
        cfg.num_classes = classes
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def _run(cuda, cls, box, coef, anchors, cfg):
    from yolact_minimal_b200.utils.output_utils import detect_batched
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    r = detect_batched(t(cls), t(box), t(coef), t(anchors), cfg)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in r.items() if not k.startswith('_')}


def _check_image(r, b, o, coef):
    d = int(r['count'][b])
    if o is None:
        assert d == 0
        return
    ids, scores, boxes, aidx = o
    assert d == len(ids)
    assert np.array_equal(r['cls'][b, :d], ids)
    assert np.array_equal(r['anchor'][b, :d], aidx)
    assert np.array_equal(r['score'][b, :d], scores)
    assert np.array_equal(r['box'][b, :d].view(np.uint32), boxes.view(np.uint32)), np.abs(r['box'][b, :d] - boxes).max()
    assert np.array_equal(r['coef'][b, :d], coef[aidx])
    assert not r['score'][b, d:].any() and not r['box'][b, d:].any()


@pytest.mark.parametrize('case', nms_cases(), ids=lambda c: c[0])
def test_fast_nms_vs_oracle_and_golden(cuda, case):
    name, S, regime, seed, mut = case
    anchors, cls, box, coef = build_nms_inputs(S, regime, seed, mut)
    r = _run(cuda, cls[None], box[None], coef[None], anchors, _cfg(S=S))
    _check_image(r, 0, pp.nms(cls, box, anchors), coef)
    g = load_golden('postprocess.npz')
    key = f'{name}/fast'
    d = int(g[key + '/count'])
    assert int(r['count'][0]) == d
    if d:
        assert np.array_equal(r['cls'][0, :d], g[key + '/class'])
        assert np.array_equal(r['anchor'][0, :d], g[key + '/anchor'])          # indices bit-exact vs the reference
        assert np.array_equal(r['score'][0, :d], g[key + '/score'])
        assert np.allclose(r['box'][0, :d], g[key + '/box'], rtol=0, atol=2.4e-7)


@pytest.mark.parametrize('case', [c for c in nms_cases() if c[1] <= 256], ids=lambda c: c[0])
def test_traditional_nms_vs_oracle_and_golden(cuda, case):
    name, S, regime, seed, mut = case
    anchors, cls, box, coef = build_nms_inputs(S, regime, seed, mut)
    r = _run(cuda, cls[None], box[None], coef[None], anchors, _cfg(True, S=S))
    _check_image(r, 0, pp.nms(cls, box, anchors, traditional=True, img_size=S), coef)
    g = load_golden('postprocess.npz')
    key = f'{name}/trad'
    if key + '/count' in g and int(g[key + '/count']):
        d = int(g[key + '/count'])
        assert np.array_equal(r['cls'][0, :d], g[key + '/class'])
        assert np.array_equal(r['anchor'][0, :d], g[key + '/anchor'])


def test_batched_mixed_regimes(cuda):
    S = 256
    items = [build_nms_inputs(S, reg, seed, None) for reg, seed in
             (('stress', 1), ('sparse', 2), ('realistic', 3), ('stress', 4), ('realistic', 5))]
    anchors = items[0][0]
    cls = np.stack([i[1] for i in items]); box = np.stack([i[2] for i in items]); coef = np.stack([i[3] for i in items])
    cls[1, :, 1:] = 0; cls[1, :, 0] = 1                      # an image with no candidates inside the batch
    r = _run(cuda, cls, box, coef, anchors, _cfg(S=S))
    for b in range(len(items)):
        _check_image(r, b, pp.nms(cls[b], box[b], anchors), coef[b])


def test_ties_and_small_topk(cuda):
    anchors, cls, box, coef = tie_case()
    for top_k, max_det in ((200, 100), (7, 5), (256, 256), (1, 1)):
        cfg = _cfg(S=128, top_k=top_k, max_detections=max_det)
        r = _run(cuda, cls[None], box[None], coef[None], anchors, cfg)
        _check_image(r, 0, pp.nms(cls, box, anchors, top_k=top_k, max_det=max_det), coef)
    for thr in (0.0, 0.3, 1.0):
        cfg = _cfg(S=128, nms_iou_thre=thr)
        r = _run(cuda, cls[None], box[None], coef[None], anchors, cfg)
        _check_image(r, 0, pp.nms(cls, box, anchors, iou_thre=thr), coef)


def test_full_size_batch_properties(cuda):
    """BASELINE size (A=19248, 81 classes), B=8: two images checked against the oracle, all
    images against size-independent properties (sorted scores, determinism, permutation
    invariance of the batch order)."""
    S, B = 550, 8
    anchors = pp.make_anchors(S)
    A = anchors.shape[0]
    assert A == 19248
    regs = ['stress', 'realistic', 'sparse', 'stress', 'realistic', 'stress', 'sparse', 'realistic']
    data = [synth.head_outputs(100 + b, A, 81, regs[b]) for b in range(B)]
    cls = np.stack([d[0] for d in data]); box = np.stack([d[1] for d in data]); coef = np.stack([d[2] for d in data])
    cfg = _cfg(S=S)
    r = _run(cuda, cls, box, coef, anchors, cfg)
    for b in (0, 1):
        _check_image(r, b, pp.nms(cls[b], box[b], anchors), coef[b])
    for b in range(B):
        d = int(r['count'][b])
        assert 0 < d <= 100
        s = r['score'][b, :d]
        assert np.all(s[:-1] >= s[1:])
        assert np.array_equal(cls[b, r['anchor'][b, :d], r['cls'][b, :d] + 1], s)       # score == cls[anchor, class]
        assert np.all((r['box'][b, :d] >= 0) & (r['box'][b, :d] <= 1))
    r2 = _run(cuda, cls, box, coef, anchors, cfg)
    for k in r:
        assert np.array_equal(r[k], r2[k]), k                                            # deterministic
    perm = np.arange(B)[::-1].copy()
    r3 = _run(cuda, cls[perm], box[perm], coef[perm], anchors, cfg)
    for k in r:
        assert np.array_equal(r[k][perm], r3[k]), k                                      # images independent


def test_sampled_cuts_cannot_change_the_result(cuda):
    """The per-class candidate lists are filled from SAMPLED score cuts (k_sample_cuts reads the anchors floor(t*A/512));
    exactness must not depend on the sample.  Adversarial images at the full head size: (0) the sampled anchors carry the high
    scores of some classes and everything else is low -> the cut is too high, the list holds < top_k entries; (1) the sampled
    anchors are low and > 2048 other anchors are high -> the list overflows; (2) > 2048 exactly tied scores at the top of a
    class; (3) sampled anchors are not candidates at all (the image looks empty to the sample).  All four must take the exact
    full-column path and equal the oracle bit for bit."""
    S = 550
    anchors = pp.make_anchors(S)
    A = anchors.shape[0]
    sampled = np.unique((np.arange(512, dtype=np.int64) * A) // 512)
    others = np.setdiff1d(np.arange(A), sampled)
    rng = np.random.default_rng(77)
    imgs = []
    for kind in range(4):
        cls, box, coef = synth.head_outputs(300 + kind, A, 81, 'realistic')
        cls = cls.copy()
        hot = [3, 17, 40, 80]
        if kind == 0:
            for c in hot:
                cls[:, c] = rng.uniform(0.06, 0.2, A).astype(np.float32)
                cls[sampled, c] = rng.uniform(0.8, 0.99, sampled.size).astype(np.float32)
        elif kind == 1:
            for c in hot:
                cls[:, c] = rng.uniform(0.06, 0.1, A).astype(np.float32)
                hi = rng.choice(others, 6000, replace=False)
                cls[hi, c] = rng.uniform(0.5, 0.99, hi.size).astype(np.float32)
                cls[sampled, c] = 0.07
        elif kind == 2:
            for c in hot:
                tied = rng.choice(A, 5000, replace=False)
                cls[tied, c] = np.float32(0.75)
        else:
            cls[sampled, 1:] = 0.0
            cls[sampled, 0] = 1.0
        imgs.append((cls, box, coef))
    cls = np.stack([i[0] for i in imgs]); box = np.stack([i[1] for i in imgs]); coef = np.stack([i[2] for i in imgs])
    r = _run(cuda, cls, box, coef, anchors, _cfg(S=S))
    for b in range(4):
        _check_image(r, b, pp.nms(cls[b], box[b], anchors), coef[b])


# Pascal's 21 and the custom set's 5 classes, and the bounds: 2 classes launch one block per image in the per-class stages, 129
# (C1 = 128) fill all four class slots of every lane of k_sample_cuts and every [128] shared array of the phase-1 kernels
CLASS_COUNTS = (2, 5, 21, 129)


def largest_max_det(C):
    """The largest max_det <= 256 whose final top-k keys (2 C1 max_det words after C1 counts) fit its 200 KiB."""
    C1 = C - 1
    return min(256, (200 * 1024 - 4 * ((C1 + 3) & ~3)) // (8 * C1))


@pytest.mark.parametrize('C', CLASS_COUNTS)
@pytest.mark.parametrize('S', [550, 128])
def test_class_counts_vs_oracle(cuda, S, C):
    """Fast-NMS and traditional NMS at C classes, bit for bit against the oracle: at S = 550 (A = 19 248 > 2048, so the per-class
    lists are filled from k_sample_cuts' sampled cuts) and S = 128 (A = 1023, no sampling).  One batch holds a stress image, a
    realistic one and a stress image with scores quantised to 1/16, whose tied groups straddle every max_det cut."""
    anchors = pp.make_anchors(S)
    assert (anchors.shape[0] > 2048) == (S == 550)
    items = [build_nms_inputs(S, reg, seed, None, C) for reg, seed in (('stress', 31), ('realistic', 32), ('stress', 33))]
    cls = np.stack([i[1] for i in items]); box = np.stack([i[2] for i in items]); coef = np.stack([i[3] for i in items])
    cls[2] = (np.round(cls[2] * 16) / 16).astype(np.float32)
    md_max = largest_max_det(C)
    assert (md_max < 256) == (C == 129)
    trad = [pp.nms(cls[b], box[b], anchors, max_det=10 ** 9, traditional=True, img_size=S) for b in range(3)]
    assert trad[0] is not None and len(trad[0][0]) > 1
    for top_k, max_det in ((200, 100), (7, 5), (1, 1), (256, md_max)):
        r = _run(cuda, cls, box, coef, anchors, _cfg(S=S, classes=C, top_k=top_k, max_detections=max_det))
        for b in range(3):
            _check_image(r, b, pp.nms(cls[b], box[b], anchors, top_k=top_k, max_det=max_det), coef[b])
        r = _run(cuda, cls, box, coef, anchors, _cfg(True, S=S, classes=C, max_detections=max_det))
        for b in range(3):
            _check_image(r, b, None if trad[b] is None else tuple(a[:max_det] for a in trad[b]), coef[b])


def test_hard_nms_vs_oracle_and_golden(cuda):
    from yolact_minimal_b200 import cython_nms
    g = load_golden('hard_nms.npz')
    for seed, n in ((1, 1), (2, 17), (3, 300), (4, 1500)):
        xy = synth.uniform(seed, 11, (n, 2)) * 400
        wh = synth.uniform(seed, 12, (n, 2)) * 120 + 1
        sc = synth.uniform(seed, 13, (n, 1))
        dets = np.concatenate([xy, xy + wh, sc], 1).astype(np.float32)
        for thr in (0.3, 0.5):
            keep = cython_nms.nms(dets, thr)                                   # host buffers -> yb_hard_nms_host
            assert keep.dtype == np.int64
            assert np.array_equal(keep, g[f's{seed}_n{n}_t{thr}'])
            assert np.array_equal(keep, pp.hard_nms(dets, thr))
            keep_dev = cython_nms.nms(torch.from_numpy(dets).to(cuda), thr)    # device pointer -> yb_hard_nms
            assert np.array_equal(keep_dev, keep)
    assert cython_nms.nms(np.zeros((0, 5), np.float32), 0.5).shape == (0,)
    # tied scores: descending score, ties by descending index (oracle/postprocess_np.hard_nms)
    dets = np.array([[0, 0, 10, 10, .5], [1, 1, 11, 11, .5], [50, 50, 60, 60, .5], [0, 0, 10, 10, .9]], np.float32)
    assert np.array_equal(cython_nms.nms(dets, 0.5), pp.hard_nms(dets, 0.5))


def test_detect_host_abi(cuda):
    """yb_detect_host with plain host buffers (what a C caller would do)."""
    from yolact_minimal_b200 import _lib
    S = 128
    anchors, cls, box, coef = build_nms_inputs(S, 'realistic', 9, None)
    A = anchors.shape[0]
    B = 2
    cls2 = np.ascontiguousarray(np.stack([cls, cls[::-1]])); box2 = np.ascontiguousarray(np.stack([box, box[::-1]]))
    coef2 = np.ascontiguousarray(np.stack([coef, coef[::-1]]))
    p = _lib.DetectParams(0.05, 0.5, 200, 100, 81, 32, 0, float(S))
    cnt = np.zeros(B, np.int32); oc = np.zeros((B, 100), np.int32); oa = np.zeros((B, 100), np.int32)
    osc = np.zeros((B, 100), np.float32); ob = np.zeros((B, 100, 4), np.float32); oco = np.zeros((B, 100, 32), np.float32)
    L = _lib.lib()
    _lib.check(L.yb_detect_host(cls2.ctypes.data, box2.ctypes.data, coef2.ctypes.data, anchors.ctypes.data, B, A,
                                ctypes.byref(p), cnt.ctypes.data, oc.ctypes.data, oa.ctypes.data, osc.ctypes.data,
                                ob.ctypes.data, oco.ctypes.data), 'yb_detect_host')
    r = dict(count=cnt, cls=oc, anchor=oa, score=osc, box=ob, coef=oco)
    for b in range(B):
        _check_image(r, b, pp.nms(cls2[b], box2[b], anchors), coef2[b])
    # error path: bad top_k is reported, not ignored
    p.top_k = 1000
    assert L.yb_detect_host(cls2.ctypes.data, box2.ctypes.data, coef2.ctypes.data, anchors.ctypes.data, B, A,
                            ctypes.byref(p), cnt.ctypes.data, oc.ctypes.data, oa.ctypes.data, osc.ctypes.data,
                            ob.ctypes.data, oco.ctypes.data) == -3
    assert b'top_k' in L.yb_last_error()


def test_reference_signature_nms_after_nms(cuda):
    """nms()/after_nms() with the reference's signatures and return conventions."""
    from yolact_minimal_b200.utils.output_utils import nms, after_nms
    g = load_golden('after_nms.npz')
    for name, S, h, w, seed in (('S128_80x120', 128, 80, 120, 5), ('S128_97x64', 128, 97, 64, 6), ('S256_60x60', 256, 60, 60, 7)):
        anchors = pp.make_anchors(S)
        cls, box, coef = synth.head_outputs(seed, anchors.shape[0], 81, 'realistic')
        proto = synth.proto(seed, S // 4)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
        cfg = _cfg(S=S)
        ids, scores, boxes, coefs, proto_p = nms(t(cls)[None], t(box)[None], t(coef)[None], t(proto)[None],
                                                 anchors.reshape(-1).astype(np.float64).tolist(), cfg)
        o = pp.nms(cls, box, anchors)
        assert ids.dtype == torch.int64 and np.array_equal(ids.cpu().numpy(), o[0])
        assert np.array_equal(coefs.cpu().numpy(), coef[o[3]])
        assert proto_p.shape == (S // 4, S // 4, 32)
        for dtype in (torch.float32, torch.uint8):
            rid, rsc, rbx, rmask = after_nms(ids, scores, boxes, coefs, proto_p, h, w, mask_dtype=dtype)
            torch.cuda.synchronize()
            om = pp.after_nms(o[0], o[1], o[2], coef[o[3]], proto, h, w)
            assert rbx.dtype == torch.int32 and np.array_equal(rbx.cpu().numpy(), om[2])
            assert np.array_equal(rbx.cpu().numpy(), g[name + '/boxes_px'])
            m = rmask.cpu().numpy().astype(np.float32)
            assert m.shape == om[3].shape and set(np.unique(m)) <= {0.0, 1.0}
            assert (m != om[3]).mean() < 5e-4                                  # fp32 dot/sigmoid rounding at the 0.5 edge
            shape = tuple(g[name + '/mask_shape'])
            ref = np.unpackbits(g[name + '/mask_bits'])[:int(np.prod(shape))].reshape(shape)
            assert (m != ref).mean() < 5e-4                                    # vs the reference itself
    # "no detections" convention
    cls0 = np.zeros((anchors.shape[0], 81), np.float32); cls0[:, 0] = 1
    r = nms(t(cls0)[None], t(box)[None], t(coef)[None], t(proto)[None], t(anchors), cfg)
    assert r == (None,) * 5
    assert after_nms(None, None, None, None, None, 10, 10) == (None,) * 4


def test_val_aug_gpu(cuda):
    """GPU pre-process (yb_val_aug) vs the oracle and the reference-minted goldens."""
    from yolact_minimal_b200.utils.augmentations import val_aug
    from test_oracle_golden import VAL_AUG_CASES
    g = load_golden('val_aug.npz')
    for name, h, w, S, seed in VAL_AUG_CASES:
        img = (synth.uniform(seed, 21, (h, w, 3)) * 256).astype(np.uint8)
        out = val_aug(img, S).cpu().numpy()
        ref = pp.val_aug(img, S)
        assert out.shape == ref.shape
        assert np.abs(out - ref).max() < 2e-5, np.abs(out - ref).max()           # same formula, fp32
        sub = int(g[name + '/sub'])
        assert np.abs(out[:, ::sub, ::sub] - g[name + '/out']).max() < 2e-4      # vs cv2 (IPP)
