"""GPU: mask assembly (yb_mask_assemble, csrc/masks.cu) op by op against fp64, at the bench's shapes and at the edges, and the
packed-mask stage (mask IoU, RLE) at full image sizes.

yb_mask_assemble is called through the C ABI with a workspace the test owns, so the low-resolution stage (k_mask_lowres's output,
d x P x P fp32) is read back from it after the call; every output buffer carries a sentinel-filled tail that must be untouched.
Error model (the style of test_forward_ops_gpu.py):

  k_mask_lowres   crop decision: EXACT against the fp32 restatement of sanitize_coordinates / crop (oracle/postprocess_np); pixels
                  outside the crop are exactly 0.0.  Inside (or everywhere with crop = 0) the value is compared with v = sigmoid(t),
                  t = the fp64 dot product of the fp32 operands:
                      |low - v| <= v (1 - v) (C_ACC K 2^-24 sum_k |p_k c_k| + 2^-22) + 2 2^-24 v + 2^-126
                  the logit error of a K-term fmaf chain (Higham 4.2, C_ACC = 2), expf's 2 ulp, the add and the divide, and the
                  denormal / overflow range of the fp32 result.  Where t > 17, 1 + e^-t rounds to 1 and the value must be exactly
                  1.0; where t < -89, expf overflows and it must be exactly 0.0.
  k_mask_resize*  input: the kernel's own low-resolution values; source indices and weights: the kernels' fp32 arithmetic
                  (pp._bilinear_axis), so a wrong tap or weight gives an O(1) error.  The value is computed in fp64; an output bit
                  must equal v64 > 0.5 wherever |v64 - 0.5| > 6 2^-24 (every product / sum of the fp32 form is rounded once and
                  all terms are in [0, 1]); the pixels inside that band are counted and reported, and there the bit must equal
                  the fp32 restatement of the kernel's arithmetic (a saturated mask interpolated with weights 0.5 / 0.5 lands
                  exactly on 0.5, which is not > 0.5).  The float32, uint8 and
                  bit-packed outputs are computed by the same arithmetic and must agree bit for bit everywhere.
  k_boxes_px      exact: numpy's truncation of the fp32 product box * max(h, w), negative and > 1 boxes included.
  mask IoU        exact: numpy's integer counts and the fp32 division inter / ((|a| + |b|) - inter).
  RLE             exact: the run lengths of the column-major scan (pp.rle_counts), which decode back to the mask.
"""
import functools

import numpy as np
import pytest
import torch

from oracle import synth, postprocess_np as pp

pytestmark = pytest.mark.gpu

C_ACC = 2.0
E24 = 2.0 ** -24
BAND = 6 * E24
TAIL = 4096
SENT = 0xA5
IMAGES = ((480, 640), (640, 480), (1080, 1920), (550, 550), (479, 641), (33, 31), (1, 97), (97, 1), (100, 60))
DETS = (1, 15, 16, 17, 100, 256)


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _sentinel(nbytes, dev):
    return torch.full((nbytes + TAIL,), SENT, dtype=torch.uint8, device=dev)


def assemble(dev, proto, coef, box, h, w, crop, fmt):
    """yb_mask_assemble with test-owned buffers.  Returns (low [d,P,P] fp32 from the workspace, masks, boxes_px) on the device,
    after checking that nothing was written past the workspace, the mask buffer or the box buffer."""
    from yolact_minimal_b200 import _lib
    d, K = coef.shape
    P = proto.shape[0]
    L = _lib.lib()
    wsb = int(L.yb_mask_workspace_bytes(d, P))
    assert wsb == d * P * P * 4
    mshape = (d, h, (w + 31) // 32) if fmt == 2 else (d, h, w)
    mdt = {0: torch.uint8, 1: torch.float32, 2: torch.int32}[fmt]
    mb = int(np.prod(mshape)) * (1 if fmt == 0 else 4)
    ws, mk, bx = _sentinel(wsb, dev), _sentinel(mb, dev), _sentinel(d * 16, dev)
    dp, dc, db = _t(proto, dev), _t(coef, dev), _t(box, dev)
    _lib.check(L.yb_mask_assemble(dp.data_ptr(), dc.data_ptr(), db.data_ptr(), d, P, K, h, w, crop, fmt, ws.data_ptr(), wsb,
                                  mk.data_ptr(), bx.data_ptr(), torch.cuda.current_stream().cuda_stream), 'yb_mask_assemble')
    torch.cuda.synchronize()
    for name, buf, n in (('workspace', ws, wsb), ('mask', mk, mb), ('boxes_px', bx, d * 16)):
        assert bool((buf[n:] == SENT).all()), f'{name}: written past its end'
    return ws[:wsb].view(torch.float32).view(d, P, P), mk[:mb].view(mdt).view(mshape), bx[:d * 16].view(torch.int32).view(d, 4)


# ----------------------------------------------------------------------------------------------------------------- references
def check_lowres(low, proto, coef, box, crop):
    """k_mask_lowres against fp64; returns the worst |err| / bound."""
    dev = low.device
    d, K = coef.shape
    P = proto.shape[0]
    p64 = _t(proto, dev).double().view(P * P, K)
    c64 = _t(coef, dev).double()
    t = (p64 @ c64.T).T.reshape(d, P, P)                                   # fp64 dot of the fp32 operands
    mag = (p64.abs() @ c64.abs().T).T.reshape(d, P, P)
    v = torch.sigmoid(t)
    bound = v * (1 - v) * (C_ACC * K * E24 * mag + 2.0 ** -22) + 2 * E24 * v + 2.0 ** -126
    low64 = low.double()
    if crop:
        x1, x2 = pp.sanitize_coordinates(box[:, 0], box[:, 2], P, 1)
        y1, y2 = pp.sanitize_coordinates(box[:, 1], box[:, 3], P, 1)
        ar = np.arange(P, dtype=np.float32)
        inx = (ar[None, :] >= x1[:, None]) & (ar[None, :] < x2[:, None])
        iny = (ar[None, :] >= y1[:, None]) & (ar[None, :] < y2[:, None])
        inside = _t(iny[:, :, None] & inx[:, None, :], dev)
        assert bool((low64[~inside] == 0).all()), 'a pixel outside the crop is not 0.0'
    else:
        inside = torch.ones_like(low64, dtype=torch.bool)
    err = (low64 - v).abs()
    worst = float((err / bound)[inside].max()) if bool(inside.any()) else 0.0
    assert bool((err <= bound)[inside].all()), f'k_mask_lowres: worst |err| / bound {worst:.3g}'
    assert bool((low64[inside & (t > 17)] == 1).all()) and bool((low64[inside & (t < -89)] == 0).all())
    return worst, int((inside & ((t > 17) | (t < -89))).sum())


def resize_ref(low, P, h, w, d0, d1, dtype=torch.float64):
    """Bilinear value of detections d0:d1 with the kernels' fp32 indices and weights, in fp64 -- or, with dtype=float32, the
    kernels' own fp32 arithmetic (separately rounded torch ops in ATen's order)."""
    dev = low.device
    ori = max(h, w)
    y0, y1, ly0, ly1 = (a[:h] for a in pp._bilinear_axis(P, ori))
    x0, x1, lx0, lx1 = (a[:w] for a in pp._bilinear_axis(P, ori))
    L = low[d0:d1].to(dtype)
    ti = lambda a: torch.from_numpy(a).to(dev)
    y0, y1, x0, x1 = ti(y0), ti(y1), ti(x0), ti(x1)
    ly0, ly1, lx0, lx1 = (ti(a).to(dtype) for a in (ly0, ly1, lx0, lx1))
    r0, r1 = L[:, y0], L[:, y1]
    top = r0[:, :, x0] * lx0 + r0[:, :, x1] * lx1
    bot = r1[:, :, x0] * lx0 + r1[:, :, x1] * lx1
    return top * ly0[:, None] + bot * ly1[:, None]


def unpack(bits, w):
    from yolact_minimal_b200.utils import mask_utils as mu
    return mu.unpack_masks(bits, w)


def check_resize(low, masks, P, h, w):
    """masks: {fmt: tensor}.  Returns the number of pixels inside the ambiguity band."""
    d = low.shape[0]
    u8 = masks[0]
    assert bool((masks[1] == u8.float()).all()), 'float32 and uint8 masks differ'
    assert bool((unpack(masks[2], w) == u8).all()), 'bit-packed and uint8 masks differ'
    assert bool(((u8 == 0) | (u8 == 1)).all())
    if w % 32:                                                             # the last word's bits past the row end are 0
        assert bool((((masks[2][..., -1].long() & 0xffffffff) >> (w % 32)) == 0).all())
    amb = 0
    step = max(1, int(4e7 // (h * w)))
    for d0 in range(0, d, step):
        v = resize_ref(low, P, h, w, d0, min(d, d0 + step))
        sure = (v - 0.5).abs() > BAND
        amb += int((~sure).sum())
        got = u8[d0:d0 + step].bool()
        bad = sure & (got != (v > 0.5))
        assert not bool(bad.any()), f'k_mask_resize: {int(bad.sum())} pixels disagree with the fp64 bilinear value'
        if not bool(sure.all()):                                           # inside the band: the fp32 restatement decides
            v32 = resize_ref(low, P, h, w, d0, min(d, d0 + step), torch.float32)
            bad = ~sure & (got != (v32 > 0.5))
            assert not bool(bad.any()), f'k_mask_resize: {int(bad.sum())} pixels near 0.5 disagree with the fp32 restatement'
    return amb


def check_boxes_px(bpx, box, h, w):
    want = (box.astype(np.float32) * np.float32(max(h, w))).astype(np.float32).astype(np.int32)
    assert np.array_equal(bpx.cpu().numpy(), want)


def run_case(dev, proto, coef, box, h, w, crop, key):
    P = proto.shape[0]
    outs = {fmt: assemble(dev, proto, coef, box, h, w, crop, fmt) for fmt in (0, 1, 2)}
    low = outs[0][0]
    for fmt in (1, 2):
        assert torch.equal(outs[fmt][0], low) and torch.equal(outs[fmt][2], outs[0][2])
    worst, saturated = check_lowres(low, proto, coef, box, crop)
    amb = check_resize(low, {f: o[1] for f, o in outs.items()}, P, h, w)
    check_boxes_px(outs[0][2], box, h, w)
    print(f'{key}: lowres worst err/bound {worst:.3f}, saturated {saturated}, ambiguous pixels {amb} of {coef.shape[0] * h * w}')
    return outs


# -------------------------------------------------------------------------------------------------------------------- inputs
@functools.lru_cache(maxsize=1)
def bench_inputs():
    """Exactly the inputs of bench.py's mask_stage leg: 550 head, 'realistic' seed 5, proto P = 138, the oracle's Fast NMS."""
    anchors = pp.make_anchors(550)
    cls, box, coef = synth.head_outputs(5, anchors.shape[0], 81, 'realistic')
    proto = synth.proto(5, 138)
    ids, scores, boxes, aidx = pp.nms(cls, box, anchors)
    return proto, coef[aidx], boxes


def adversarial_boxes(P, n, seed):
    """Reversed corners, boxes outside [0, 1], zero widths / heights, and corners k / P that land exactly on pixel edges after the
    x P -/+ 1 of sanitize_coordinates; the rest random, and the unclipped boxes of the numpy twin (negative and > 1)."""
    fP = np.float32(P)
    k = np.arange(n)
    u = synth.uniform(seed, 1, (n, 4))
    edge = (np.floor(u * (P + 1)) / fP).astype(np.float32)                # k / P: x P is exact
    rnd = (u * 1.4 - 0.2).astype(np.float32)
    b = np.where((k % 2 == 0)[:, None], edge, rnd).astype(np.float32)
    b[k % 5 == 1] = b[k % 5 == 1][:, [2, 3, 0, 1]]                        # reversed (x1 > x2, y1 > y2)
    z = k % 7 == 3
    b[z, 2] = b[z, 0]                                                      # zero width
    z = k % 11 == 4
    b[z, 3] = b[z, 1]                                                      # zero height
    b[k % 13 == 6] = [-0.5, -0.25, 1.5, 1.25]
    b[k % 17 == 8] = [0.0, 0.0, 1.0, 1.0]
    wild = wild_boxes()
    m = min(len(wild), n // 4)
    b[n - m:] = wild[seed % 7:seed % 7 + m]
    return np.ascontiguousarray(b)


@functools.lru_cache(maxsize=1)
def wild_boxes():
    """The unclipped boxes of the numpy twin (nms_numpy) on large regressions: negative and > 1 coordinates."""
    anchors = pp.make_anchors(128)
    cls, bx, _ = synth.head_outputs(4, anchors.shape[0], 81, 'stress')
    wild = pp.nms_numpy(cls, (bx * 3).astype(np.float32), anchors)[2]
    assert wild.min() < 0 and wild.max() > 1 and len(wild) == 100
    return wild


def synth_coef(n, K, seed):
    """tanh-normal rows; every fourth row scaled x 30 so that the logits reach +-100 (expf overflows / 1 + e^-t rounds to 1)."""
    c = np.tanh(synth.normal(seed, 3, (n, K))).astype(np.float32)
    c[3::4] *= np.float32(30)
    return c


def sweep_cases():
    cases = []
    i = 0
    for P in (138, 136, 32):
        for d in DETS:
            h, w = IMAGES[i % len(IMAGES)]
            cases.append((P, d, h, w, i % 2))
            i += 1
    return cases


# --------------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize('crop', [1, 0])
@pytest.mark.parametrize('hw', IMAGES, ids=lambda x: f'{x[0]}x{x[1]}')
def test_bench_inputs(cuda, hw, crop):
    proto, coef, box = bench_inputs()
    assert proto.shape[0] == 138 and coef.shape[0] == 100
    run_case(cuda, proto, coef, box, hw[0], hw[1], crop, f'bench {hw[0]}x{hw[1]} crop={crop}')


@pytest.mark.parametrize('case', sweep_cases(), ids=lambda c: f'P{c[0]}-d{c[1]}-{c[2]}x{c[3]}-crop{c[4]}')
def test_adversarial_sweep(cuda, case):
    P, d, h, w, crop = case
    seed = 1000 + P + d
    proto = synth.proto(seed, P)
    coef = synth_coef(d, 32, seed)
    box = adversarial_boxes(P, d, seed) if d >= 4 else np.array([[0.25, 0.75, 0.5, 0.125]], np.float32)[:d]
    run_case(cuda, proto, coef, box, h, w, crop, f'P{P} d{d} {h}x{w} crop={crop}')


def test_res101_forward_detections(cuda):
    """Masks of real detections: a res101 550 fp16 forward of the synthetic weights, B = 2, through the GPU Fast NMS."""
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    from yolact_minimal_b200.utils.output_utils import detect_batched
    from oracle import forward_torch as ft
    cfg = make_config('res101_coco', 550)
    cfg.precision, cfg.max_batch = 'fp16', 2
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict('res101', seed=0), strict=True)
    net = net.to(cuda).eval()
    with torch.no_grad():
        cls, box, coef, proto = net(torch.from_numpy(synth.image_batch(3, 2, 550)).to(cuda))
    det = detect_batched(cls, box, coef, net.anchors, net.cfg)
    for b, (h, w) in enumerate(((480, 640), (1080, 1920))):
        d = int(det['count'][b])
        assert d > 0
        pr = proto[b].float().contiguous().cpu().numpy()
        assert pr.shape == (138, 138, 32)
        run_case(cuda, pr, det['coef'][b, :d].cpu().numpy(), det['box'][b, :d].cpu().numpy(), h, w, 1, f'res101 image {b} {h}x{w}')


# ------------------------------------------------------------------------------------------------------ packed masks, full size
def _rle_np(mask):
    """Vectorised pp.rle_counts: column-major runs, the first one of zeros (possibly empty)."""
    v = np.asarray(mask).astype(np.int8).reshape(-1, order='F')
    cuts = np.flatnonzero(np.diff(v)) + 1
    edges = np.concatenate([[0], cuts, [v.size]])
    runs = np.diff(edges)
    return (np.concatenate([[0], runs]) if v[0] else runs).astype(np.uint32)


def _bits_masks(cuda, h, w, d=100, crop=1):
    proto, coef, box = bench_inputs()
    _, bits, _ = assemble(cuda, proto, coef[:d], box[:d], h, w, crop, 2)
    return bits


def test_mask_iou_bits_full_size(cuda):
    from yolact_minimal_b200.utils import mask_utils as mu
    for h, w, n, m in ((480, 640, 100, 20), (1080, 1920, 100, 5)):
        a = _bits_masks(cuda, h, w, n, 1)
        b = _bits_masks(cuda, h, w, n, 0)[::n // m][:m].contiguous()          # uncropped masks of other detections
        got = mu.mask_iou_bits(a, b).cpu().numpy()
        A = unpack(a, w).reshape(n, -1).double()
        Bm = unpack(b, w).reshape(m, -1).double()
        inter = (A @ Bm.T).cpu().numpy().astype(np.int64)                     # exact: < 2^53
        ca, cb = A.sum(1).cpu().numpy().astype(np.int64), Bm.sum(1).cpu().numpy().astype(np.int64)
        assert inter.max() > 0 and (inter < np.minimum(ca[:, None], cb[None, :])).any()
        fi = inter.astype(np.float32)
        with np.errstate(invalid='ignore'):
            want = fi / ((ca.astype(np.float32)[:, None] + cb.astype(np.float32)[None, :]) - fi)
        assert np.array_equal(got.view(np.uint32), want.astype(np.float32).view(np.uint32)), (h, w)


def test_rle_full_size(cuda):
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.utils import mask_utils as mu
    sets = [(480, 640, _bits_masks(cuda, 480, 640, 100, 1)), (1080, 1920, _bits_masks(cuda, 1080, 1920, 20, 1)),
            (48, 4096, _bits_masks(cuda, 48, 4096, 8, 0))]
    stripes = np.zeros((2, 480, 640), np.uint8)
    stripes[0, 1::2] = 1                                                    # 480 runs per column: 307 201 runs > max_runs = 4096
    stripes[1, :, 3::7] = 1
    sets.append((480, 640, mu.pack_masks(torch.from_numpy(stripes).to(cuda))))
    for h, w, bits in sets:
        host = unpack(bits, w).cpu().numpy()
        counts = mu.rle_counts(bits, h, w)
        rles = mu.encode_rle(bits, h, w)
        for i in range(host.shape[0]):
            ref = _rle_np(host[i])
            if i < 2 and h * w <= 480 * 640:
                assert np.array_equal(ref, pp.rle_counts(host[i]))         # the vectorised restatement is pp.rle_counts
            assert np.array_equal(counts[i], ref), (h, w, i)
            assert int(counts[i].sum()) == h * w
            assert rles[i]['size'] == [h, w] and mu.rle_string_to_counts(rles[i]['counts']) == [int(c) for c in ref]
            assert np.array_equal(pp.rle_decode(counts[i], h, w), host[i])
    assert len(counts[0]) > 4096                                            # the striped mask took the retry path
    # w = 4097 is refused
    bits = torch.zeros(1, 4, (4097 + 31) // 32, dtype=torch.int32, device=cuda)
    out = torch.zeros(1, 64, dtype=torch.int32, device=cuda)
    nr = torch.zeros(1, dtype=torch.int32, device=cuda)
    L = _lib.lib()
    assert L.yb_mask_rle(bits.data_ptr(), 1, 4, 4097, out.data_ptr(), 64, nr.data_ptr(), None) == -3
    assert b'4097' in L.yb_last_error()
    with pytest.raises(_lib.YolactB200Error):
        mu.rle_counts(bits, 4, 4097)
