"""GPU: the training loss stage (yb_losses, csrc/losses.cu) element by element against an fp64 restatement of the reference.

The inputs are the ones a trained network produces rather than easy ones: class 0 dominating most rows with batch maxima up to 60,
mask logits saturated up to |z| = 100, COCO-scale target sets (up to 256 gts per image, duplicates, gts smaller than every anchor,
empty images anywhere in the batch) and ragged masks.  Everything runs at the 550 anchor set (A = 19248).

The reference is torch float64 except where the reference itself decides something in fp32: IoU, thresholds and encode
(oracle/train_torch.assign_targets on CPU), the OHEM marks that are ranked (torch on the GPU, the reference's training device), the
stored sigmoid p whose saturation to 0 / 1 switches torch's BCE clamp max(p (1 - p), 1e-12), and the down-sampled targets
(F.interpolate on the GPU, > 0.5).

Error model (u = 2^-24, fp32 round to nearest; expf <= 2 ulp, logf <= 1 ulp, ulp(v) <= 2u |v|; a sum of n terms in any order errs
by <= n u sum|terms| (Higham 4.2)); every bound below is twice the model, and the worst err / bound ratio of each check is printed:
  d_cls   the softmax of a row x: the argument x - max rounds (u |x - max|), each exp term 4u, the lane sum NC u, logf 1 ulp,
          lse = log s + max rounds (u |lse|), x - lse rounds (u |x - lse|), the final expf 4u; then p - onehot rounds, and the
          scale gs * gsd / num_pos (two roundings and one divide) and the product add 3u of the result.  Logits that underflow expf
          add an absolute 2^-125 times the scale.
  d_box   d = box - offset rounds (u), the scale and product 3u: 5u of the result (exact 0 at d = 0 and off positives).
  mask    z = sum_k proto_k coef_k by a K-term fma chain errs by K u sum|proto coef|; with expf's 2 ulp this is an uncertainty ez
          of z.  p = 1 / (1 + e) is stored in fp32 and the rounding of 1 + e can go either way: 2u of p, absolute (p - t
          cancels near p = 1).  The reference gradient / loss is evaluated at z and z +- ez, and the spread is allowed (it covers a p that
          saturates to 1 inside the window); the weight 1 / area * n_all / n, the scale and the chain add 12u of |g|.  d_proto
          sums n selected masks (n u), d_coef sums P^2 pixels through a warp tree and one float atomic per warp
          (5 + P^2 / 32 terms).
  seg     p = 1 / (1 + expf(-v)) is 6u of p; p - t, the scale and the product 3u of the result.
"""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import train_checks as tc
from oracle import synth, train_torch as tt

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
NCLS = 81


@pytest.fixture(scope='module')
def env(cuda):
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    cfg = make_config('res50_coco', 550, mode='train', train_bs=2)
    a = Yolact(cfg).anchors
    a = (a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)).reshape(-1, 4).astype(np.float32)
    assert a.shape[0] == 19248
    return types.SimpleNamespace(cfg=cfg, anchors=a, A=a.shape[0], dev=cuda)


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def assign(env, tg, pos=0.5, neg=0.4):
    """The checker's assign_targets (fp32 on CPU) per image -> labels, matched idx, offsets [B, A(, 4)]; an empty image is all 0."""
    anc = torch.from_numpy(env.anchors)
    th = types.SimpleNamespace(pos_iou_thre=pos, neg_iou_thre=neg)
    L, I, O = [], [], []
    for t in tg:
        if len(t) == 0:
            L.append(np.zeros(env.A, np.int64)); I.append(np.zeros(env.A, np.int64)); O.append(np.zeros((env.A, 4), np.float32))
            continue
        o, lab, _, i = tt.assign_targets(th, torch.from_numpy(t[:, :4]).float(), anc, torch.from_numpy(t[:, 4]).long())
        L.append(lab.numpy()); I.append(i.numpy()); O.append(o.numpy())
    return np.stack(L), np.stack(I), np.stack(O)


def call(env, tg, mk, cls, box=None, coef=None, proto=None, seg=None, P=None, Hs=None, K=32, **kw):
    """yb_losses with zero defaults for the outputs a sub-test does not look at."""
    B, A, C = cls.shape
    S = mk[0].shape[-1]
    P = P or -(-S // 4)
    Hs = Hs or -(-S // 8)
    box = np.zeros((B, A, 4), np.float32) if box is None else box
    coef = np.zeros((B, A, K), np.float32) if coef is None else coef
    proto = np.zeros((B, P, P, coef.shape[-1]), np.float32) if proto is None else proto
    seg = np.zeros((B, C - 1, Hs, Hs), np.float32) if seg is None else seg
    kw.setdefault('grad_scale', (1.0, 1.0, 1.0, 1.0))
    return tc.run_native_losses(env.dev, env.cfg, env.anchors, tg, mk, f32(cls), f32(box), f32(coef), f32(proto), f32(seg), **kw)


def down(masks, size, device):
    """The reference's binarised down-sampled targets: F.interpolate(bilinear, align_corners=False) > 0.5, fp32."""
    m = torch.from_numpy(np.ascontiguousarray(masks, np.float32)).to(device)
    return F.interpolate(m[None], (size, size), mode='bilinear', align_corners=False)[0] > 0.5


def targets(env, masks, size):
    """GPU targets with the pixels where torch's CPU and CUDA results disagree (listed; there should be none)."""
    g, c = down(masks, size, env.dev).cpu().numpy(), down(masks, size, 'cpu').numpy()
    bad = np.argwhere(g != c)
    if len(bad):
        print(f'torch CPU / CUDA down-sampling disagree at {len(bad)} pixels (size {size}): {bad[:8].tolist()}')
    return g, g == c


def report(name, err, bound):
    err, bound = np.asarray(err, np.float64), np.asarray(bound, np.float64)
    over = (err > bound)
    worst = float(np.max(np.where(bound > 0, err / np.where(bound > 0, bound, 1), np.where(err > 0, np.inf, 0)))) if err.size else 0.0
    print(f'{name}: worst err/bound {worst:.3g} over {err.size} elements')
    assert not over.any(), f'{name}: {int(over.sum())} elements over the bound, worst err/bound {worst:.3g}, first at {np.argwhere(over)[:4].tolist()}'
    return worst


def rect_gts(rng, n, lo=0.05, hi=0.5, ncls=80):
    xy = rng.uniform(0, 1 - hi, (n, 2))
    wh = rng.uniform(lo, hi, (n, 2))
    return f32(np.concatenate([xy, xy + wh, np.floor(rng.uniform(0, ncls, (n, 1)))], 1))


def ragged_masks(rng, n, S):
    """Blobs with holes, one-pixel lines and checkerboards: masks whose down-sampled edges are not box edges."""
    yy, xx = np.mgrid[0:S, 0:S]
    out = np.zeros((n, S, S), np.float32)
    for j in range(n):
        kind = j % 4
        if kind == 0:
            cy, cx, r = rng.uniform(0.2, 0.8) * S, rng.uniform(0.2, 0.8) * S, rng.uniform(0.1, 0.35) * S
            m = ((yy - cy) ** 2 + (xx - cx) ** 2 < r * r) & (rng.uniform(size=(S, S)) < 0.8)
        elif kind == 1:
            m = np.zeros((S, S), bool)
            for _ in range(6):
                i = rng.integers(0, S)
                if rng.uniform() < 0.5:
                    m[i, :] = True
                else:
                    m[:, i] = True
            m |= (yy == xx)
        elif kind == 2:
            p = int(rng.integers(1, 5))
            m = ((yy // p + xx // p) % 2) == 0
        else:
            m = rng.uniform(size=(S, S)) < 0.5
        out[j] = m
    return out


# ------------------------------------------------------------------------------------------------
# OHEM at trained-network logits
# ------------------------------------------------------------------------------------------------
def ohem_logits(rng, B, A, gm, hard):
    """Easy rows: class 0 at gm - delta, the other 80 classes 25 below it (fp64 mark ~1e-9, fp32 mark -ulp, 0 or +ulp).
    Hard rows: a mark in [0.5, 8] from one other class near class 0."""
    x0 = gm - rng.uniform(0, gm, (B, A))
    x = x0[..., None] - 25 - rng.uniform(0, 1, (B, A, NCLS))
    x[..., 0] = x0
    h0 = gm - rng.uniform(10, 20, (B, A))
    mu = rng.uniform(0.5, 8, (B, A))
    c1 = rng.integers(1, NCLS, (B, A))
    xh = h0[..., None] - 25 - rng.uniform(0, 1, (B, A, NCLS))
    xh[..., 0] = h0
    np.put_along_axis(xh, c1[..., None], (h0 + np.log(np.expm1(mu)))[..., None], -1)
    return f32(np.where(hard[..., None], xh, x))


def ohem_reference(cls, labels, A):
    """modules/yolact.py's mining in fp32 on the GPU (stable descending sort: ties by ascending anchor index), and fp64 marks."""
    B = cls.shape[0]
    flat = cls.reshape(-1, NCLS)
    mx = flat.max()
    m32 = (torch.log(torch.sum(torch.exp(flat - mx), 1)) + mx - flat[:, 0]).reshape(B, A)
    m64 = (torch.logsumexp(cls.double(), -1) - cls[..., 0].double())
    lab = torch.from_numpy(labels).to(cls.device)
    pos = lab > 0
    m32[pos] = 0
    m32[lab < 0] = 0
    rank = m32.sort(dim=1, descending=True, stable=True)[1].sort(1)[1]
    num_neg = torch.clamp(3 * pos.long().sum(1, keepdim=True), max=A - 1)
    neg = rank < num_neg
    neg[pos] = False
    neg[lab < 0] = False
    kth = m32.sort(dim=1, descending=True, stable=True)[0].gather(1, num_neg - 1)[:, 0]
    return m32.cpu().numpy(), m64.cpu().numpy(), neg.cpu().numpy(), num_neg[:, 0].cpu().numpy(), kth.cpu().numpy()


def check_ohem(r, cls, labels, A, gm, tag):
    m32, m64, rneg, num_neg, kth = ohem_reference(cls, labels, A)
    band = 4 * float(np.spacing(np.float32(gm)))
    kneg = r['neg'].astype(bool)
    out = []
    for b in range(cls.shape[0]):
        negl = labels[b] == 0
        n_neg32 = int((m32[b][negl] < 0).sum())
        print(f'OHEM gm={gm} {tag}[{b}]: num_neg {num_neg[b]}, k-th fp32 mark {kth[b]:.3g}, negative fp32 marks {n_neg32}, '
              f'selected {int(kneg[b].sum())} (reference {int(rneg[b].sum())})')
        assert not (kneg[b] & ~negl).any(), 'a positive or neutral anchor was mined'
        assert int(kneg[b].sum()) == int(rneg[b].sum())
        sel, uns = m64[b][kneg[b]], m64[b][negl & ~kneg[b]]
        if len(sel) and len(uns):
            assert sel.min() >= uns.max() - band, (f'image {b}: an unselected negative is harder than a selected one by '
                                                    f'{uns.max() - sel.min():.3g} (fp64 marks)')
        distinct = negl & (m32[b] != kth[b])
        bad = distinct & (kneg[b] != rneg[b])
        assert not bad.any(), f'image {b}: {int(bad.sum())} anchors differ from the reference rank set, e.g. {np.argwhere(bad)[:4, 0].tolist()}'
        out.append((num_neg[b], kth[b], n_neg32))
    return out


@pytest.mark.parametrize('gm', [8.0, 20.0, 30.0, 60.0])
def test_ohem_at_trained_logits(env, gm):
    """The 3 num_pos boundary inside the hard set (image 0), inside the ~0 set (image 1) and at the A - 1 cap (separate call: an
    image with > A / 3 positives, whose last anchor is an easy negative holding the batch maximum in class 0, mark exactly 0)."""
    A, rng = env.A, np.random.default_rng(int(gm))
    tg, mk = synth.train_targets(9, 2, 128, n=4)
    labels, _, _ = assign(env, tg)
    hard = np.zeros((2, A), bool)
    for b in (0, 1):
        negs = np.flatnonzero(labels[b] == 0)
        k = 3 * int((labels[b] > 0).sum())
        h = min(k + 150, len(negs)) if b == 0 else max(k // 3, 1)
        hard[b, rng.choice(negs, h, replace=False)] = True
    cls = ohem_logits(rng, 2, A, gm, hard)
    e = int(np.flatnonzero((labels[1] == 0) & ~hard[1])[0])
    cls[1, e, 0], cls[1, e, 1:] = gm, gm - 25
    r = call(env, tg, mk, cls)
    assert np.array_equal(r['labels'], labels)
    res = check_ohem(r, torch.from_numpy(cls).to(env.dev), labels, A, gm, 'hard/~0')
    assert res[0][1] >= 0.5 and abs(res[1][1]) < 1e-3, res

    # the cap: k = min(3 num_pos, A - 1) = A - 1
    tg_c = [f32([[0.0, 0.0, 0.35, 1.0, 3.0]])]
    mk_c = [np.ones((1, 128, 128), np.float32)]
    lab_c, _, _ = assign(env, tg_c, 0.0005, 0.0005)
    assert 3 * int((lab_c > 0).sum()) > A - 1 and lab_c[0, A - 1] == 0
    hard_c = np.zeros((1, A), bool)
    hard_c[0, rng.choice(np.flatnonzero(lab_c[0] == 0)[:-1], 300, replace=False)] = True
    cls_c = ohem_logits(rng, 1, A, gm, hard_c)
    cls_c[0, A - 1, 0], cls_c[0, A - 1, 1:] = gm, gm - 25
    r = call(env, tg_c, mk_c, cls_c, pos_iou_thr=0.0005, neg_iou_thr=0.0005)
    assert np.array_equal(r['labels'], lab_c)
    res = check_ohem(r, torch.from_numpy(cls_c).to(env.dev), lab_c, A, gm, 'cap')
    assert res[0][0] == A - 1
    assert int(r['neg'].sum()) == int((lab_c == 0).sum()) - 1           # the one anchor the cap leaves out is a real negative


# ------------------------------------------------------------------------------------------------
# class and box losses and their gradients
# ------------------------------------------------------------------------------------------------
def test_class_and_box_gradients_elementwise(env):
    A, B, rng = env.A, 2, np.random.default_rng(7)
    tg = [rect_gts(rng, 12, 0.03, 0.4), rect_gts(rng, 7, 0.03, 0.4)]
    mk = [np.zeros((len(t), 128, 128), np.float32) for t in tg]
    labels, _, off = assign(env, tg)
    cls = np.clip(rng.normal(0, 20, (B, A, NCLS)), -80, 80)
    trained = rng.uniform(size=(B, A)) < 0.6                            # background dominates
    cls[trained] = rng.normal(-10, 3, (int(trained.sum()), NCLS))
    cls[trained, 0] = 60
    edge = rng.uniform(size=(B, A)) < 0.05
    cls[edge, 0] = 80
    cls[edge, 1] = -80
    cls[:, :, NCLS - 1] = np.where(rng.uniform(size=(B, A)) < 0.02, 80.0, cls[:, :, NCLS - 1])
    cls = f32(cls)
    # box: offset + d with d in {0, +-1 exactly, +-1e3, N(0, 1)}
    d = rng.normal(0, 1, (B, A, 4))
    pick = rng.integers(0, 4, (B, A, 4))
    d = np.where(pick == 0, 0.0, np.where(pick == 1, np.sign(d), np.where(pick == 2, 1e3 * np.sign(d), d)))
    box = f32(off + d)
    gs = (0.7, 1.3, 1.0, 1.0)
    r = call(env, tg, mk, cls, box=box, grad_scale=gs)
    assert np.array_equal(r['labels'], labels)
    posm = labels > 0
    npos = max(int(posm.sum()), 1)
    dd = box.astype(np.float64) - r['offsets'].astype(np.float64)
    assert (np.abs(dd[posm][:, :2]) == 1).any() and (dd[posm] == 0).any() and (np.abs(dd[posm]) >= 999).any()
    chosen = posm | r['neg'].astype(bool)
    assert r['neg'].sum() > 0
    # d_cls
    x = torch.from_numpy(cls).to(env.dev).double()
    mx = x.max(-1, keepdim=True)[0]
    lse = torch.logsumexp(x, -1, keepdim=True)
    p = torch.exp(x - lse)
    tgt = torch.from_numpy(np.where(labels > 0, labels, 0)).to(env.dev)
    oh = F.one_hot(tgt, NCLS).double()
    g = float(np.float32(env.cfg.conf_alpha) * np.float32(gs[0])) / npos
    ref = g * (p - oh)
    s = torch.exp(x - mx).sum(-1, keepdim=True)
    E = U * ((x - mx).abs().max(-1, keepdim=True)[0] + 4 + NCLS) + 2 * U * torch.log(s).abs() + U * lse.abs() + U * (x - lse).abs()
    bound = 2 * (abs(g) * (p * (1.01 * E + 4 * U) + U * (p - oh).abs() + 2.0 ** -125) + 3 * U * ref.abs())
    ch = torch.from_numpy(chosen).to(env.dev)
    kd = torch.from_numpy(r['d_cls']).to(env.dev).double()
    assert bool((kd[~ch] == 0).all()), 'rows neither positive nor mined must be exactly 0'
    report('d_cls (chosen rows)', (kd - ref).abs()[ch].cpu().numpy(), bound[ch].cpu().numpy())
    # d_box
    gb = float(np.float32(env.cfg.bbox_alpha) * np.float32(gs[1])) / npos
    refb = gb * np.clip(dd, -1, 1) * posm[..., None]
    assert (r['d_box'][~posm] == 0).all(), 'd_box must be exactly 0 off positives'
    report('d_box', np.abs(r['d_box'] - refb), 2 * 5 * U * np.abs(refb))
    # the two losses
    lc = (lse[..., 0] - x.gather(-1, tgt[..., None])[..., 0])[ch]
    Ec = (E[..., 0][ch] + U * (lse[..., 0][ch].abs() + lc.abs()))
    ref_c = env.cfg.conf_alpha * float(lc.sum()) / npos
    b_c = 2 * (float(Ec.sum()) + 8 * U * float(lc.abs().sum())) / npos + 2 * U * abs(ref_c)
    print(f'class loss {r["losses"][0]:.8g} vs fp64 {ref_c:.8g}: err/bound {abs(r["losses"][0] - ref_c) / b_c:.3g}')
    assert abs(r['losses'][0] - ref_c) <= b_c
    ad = np.abs(dd[posm])
    sl1 = np.where(ad < 1, 0.5 * ad * ad, ad - 0.5)
    ref_b = env.cfg.bbox_alpha * sl1.sum() / npos
    b_b = 2 * (8 * U * sl1.sum() + 2 * U * (ad * ad.clip(max=1)).sum()) / npos * env.cfg.bbox_alpha + 2 * U * ref_b
    print(f'box loss {r["losses"][1]:.8g} vs fp64 {ref_b:.8g}: err/bound {abs(r["losses"][1] - ref_b) / b_b:.3g}')
    assert abs(r['losses'][1] - ref_b) <= b_b


# ------------------------------------------------------------------------------------------------
# mask loss
# ------------------------------------------------------------------------------------------------
def bce_unit(z, t):
    """dL/dz and L per unit weight at mask logit z (fp64) and target t, with torch's fp32 stored sigmoid."""
    e = torch.exp(-z).float()                        # rounded to fp32 (overflow -> inf)
    p = (1 / (1 + e)).double()                       # fp32 add and divide
    pq = p * (1 - p)
    G = (p - t) / pq.clamp_min(1e-12) * pq
    L = -(t * torch.log(p).clamp_min(-100) + (1 - t) * torch.log(1 - p).clamp_min(-100))
    return G, L, p


def mask_reference(env, r, tg, mk, proto, coef, sel, n_all, P, gsd2):
    """fp64 mask loss, d_proto, d_coef and their bounds.  sel[b] = selected anchors of image b (matched gt from the kernel's
    matched_idx, itself checked against the checker)."""
    dev, K = env.dev, proto.shape[-1]
    B = proto.shape[0]
    npos = max(int((r['labels'] > 0).sum()), 1)
    gscale = float(np.float32(env.cfg.mask_alpha) * np.float32(gsd2)) / (P * P * npos)
    dp = torch.zeros(B, P * P, K, dtype=torch.float64, device=dev)
    dp_b = torch.zeros_like(dp)
    dc, dc_b = {}, {}
    loss, loss_b = 0.0, 0.0
    ar = torch.arange(P, device=dev, dtype=torch.float32)
    for b in range(B):
        if len(sel[b]) == 0:
            continue
        tb, ok = targets(env, mk[b], P)
        a = np.asarray(sel[b])
        gi = r['matched_idx'][b, a]
        boxes = torch.from_numpy(tg[b][gi, :4]).to(dev)
        t = torch.from_numpy(tb[gi].reshape(len(a), -1)).to(dev).double()
        x1, x2 = torch.minimum(boxes[:, 0] * P, boxes[:, 2] * P), torch.maximum(boxes[:, 0] * P, boxes[:, 2] * P)
        y1, y2 = torch.minimum(boxes[:, 1] * P, boxes[:, 3] * P), torch.maximum(boxes[:, 1] * P, boxes[:, 3] * P)
        x1, x2 = (x1 - 1).clamp_min(0), (x2 + 1).clamp_max(P)
        y1, y2 = (y1 - 1).clamp_min(0), (y2 + 1).clamp_max(P)
        inside = ((ar[None, None, :] >= x1[:, None, None]) & (ar[None, None, :] < x2[:, None, None]) &
                  (ar[None, :, None] >= y1[:, None, None]) & (ar[None, :, None] < y2[:, None, None])).reshape(len(a), -1)
        area = ((boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1])).double()
        w = (1 / area) * (n_all[b] / len(a) if n_all[b] > len(a) else 1.0)
        pr = torch.from_numpy(proto[b].reshape(P * P, K)).to(dev).double()
        c = torch.from_numpy(coef[b, a]).to(dev).double()
        z = c @ pr.T                                                  # [n, P*P]
        ez = 2 * (K * U * (c.abs() @ pr.abs().T) + 5 * 2.0 ** -23 * (1 + z.abs()))
        G, L, p = bce_unit(z, t)
        # the fp32 rounding of 1 + e may go either way under expf's 2 ulp: p is uncertain by 2u absolute (p - t cancels near p = 1)
        inner = (p > 0) & (p < 1)
        dG = torch.full_like(G, 4 * U)
        dL = torch.where(inner, (4 * U * (t / p.clamp_min(1e-300) + (1 - t) / (1 - p).clamp_min(1e-300))).clamp_max(100), 0.0)
        for s in (-1, 1):
            Gs, Ls, _ = bce_unit(z + s * ez, t)
            dG, dL = torch.maximum(dG, (Gs - G).abs() + 4 * U), torch.maximum(dL, (Ls - L).abs())
        wg = (w * gscale)[:, None]
        g = torch.where(inside, wg * G, 0.0)
        gerr = torch.where(inside, wg.abs() * (dG + 12 * U * G.abs()), 0.0)
        n = len(a)
        dp[b] = g.T @ c
        dp_b[b] = 2 * (gerr.T @ c.abs() + n * U * (g.abs().T @ c.abs()))
        chain = 5 + P * P / 32
        dcv = g @ pr
        dcb = 2 * (gerr @ pr.abs() + chain * U * (g.abs() @ pr.abs()))
        for i, ai in enumerate(a):
            dc[(b, int(ai))], dc_b[(b, int(ai))] = dcv[i], dcb[i]
        Lt = torch.where(inside, L, 100 * t)
        dLt = torch.where(inside, dL, 0.0)
        loss += float((w[:, None] * Lt).sum())
        loss_b += float((w.abs()[:, None] * (dLt + (8 + n + 5) * U * Lt.abs())).sum()) * 2
        if not ok.all():
            bad = torch.from_numpy(~ok[gi].reshape(len(a), -1)).to(dev)
            bad_pix = bad.any(0)
            dp_b[b][bad_pix] = float('inf')
            for i, ai in enumerate(a):
                dc_b[(b, int(ai))] = dc_b[(b, int(ai))] + float('inf') * bool(bad[i].any())
    k = env.cfg.mask_alpha / (P * P * npos)
    return dp, dp_b, dc, dc_b, loss * k, loss_b * k + 2 * U * abs(loss * k)


def check_mask(env, r, tg, mk, proto, coef, sel, n_all, P, gsd2, tag):
    dp, dp_b, dc, dc_b, loss, loss_b = mask_reference(env, r, tg, mk, proto, coef, sel, n_all, P, gsd2)
    K = proto.shape[-1]
    kd = torch.from_numpy(r['d_proto'].reshape(proto.shape[0], P * P, K)).to(env.dev).double()
    w1 = report(f'{tag} d_proto', (kd - dp).abs().cpu().numpy(), dp_b.cpu().numpy())
    errs, bnds = [], []
    for (b, a), v in dc.items():
        errs.append((torch.from_numpy(r['d_coef'][b, a]).to(env.dev).double() - v).abs().cpu().numpy())
        bnds.append(dc_b[(b, a)].cpu().numpy())
    w2 = report(f'{tag} d_coef', np.concatenate(errs), np.concatenate(bnds))
    print(f'{tag} mask loss {r["losses"][2]:.8g} vs fp64 {loss:.8g}: err/bound {abs(r["losses"][2] - loss) / loss_b:.3g}')
    assert abs(r['losses'][2] - loss) <= loss_b
    return w1, w2


@pytest.mark.parametrize('P,K', [(138, 32), (138, 17), (32, 1), (32, 31)])
def test_mask_loss_saturated_logits_and_crop_edges(env, P, K):
    """One gt per image and pos_iou_thr = 1.5: only the forced match is positive, so d_proto[pix, :] is one mask's gradient times
    its coefficients.  z spans [-100, 100]; the boxes are ordinary, reversed, narrower than a pixel, partly outside the image, and
    just past the right edge (a crop that holds no pixel)."""
    A, rng = env.A, np.random.default_rng(P * 100 + K)
    S = 550 if P == 138 else 128
    boxes = [[0.2, 0.3, 0.6, 0.7], [0.7, 0.8, 0.3, 0.25], [0.5, 0.5, 0.5 + 0.4 / P, 0.5 + 0.6 / P], [-0.2, 0.6, 0.35, 1.3],
             [1 + 0.5 / P, 0.2, 1 + 0.9 / P, 0.5]]
    B = len(boxes)
    tg = [f32([bx + [float(3 * b + 1)]]) for b, bx in enumerate(boxes)]
    mk = [ragged_masks(np.random.default_rng(S + b), 4, S)[b % 4:b % 4 + 1] for b in range(B)]
    labels, idx, _ = assign(env, tg, 1.5, 0.4)
    assert ((labels > 0).sum(1) == 1).all()
    sel = [list(np.flatnonzero(labels[b] > 0)) for b in range(B)]
    coef = f32(rng.uniform(-1, 1, (B, A, K)))
    proto = np.zeros((B, P, P, K), np.float64)
    for b in range(B):
        a = sel[b][0]
        coef[b, a, 0] = 1.0
        zt = rng.uniform(-100, 100, P * P)
        zt[:8] = [-100, -40, -30, -17, 17, 30, 40, 100]
        pr = rng.uniform(0, 3, (P * P, K))
        pr[:, 0] = zt - pr[:, 1:] @ coef[b, a, 1:].astype(np.float64)
        proto[b] = pr.reshape(P, P, K)
    proto = f32(proto)
    gsd = (1.0, 1.0, 0.8, 1.0)
    r = call(env, tg, mk, np.zeros((B, A, NCLS), np.float32), coef=coef, proto=proto, P=P, K=K, grad_scale=gsd,
             pos_iou_thr=1.5)
    assert np.array_equal(r['labels'], labels)
    pos = labels > 0
    assert np.array_equal(r['matched_idx'][pos], idx[pos])
    assert (r['d_coef'][~pos] == 0).all()
    check_mask(env, r, tg, mk, proto, coef, sel, [1] * B, P, gsd[2], f'mask P={P} K={K}')


@pytest.mark.parametrize('mtt', [1, 100, 128])
def test_mask_loss_random_subset(env, mtt):
    """More positives than masks_to_train: the subset is read back from the non-zero rows of d_coef and the reference is
    recomputed on exactly that subset, with the n_all / n reweighting.  masks_to_train = 129 is refused."""
    A, B, P, K, rng = env.A, 2, 32, 8, np.random.default_rng(mtt)
    tg, _ = synth.train_targets(3, B, 128, n=60)
    mk = [ragged_masks(rng, len(t), 128) for t in tg]
    labels, _, _ = assign(env, tg, 0.3, 0.2)
    n_all = (labels > 0).sum(1)
    assert (n_all > 128).all()
    coef = f32(np.tanh(rng.normal(0, 1, (B, A, K))))
    proto = f32(np.maximum(rng.normal(0, 2, (B, P, P, K)), 0))
    gsd = (1.0, 1.0, 1.0, 1.0)
    r = call(env, tg, mk, np.zeros((B, A, NCLS), np.float32), coef=coef, proto=proto, P=P, K=K, grad_scale=gsd, pos_iou_thr=0.3,
             neg_iou_thr=0.2, masks_to_train=mtt)
    assert np.array_equal(r['labels'], labels)
    sel = [list(np.flatnonzero((r['d_coef'][b] != 0).any(-1))) for b in range(B)]
    for b in range(B):
        assert len(sel[b]) == min(n_all[b], mtt), (len(sel[b]), n_all[b], mtt)
        assert (labels[b, sel[b]] > 0).all()
    check_mask(env, r, tg, mk, proto, coef, sel, list(n_all), P, gsd[2], f'mask subset {mtt}')
    if mtt == 128:
        bad = call(env, tg, mk, np.zeros((B, A, NCLS), np.float32), coef=coef, proto=proto, P=P, K=K, masks_to_train=129, sentinel=-3,
                   check=False)
        assert bad['status'] != 0
        assert (bad['labels'] == -3).all() and (bad['d_proto'] == -3).all() and (bad['losses'] == -3).all()


# ------------------------------------------------------------------------------------------------
# down-sampled targets, bit for bit
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('S', [550, 544, 512, 128])
def test_downsampled_targets_bit_exact(env, S):
    """Seg logits 0: d_seg = gs (0.5 - t) at Hs.  Proto 0, coefficients 1, one positive per image whose gt is the whole image (the
    crop covers every pixel): d_proto = w gscale (0.5 - t) at P.  Both signs give the kernel's binarised targets."""
    A, B, rng = env.A, 4, np.random.default_rng(S)
    P, Hs = -(-S // 4), -(-S // 8)
    tg = [f32([[0.0, 0.0, 1.0, 1.0, float(b)]]) for b in range(B)]
    mk = [ragged_masks(np.random.default_rng(S + b), 4, S)[b:b + 1] for b in range(B)]
    r = call(env, tg, mk, np.zeros((B, A, NCLS), np.float32), coef=np.ones((B, A, 4), np.float32), P=P, Hs=Hs, K=4, pos_iou_thr=1.5)
    assert ((r['labels'] > 0).sum(1) == 1).all()
    for b in range(B):
        for size, got, name in ((P, r['d_proto'][b, ..., 0] < 0, 'P'), (Hs, r['d_seg'][b, b] < 0, 'Hs')):
            ref, ok = targets(env, mk[b], size)
            assert ok.all(), 'torch CPU and CUDA disagree'
            nz = r['d_proto'][b, ..., 0] if name == 'P' else r['d_seg'][b, b]
            assert (nz != 0).all()
            diff = np.argwhere(got != ref[0])
            assert len(diff) == 0, f'S={S} image {b} at {name}={size}: {len(diff)} target pixels differ, e.g. {diff[:6].tolist()}'


# ------------------------------------------------------------------------------------------------
# matching at COCO scale
# ------------------------------------------------------------------------------------------------
def coco_gts(env, rng, n):
    """n gts: random boxes, gts smaller than every anchor, identical duplicates, pairs sharing a best anchor, whole-image gts and
    gts snapped to anchor edges so that an IoU lands exactly on 0.5 / 0.4."""
    a = env.anchors
    corners = np.concatenate([a[:, :2] - a[:, 2:] / np.float32(2), a[:, :2] + a[:, 2:] / np.float32(2)], 1).astype(np.float32)
    g = [rect_gts(rng, n - 52, 0.02, 0.6)]
    tiny = rng.uniform(0.1, 0.9, (12, 2))
    g.append(f32(np.concatenate([tiny, tiny + 0.004, np.full((12, 1), 5.0)], 1)))
    g.append(np.repeat(g[0][:6], 2, 0))                                 # identical duplicates
    sh = g[0][6:12].copy()
    sh[:, :4] += f32(1e-4)
    g.append(np.concatenate([g[0][6:12], sh]))                          # pairs sharing a best anchor
    g.append(f32([[0, 0, 1, 1, 7], [0, 0, 1, 1, 9]]))
    pick = rng.choice(len(a), 14, replace=False)
    snap = []
    for j, i in enumerate(pick):
        x1, y1, x2, y2 = corners[i]
        f = np.float32(2.0 if j % 2 == 0 else 2.5)
        snap.append([x1, y1, x1 + f * (x2 - x1), y2, 11.0])
    g.append(f32(snap))
    out = f32(np.concatenate(g))
    assert len(out) == n, len(out)
    return out


def test_matching_at_coco_scale(env):
    A, rng = env.A, np.random.default_rng(3)
    big = coco_gts(env, rng, 256)
    small = rect_gts(rng, 4)
    empty = np.zeros((0, 5), np.float32)
    iou = tt.pairwise_iou(torch.from_numpy(big[:, :4]), torch.from_numpy(np.concatenate(
        [env.anchors[:, :2] - env.anchors[:, 2:] / 2, env.anchors[:, :2] + env.anchors[:, 2:] / 2], 1)))
    assert bool((iou == np.float32(0.5)).any()) and bool((iou == np.float32(0.4)).any()), 'no IoU lands exactly on a threshold'
    for order in ((big, small, empty), (empty, big, small), (small, empty, big)):
        tg = list(order)
        mk = [np.zeros((len(t), 64, 64), np.float32) for t in tg]
        labels, idx, off = assign(env, tg)
        r = call(env, tg, mk, np.zeros((3, A, NCLS), np.float32), grads=False)
        assert np.array_equal(r['labels'], labels)
        assert np.array_equal(r['matched_idx'], idx)
        assert np.array_equal(r['offsets'][..., :2], off[..., :2])
        ulp = np.spacing(np.abs(off[..., 2:]).astype(np.float32))
        # log: torch's CPU logf and CUDA's logf are each within 1 ulp, then / 0.2 rounds: 2 ulp of the offset
        assert (np.abs(r['offsets'][..., 2:].astype(np.float64) - off[..., 2:]) <= 2 * ulp).all()
    # the later gt wins a shared anchor; gts smaller than every anchor are forced positive
    ia = iou.max(1)[1].numpy()
    for j in range(len(big)):
        later = [k for k in range(j + 1, len(big)) if ia[k] == ia[j]]
        want = later[-1] if later else j
        assert r['matched_idx'][2, ia[j]] == want and r['labels'][2, ia[j]] > 0
    # 257 gts in one image: refused, outputs untouched
    tg = [np.concatenate([big, big[:1]]), small]
    mk = [np.zeros((len(t), 64, 64), np.float32) for t in tg]
    bad = call(env, tg, mk, np.zeros((2, A, NCLS), np.float32), sentinel=-5, check=False)
    assert bad['status'] != 0
    for k in ('labels', 'matched_idx', 'offsets', 'd_cls', 'd_box', 'd_coef', 'd_proto', 'losses'):
        assert (bad[k] == -5).all(), k


# ------------------------------------------------------------------------------------------------
# semantic loss
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('NC', [2, 21, 81, 129])
def test_semantic_loss(env, NC):
    """Overlapping same-class masks (the target is their max), classes 0 and NC - 2, and ld_seg > NC - 1: the padding columns of
    d_seg must be exactly 0 (the input's padding holds NaN, which the kernels must not read)."""
    A, B, S, rng = env.A, 2, 550, np.random.default_rng(NC)
    Hs = -(-S // 8)
    tg, mk = [], []
    for b in range(B):
        cl = [0, 0, 0, NC - 2, int(rng.integers(0, NC - 1))]
        tg.append(f32(np.concatenate([rect_gts(rng, len(cl), 0.1, 0.5)[:, :4], np.asarray(cl, np.float32)[:, None]], 1)))
        mk.append(ragged_masks(rng, len(cl), S))
    seg = rng.normal(0, 8, (B, NC - 1, Hs, Hs))
    seg[:, :, 0, :4] = [-80, 80, -20, 20]
    seg = f32(seg)
    gs = (1.0, 1.0, 1.0, 0.6)
    ld = NC - 1 + 3
    r = call(env, tg, mk, np.zeros((B, A, NC), np.float32), seg=seg, Hs=Hs, grad_scale=gs, ld_seg=ld)
    assert (r['d_seg_nhwc'][..., NC - 1:] == 0).all()
    t = np.zeros((B, NC - 1, Hs, Hs))
    for b in range(B):
        tb, ok = targets(env, mk[b], Hs)
        assert ok.all()
        for j, c in enumerate(tg[b][:, 4].astype(int)):
            t[b, c] = np.maximum(t[b, c], tb[j])
    v = seg.astype(np.float64)
    p = 1 / (1 + np.exp(-v))
    g = float(np.float32(env.cfg.semantic_alpha / np.float32(Hs * Hs * B)) * np.float32(gs[3]))
    ref = g * (p - t)
    report(f'd_seg NC={NC}', np.abs(r['d_seg'] - ref), 2 * (abs(g) * (6 * U * p + U * np.abs(p - t) + 2.0 ** -140) + 3 * U * np.abs(ref)))
    terms = np.maximum(v, 0) - v * t + np.log1p(np.exp(-np.abs(v)))
    k = env.cfg.semantic_alpha / (Hs * Hs * B)
    ref_l = k * terms.sum()
    bnd = 2 * k * ((NC + 8) * U * terms.sum() + 4 * U * (np.abs(v) + 1).sum()) + 2 * U * ref_l
    print(f'semantic loss NC={NC} {r["losses"][3]:.8g} vs fp64 {ref_l:.8g}: err/bound {abs(r["losses"][3] - ref_l) / bnd:.3g}')
    assert abs(r['losses'][3] - ref_l) <= bnd


# ------------------------------------------------------------------------------------------------
# stability
# ------------------------------------------------------------------------------------------------
def test_two_identical_calls(env):
    """Everything but the float-atomic sums is bit-identical across calls; d_coef (one atomic per warp and coefficient) and the
    losses agree within the reordering of their fp32 sums."""
    A, B, P, K, rng = env.A, 2, 69, 32, np.random.default_rng(11)
    tg = [rect_gts(rng, 20, 0.05, 0.5) for _ in range(B)]
    mk = [ragged_masks(rng, len(t), 276) for t in tg]
    args = dict(box=f32(rng.normal(0, 1, (B, A, 4))), coef=f32(np.tanh(rng.normal(0, 1, (B, A, K)))),
                proto=f32(np.maximum(rng.normal(0, 1, (B, P, P, K)), 0)), seg=f32(rng.normal(0, 2, (B, NCLS - 1, 35, 35))), P=P, Hs=35)
    cls = f32(rng.normal(0, 5, (B, A, NCLS)))
    r1, r2 = call(env, tg, mk, cls, **args), call(env, tg, mk, cls, **args)
    for k in ('labels', 'neg', 'd_cls', 'd_box', 'd_proto', 'd_seg'):
        assert np.array_equal(r1[k], r2[k]), k
    scale = np.abs(r1['d_coef']).max(-1, keepdims=True)
    assert (np.abs(r1['d_coef'] - r2['d_coef']) <= 1e-4 * scale).all()             # 1e-4 of the row's largest coefficient gradient
    assert np.allclose(r1['losses'], r2['losses'], rtol=1e-6, atol=0)
