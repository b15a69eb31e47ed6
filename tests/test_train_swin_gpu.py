"""GPU: training `swin_tiny_coco` on the native engine (csrc/train.cu's Swin-T program, csrc/swin_train.cu) against the torch-autograd
checker of tests/swin_train_torch.py, with the engine's own stochastic-depth draws handed to the checker.

  * backward at the engine's own activations (subst): every parameter gradient, the losses;
  * window attention backward against fp64 at the engine's operands, padding tokens' dK / dV in the qkv bias gradient;
  * stochastic depth: reproducible per seed, block 0 never dropped, keep rate per block;
  * AdamW steps reduce the loss, and inference reads the trained parameters."""
import math

import numpy as np
import pytest
import torch

import swin_train_torch as st
import train_checks as tc

pytestmark = pytest.mark.gpu


def _batch(dev, S, B):
    from oracle import synth
    img = torch.from_numpy(synth.image_batch(11, B, S)).to(dev)
    tg, mk = synth.train_targets(5, B, S)
    return img, [torch.from_numpy(t).to(dev) for t in tg], [torch.from_numpy(m).to(dev) for m in mk]


def _engine_step(dev, S, B, precision, seed=0):
    net = tc.make_train_net('swin_tiny', S, B, dev)
    net.cfg.train_precision = precision
    img, tgt, mks = _batch(dev, S, B)
    torch.manual_seed(seed)
    losses = net(img, tgt, mks)
    sum(losses).backward()
    torch.cuda.synchronize()
    eng = next(iter(net._train_engines.values()))
    return net, eng, losses, (img, tgt, mks)


@pytest.mark.parametrize('S,precision', [(128, 'bf16'), (128, 'fp16'), (550, 'bf16'), (550, 'fp16')])
def test_swin_engine_backward_at_its_own_activations(cuda, S, precision):
    """The checker evaluated AT the engine's stored activations with the engine's drop-path masks: what is compared is the backward
    arithmetic (LayerNorm, attention, GELU, merge, residual and the linear layers' dgrad / weight-gradient GEMMs) against fp32 autograd."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    B = 2
    net, eng, losses, (img, tgt, mks) = _engine_step(cuda, S, B, precision)
    masks = eng.read_output('drop_path')
    assert set(np.unique(masks.cpu().numpy())) <= {0.0, 1.0}
    ref = tc.make_train_net('swin_tiny', S, B, cuda)
    act = torch.bfloat16 if precision == 'bf16' else torch.float16
    cache = {}

    def subst(name):
        if name not in cache:
            try:
                if name.startswith('out.'):
                    v = eng.read_output(name[4:])
                    cache[name] = v[..., :80].permute(0, 3, 1, 2).contiguous() if name == 'out.seg' else v
                else:
                    cache[name] = eng.read(name)
            except Exception:
                cache[name] = None
        return cache[name]
    ref_losses = st.training_step_forward(ref, img, tgt, mks, masks, {}, act, subst)
    sum(ref_losses).backward()
    assert sum(v is not None for v in cache.values()) > 150
    got, want = [float(l.detach()) for l in losses], [float(l.detach()) for l in ref_losses]
    assert np.allclose(got, want, rtol=1e-4), (got, want)
    rp = dict(ref.named_parameters())
    rels = {}
    for n, p in net.named_parameters():
        assert p.grad is not None and rp[n].grad is not None, n                   # the engine binds every parameter of the module
        g, r = p.grad.cpu().numpy(), rp[n].grad.cpu().numpy()
        rels[n] = (tc.rel(g, r), tc.cos(g, r), float(np.linalg.norm(r)))
    worst = sorted(rels.items(), key=lambda kv: -kv[1][0])[:5]
    print(f'swin@{S} {precision}: median rel {np.median([v[0] for v in rels.values()]):.3g}, worst', worst, 'launches/step', eng.launches_per_step())
    tol_max, tol_med = (0.15, 3e-2) if precision == 'bf16' else (2e-2, 4e-3)
    for n, (r, c, nr) in rels.items():
        assert r < tol_max and (c > 0.99 or r == 0), (n, r, c, nr)
    assert float(np.median([v[0] for v in rels.values()])) < tol_med


def _attention_fp64(qkv_tok, bias, table, H, heads, shift):
    """fp64 shifted-window attention of modules/swin_transformer.py over [B, H*H, 3C] tokens, padding tokens = the qkv bias."""
    from oracle import forward_torch as ft
    B, C, ws = qkv_tok.shape[0], qkv_tok.shape[-1] // 3, ft.SWIN_WS
    Hp = -(-H // ws) * ws
    padded = bias.view(1, 1, 1, -1).expand(B, Hp, Hp, 3 * C).clone()
    padded[:, :H, :H] = qkv_tok.view(B, H, H, 3 * C)
    if shift:
        padded = torch.roll(padded, shifts=(-shift, -shift), dims=(1, 2))
    win = padded.view(B, Hp // ws, ws, Hp // ws, ws, 3 * C).permute(0, 1, 3, 2, 4, 5).reshape(-1, ws * ws, 3 * C)
    B_, N = win.shape[0], ws * ws
    qkv = win.reshape(B_, N, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    attn = (qkv[0] * (C // heads) ** -0.5) @ qkv[1].transpose(-2, -1)
    attn = attn + table[ft._rel_index(ws).view(-1).to(table.device)].view(N, N, -1).permute(2, 0, 1).unsqueeze(0)
    if shift:
        mask = ft._shift_mask(Hp, Hp, ws, shift).to(attn)
        nW = mask.shape[0]
        attn = (attn.view(B_ // nW, nW, heads, N, N) + mask.unsqueeze(1).unsqueeze(0)).view(-1, heads, N, N)
    o = (attn.softmax(-1) @ qkv[2]).transpose(1, 2).reshape(B_, N, C)
    o = o.view(B, Hp // ws, Hp // ws, ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(B, Hp, Hp, C)
    if shift:
        o = torch.roll(o, shifts=(shift, shift), dims=(1, 2))
    return o[:, :H, :H].reshape(B, H * H, C)


def test_swin_attention_backward_vs_fp64_at_engine_operands(cuda):
    """dqkv, the relative-position table gradient and the qkv bias gradient of the engine's attention backward against fp64 autograd
    at the engine's own qkv and output gradient, 550x550: grids 138 / 69 / 35 / 18 (windows padded to 140 / 70 / 35 / 21), shifted and
    unshifted blocks.  Where the grid is padded, the padding tokens' dK / dV are part of the bias gradient and of no token's gradient."""
    S, B = 550, 2
    net, eng, _, _ = _engine_step(cuda, S, B, 'fp16')
    P = dict(net.named_parameters())
    checked = 0
    for p, heads, shift in (('backbone.layers.0.blocks.0', 3, 0), ('backbone.layers.0.blocks.1', 3, 3), ('backbone.layers.1.blocks.1', 6, 3),
                            ('backbone.layers.2.blocks.4', 12, 0), ('backbone.layers.3.blocks.1', 24, 3)):
        tok = lambda t: t.flatten(2).transpose(1, 2).double()
        qkv = tok(eng.read(p + '.attn.qkv')).requires_grad_(True)
        H = int(math.isqrt(qkv.shape[1]))
        dout = tok(eng.read(p + '.attn', grad=True))
        if not bool(dout.any()):                                              # both images dropped this attention branch
            continue
        checked += 1
        bias = P[p + '.attn.qkv.bias'].detach().double().requires_grad_(True)
        table = P[p + '.attn.relative_position_bias_table'].detach().double().requires_grad_(True)
        o = _attention_fp64(qkv, bias, table, H, heads, shift)
        o.backward(dout)
        dq = tok(eng.read(p + '.attn.qkv', grad=True))
        e = tc.rel(dq.cpu().numpy(), qkv.grad.cpu().numpy())
        et = tc.rel(P[p + '.attn.relative_position_bias_table'].grad.cpu().numpy(), table.grad.cpu().numpy())
        # the bias gradient: the tokens' dqkv column sums (fp64 of the engine's dqkv) + the padding tokens' dK / dV (bias.grad here: the
        # padding tokens are the only place the bias enters this fp64 attention)
        want_b = dq.sum((0, 1)) + bias.grad
        eb = tc.rel(P[p + '.attn.qkv.bias'].grad.cpu().numpy(), want_b.cpu().numpy())
        pad_share = float(bias.grad.norm() / want_b.norm())
        print(p, H, 'dqkv', e, 'table', et, 'bias', eb, 'padding share of the bias gradient', pad_share)
        assert e < 5e-3 and et < 1e-3 and eb < 1e-3, (p, e, et, eb)
        if H % 7:
            assert pad_share > 1e-3, (p, pad_share)
    assert checked >= 3


def test_swin_drop_path_masks(cuda):
    """Same seed, same masks; another seed, other masks; block 0 (rate 0) never dropped; keep rate per block = 1 - p_i within 5 sigma."""
    S, B, steps = 128, 2, 160
    net = tc.make_train_net('swin_tiny', S, B, cuda)
    img, tgt, mks = _batch(cuda, S, B)
    eng = None
    draws = []
    with torch.no_grad():
        for k in range(steps):
            torch.manual_seed(1000 + k)
            net(img, tgt, mks)
            eng = eng or next(iter(net._train_engines.values()))
            draws.append(eng.read_output('drop_path').cpu().numpy())
        torch.manual_seed(1000)
        net(img, tgt, mks)
        again = eng.read_output('drop_path').cpu().numpy()
    d = np.stack(draws)                                                       # [steps, B, 12, 2]
    assert np.array_equal(again, d[0])
    assert sum(not np.array_equal(d[i], d[0]) for i in range(1, steps)) > steps // 2
    assert (d[:, :, 0] == 1).all()
    n = steps * B * 2
    for blk, p in enumerate(st.drop_rates()):
        rate = d[:, :, blk].mean()
        sigma = math.sqrt(max(p * (1 - p), 1e-12) / n)
        assert abs(rate - (1 - p)) < 5 * sigma + 1e-9, (blk, rate, 1 - p, sigma)
    assert abs(np.corrcoef(d[:, :, 11, 0].ravel(), d[:, :, 11, 1].ravel())[0, 1]) < 0.2      # the two branches draw independently


def test_swin_adamw_steps_reduce_the_loss_and_inference_reads_the_trained_parameters(cuda):
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    S, B = 128, 2
    net = tc.make_train_net('swin_tiny', S, B, cuda)
    cfg = net.cfg
    opt = torch.optim.AdamW(net.parameters(), lr=cfg.lr, weight_decay=0.05)        # train.py's optimizer for swin_tiny_coco
    img, tgt, mks = _batch(cuda, S, B)
    torch.manual_seed(0)
    hist = []
    for _ in range(8):
        losses = net(img, tgt, mks)
        total = sum(losses)
        opt.zero_grad()
        total.backward()
        opt.step()
        hist.append(float(total.detach()))
    print('AdamW losses', hist)
    assert all(np.isfinite(hist)) and min(hist[4:]) < 0.95 * hist[0], hist        # (measured on an H100: 117 -> 99 after 4 steps -> 91 after 8)
    net.eval()
    fresh = Yolact(net.cfg)
    fresh.load_state_dict(net.state_dict(), strict=True)
    fresh = fresh.to(cuda).eval()
    with torch.no_grad():
        a, b = net(img), fresh(img)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize('precision', ['bf16', 'fp16'])
def test_swin_engine_losses_vs_reference_golden(cuda, precision):
    """The engine's train-mode forward against the reference (tests/golden/train_swin.npz, minted on the CPU with the draws the engine
    makes for the golden step's seed): the same masks, and the four losses within 5 % (16-bit activations)."""
    from conftest import load_golden
    from swin_golden import S, B, SEED_STEP
    g = load_golden('train_swin.npz')
    net, eng, losses, _ = _engine_step(cuda, S, B, precision, seed=SEED_STEP)
    assert np.array_equal(eng.read_output('drop_path').cpu().numpy(), g['masks'])
    got = np.asarray([float(l.detach()) for l in losses])
    print(precision, 'engine losses', got.tolist(), 'reference', g['losses'].tolist())
    assert np.allclose(got, g['losses'], rtol=5e-2), (got, g['losses'])


def _tok(t):
    return t.flatten(2).transpose(1, 2).double()


def _rounded(got, want, u, what):
    """got = want rounded to the 16-bit activation type (unit roundoff u), up to fp32 arithmetic: |got - want| <= u |want| + slack."""
    err = (got - want).abs()
    bound = 1.01 * u * want.abs() + 1e-5 * float(want.abs().max()) + 1e-7
    assert bool((err <= bound).all()), (what, float((err - bound).max()), float(err.max()))


def _ln64(x, g, b, dy=None):
    """fp64 LayerNorm; with dy: (y, dx, dgamma, dbeta) by autograd."""
    import torch.nn.functional as F
    x = x.detach().double().requires_grad_(dy is not None)
    g = g.detach().double().requires_grad_(dy is not None)
    b = b.detach().double().requires_grad_(dy is not None)
    y = F.layer_norm(x, (x.shape[-1],), g, b, 1e-5)
    if dy is None:
        return y
    y.backward(dy)
    return y, x.grad, g.grad, b.grad


def _unmerge(dm, H):
    """The inverse of the patch-merging gather: [B, Ho*Ho, 4C] -> [B, H*H, C] (padding positions dropped)."""
    B, L, C4 = dm.shape
    Ho, C = int(math.isqrt(L)), C4 // 4
    d = dm.view(B, Ho, Ho, C4)
    out = torch.zeros(B, 2 * Ho, 2 * Ho, C, dtype=dm.dtype, device=dm.device)
    out[:, 0::2, 0::2], out[:, 1::2, 0::2], out[:, 0::2, 1::2], out[:, 1::2, 1::2] = d[..., :C], d[..., C:2 * C], d[..., 2 * C:3 * C], d[..., 3 * C:]
    return out[:, :H, :H].reshape(B, H * H, C)


@pytest.mark.parametrize('precision', ['bf16', 'fp16'])
def test_swin_ops_vs_fp64_at_engine_operands(cuda, precision):
    """Each Swin op of the engine against fp64 at the engine's own operands, 550x550 (grids 138 / 69 / 35 / 18, both odd merges), every
    input read from the engine's stored tensors: patch embedding (+ its weight / bias / norm gradients), LayerNorm forward and
    backward, attention forward, GELU forward and backward, the masked residual forward and backward, patch merging forward (exact)
    and backward.  Rounded outputs are bounded element by element by the 16-bit unit roundoff; the merge gather is bit for bit."""
    import torch.nn.functional as F
    from oracle import forward_torch as ft
    S, B = 550, 2
    u = 2.0 ** -8 if precision == 'bf16' else 2.0 ** -11
    net, eng, _, (img, _, _) = _engine_step(cuda, S, B, precision)
    P = {n: p.detach().double() for n, p in net.named_parameters()}
    G = {n: p.grad.double() for n, p in net.named_parameters()}
    rd = lambda n, grad=False: _tok(eng.read(n, grad=grad))
    masks = eng.read_output('drop_path').double()
    # ---- patch embedding: conv (fp32 in the engine) + LayerNorm; backward: the LayerNorm and the conv's weight / bias gradient ----
    pe = 'backbone.patch_embed'
    w = P[pe + '.proj.weight'].clone().requires_grad_(True)
    bb = P[pe + '.proj.bias'].clone().requires_grad_(True)
    ip = F.pad(img.double(), (0, (4 - S % 4) % 4, 0, (4 - S % 4) % 4))
    raw = F.conv2d(ip, w, bb, stride=4).flatten(2).transpose(1, 2)
    gn = P[pe + '.norm.weight'].clone().requires_grad_(True)
    bn = P[pe + '.norm.bias'].clone().requires_grad_(True)
    y = F.layer_norm(raw, (96,), gn, bn, 1e-5)
    _rounded(rd('patch_embed'), y.detach(), u, 'patch embedding')
    y.backward(rd('patch_embed', True))
    for n, r in ((pe + '.proj.weight', w.grad), (pe + '.proj.bias', bb.grad), (pe + '.norm.weight', gn.grad), (pe + '.norm.bias', bn.grad)):
        assert tc.rel(G[n].cpu().numpy(), r.cpu().numpy()) < 1e-3, (n, tc.rel(G[n].cpu().numpy(), r.cpu().numpy()))
    # ---- blocks: LayerNorms, attention, GELU, residuals (a shifted and an unshifted block per stage) ----
    rates, blk, prev = st.drop_rates(), 0, 'patch_embed'
    for s, depth in enumerate(ft.SWIN_DEPTHS):
        for b in range(depth):
            p = f'backbone.layers.{s}.blocks.{b}'
            x, x1 = rd(prev), rd(p + '.x1')
            _rounded(rd(p + '.norm1'), _ln64(x, P[p + '.norm1.weight'], P[p + '.norm1.bias']), u, p + '.norm1')
            _rounded(rd(p + '.norm2'), _ln64(x1, P[p + '.norm2.weight'], P[p + '.norm2.bias']), u, p + '.norm2')
            qkv = rd(p + '.attn.qkv')
            H = int(math.isqrt(qkv.shape[1]))
            o = _attention_fp64(qkv, P[p + '.attn.qkv.bias'], P[p + '.attn.relative_position_bias_table'], H, ft.SWIN_HEADS[s], 3 if b % 2 else 0)
            _rounded(rd(p + '.attn'), o, u, p + '.attn')
            h = rd(p + '.mlp.fc1')
            _rounded(rd(p + '.mlp.gelu'), F.gelu(h), u, p + '.gelu')
            cdf, pdf = 0.5 * (1 + torch.erf(h / math.sqrt(2))), torch.exp(-0.5 * h * h) / math.sqrt(2 * math.pi)
            _rounded(rd(p + '.mlp.fc1', True), rd(p + '.mlp.gelu', True) * (cdf + h * pdf), u, p + '.gelu backward')
            keep = 1 - float(np.float32(np.float32(0.2) * np.float32(blk)) / np.float32(11))
            for br, (a, yy, z) in enumerate(((x, p + '.attn.proj', p + '.x1'), (x1, p + '.mlp.fc2', p + '.out'))):
                sc = (masks[:, blk, br] / keep).view(B, 1, 1)
                _rounded(rd(z), a + sc * rd(yy), u, f'{p} residual {br}')
                dy, dz = rd(yy, True), rd(z, True)
                _rounded(dy, sc * dz, u, f'{p} residual {br} backward')
                assert bool((dy[masks[:, blk, br] == 0] == 0).all())              # a dropped branch gets no gradient
            prev, blk = p + '.out', blk + 1
        last = prev
        if s > 0:
            c = f'c{s + 2}'
            _rounded(rd(c), _ln64(rd(last), P[f'backbone.norm{s}.weight'], P[f'backbone.norm{s}.bias']), u, c)
        if s < 3:
            d = f'backbone.layers.{s}.downsample'
            xs = rd(last)
            H = int(math.isqrt(xs.shape[1]))
            gpad = F.pad(xs.view(B, H, H, -1), (0, 0, 0, H % 2, 0, H % 2))
            mg = torch.cat([gpad[:, 0::2, 0::2], gpad[:, 1::2, 0::2], gpad[:, 0::2, 1::2], gpad[:, 1::2, 1::2]], -1).reshape(B, -1, 4 * xs.shape[-1])
            assert torch.equal(rd(d + '.merge'), mg), d                             # the gather is exact
            yn, dx, dg, dbe = _ln64(mg, P[d + '.norm.weight'], P[d + '.norm.bias'], rd(d + '.norm', True))
            _rounded(rd(d + '.norm'), yn.detach(), u, d + '.norm')
            dmg = rd(d + '.merge', True)
            assert tc.rel(dmg.cpu().numpy(), dx.cpu().numpy()) < 2 * u, (d, 'LayerNorm backward', tc.rel(dmg.cpu().numpy(), dx.cpu().numpy()))
            assert tc.rel(G[d + '.norm.weight'].cpu().numpy(), dg.cpu().numpy()) < 1e-3
            assert tc.rel(G[d + '.norm.bias'].cpu().numpy(), dbe.cpu().numpy()) < 1e-3
            want = _unmerge(dmg, H)
            if s > 0:                                                            # the stage output also feeds backbone.norm<s>
                want = want + _ln64(rd(last), P[f'backbone.norm{s}.weight'], P[f'backbone.norm{s}.bias'], rd(f'c{s + 2}', True))[1]
                e = tc.rel(rd(last, True).cpu().numpy(), want.cpu().numpy())
                assert e < 2 * u, (d, 'merge + LayerNorm backward', e)
            else:
                assert torch.equal(rd(last, True), want), d                         # stage 1's output feeds the merge only: exact
            prev = d + '.reduction'
