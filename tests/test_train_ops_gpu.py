"""GPU: the training engine op by op against fp64, at the engine's own operands, at the benchmarked 550x550 shape.

Every operand is read back from the engine after the third (CUDA-graph replayed) step of a fixed input: activations and their
gradients through TrainEngine.read, weights as the fp32 master parameters rounded to the engine's 16-bit type, the gradients of
the dense network outputs from the torch loss checker at the engine's own outputs.  Each op is then recomputed in fp64 with torch
on the GPU from exactly those operands -- ReLU masks and batch statistics are the engine's by construction -- and compared
element by element under ONE error model:

    |eng - ref| <= u * rnd  +  eta * nr  +  C_ACC * 2^-24 * n * ref_abs

  u        unit roundoff of the 16-bit type (2^-8 bf16, 2^-11 fp16); 0 for fp32 results (parameter gradients, dense outputs)
  eta, nr  the absolute rounding error of a subnormal (2^-25 fp16: small gradients underflow), times the number of roundings
  rnd      the magnitude of every value the engine rounds to 16 bits on the way: |ref| for one store, plus the partial sum at
           each further accumulation (k_add16, residual epilogue, accumulating bilinear backward), plus a separately rounded
           contribution (stride-2 dgrad planes added by k_add16).  Without cancellation this is r * |ref| for r roundings.
  ref_abs  the same op on absolute values (|dY| * |W|, |dY|^T |X|, ...): what fp32 accumulation error scales with
  n        terms per output (Cin*k*k, pixels of a reduction ...) or the longest fp32 accumulation chain of a reduction
  C_ACC    stated once below: any fp32 sum of n terms, in any order, errs by at most gamma_n * sum|terms|, gamma_n ~ n * u_acc
           (Higham, Accuracy and Stability of Numerical Algorithms, 4.2); u_acc = 2^-23 covers an accumulator that truncates.

Exact ops (max-pool forward, phase merge, the residual-gradient copy) have no accumulation term.  Alongside the elementwise
rule, each tensor's relative L2 error must stay below L2_U * u * max(1, |rnd| / |ref|).
Bilinear interpolation is defined with the kernels' own fp32 source-coordinate arithmetic (as torch's fp32 kernels do), so the
reference weights are exact and a wrong weight or index shows up as an O(1) error.
"""
import gc
import math
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import train_checks as tc

pytestmark = pytest.mark.gpu

C_ACC = 2.0                  # fp32 accumulation: error <= C_ACC * 2^-24 * n * ref_abs
L2_U = 2.0                   # relative L2 error <= L2_U * u * max(1, |rnd| / |ref|)
U = {'bf16': 2.0 ** -8, 'fp16': 2.0 ** -11}
ETA = {'bf16': 2.0 ** -134, 'fp16': 2.0 ** -25}
DT = {'bf16': torch.bfloat16, 'fp16': torch.float16}
# the loss kernels agree with the torch loss checker to ~1e-7 relative (1e-5 is asserted); a 16-bit rounding of such a value is
# ambiguous only inside this window around it, and there the engine's and the checker's dY may differ by one ulp
LOSS_GRAD_EPS = 2.0 ** -16

# (arch, S, B, precision, big-mean stem channel, which bottleneck blocks are checked (None = all)[, config name[, class count]])
# The config name defaults to arch + '_coco'; the class count (background included) to the config's.  The class count sizes the
# head conv (3 (NC + 36) columns), the seg conv (NC - 1: Cout = 1 at two classes) and k_head_train / k_head_grad's row addressing.
CONFIGS = {
    'res50-550-B2-bf16': ('res50', 550, 2, 'bf16', False, None),
    'res101-550-B2-bf16': ('res101', 550, 2, 'bf16', False, {'0.0', '1.0', '2.0', '2.1', '2.22', '3.0'}),
    'res50-550-B3-fp16': ('res50', 550, 3, 'fp16', True, None),
    'res50-128-B2-fp16': ('res50', 128, 2, 'fp16', False, None),
    'pascal-550-B2-bf16': ('res50', 550, 2, 'bf16', False, None, 'res50_pascal'),
    'custom-res101-550-B2-fp16': ('res101', 550, 2, 'fp16', False, {'0.0', '1.0', '2.0', '2.1', '2.22', '3.0'}, 'res101_custom'),
    'nc2-128-B2-fp16': ('res50', 128, 2, 'fp16', False, None, None, 2),
    'nc129-128-B2-bf16': ('res50', 128, 2, 'bf16', False, None, None, 129),
}
MEAN_SHIFT = 30.0            # added to the image; channel 0 of the stem sees no zero padding, so its |mean| / std is ~ 3 * shift


# ------------------------------------------------------------------------------------------------
# the training graph, in the engine's op order (csrc/train.cu build()): backward contributions arrive in REVERSE of this order
# ------------------------------------------------------------------------------------------------
def graph(depth, R, NC, K):
    ops = []

    def conv(w, x, y, k, s, relu=False, bias=True, dense=False, name=None):
        ops.append(dict(kind='conv', w=w, b=(w.rsplit('.', 1)[0] + '.bias') if bias else None, x=x, y=y, k=k, s=s, relu=relu, dense=dense,
                        name=name or w.rsplit('.', 1)[0]))

    def bn(p, y, z, relu, res=None):
        ops.append(dict(kind='bn', p=p, y=y, z=z, relu=relu, res=res))

    conv('backbone.conv1.weight', 'img', 'stem.y', 7, 2, bias=False, name='stem')
    bn('backbone.bn1', 'stem.y', 'stem.z', True)
    ops.append(dict(kind='pool', x='stem.z', y='pool'))
    nblk = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3)}[depth]
    x, c = 'pool', []
    for st in range(4):
        for b in range(nblk[st]):
            p, s = f'backbone.layers.{st}.{b}', (2 if b == 0 and st > 0 else 1)
            conv(p + '.conv1.weight', x, p + '.conv1.y', 1, 1, bias=False)
            bn(p + '.bn1', p + '.conv1.y', p + '.bn1.z', True)
            conv(p + '.conv2.weight', p + '.bn1.z', p + '.conv2.y', 3, s, bias=False)
            bn(p + '.bn2', p + '.conv2.y', p + '.bn2.z', True)
            r = x
            if b == 0:
                conv(p + '.downsample.0.weight', x, p + '.downsample.y', 1, s, bias=False)
                bn(p + '.downsample.1', p + '.downsample.y', p + '.downsample.z', False)
                r = p + '.downsample.z'
            conv(p + '.conv3.weight', p + '.bn2.z', p + '.conv3.y', 1, 1, bias=False)
            bn(p + '.bn3', p + '.conv3.y', p + '.out', True, res=r)
            for o in ops[-7:]:
                o['block'] = f'{st}.{b}'
            x = p + '.out'
        c.append(x)
    lat = lambda i, y: conv(f'fpn.lat_layers.{i}.weight', c[i + 1], y, 1, 1)
    upadd = lambda coarse, fine: ops.append(dict(kind='upadd', x=coarse, y=fine))
    lat(2, 'p5_1'); lat(1, 'p4_1'); upadd('p5_1', 'p4_1'); lat(0, 'p3_1'); upadd('p4_1', 'p3_1')
    for i in (2, 1, 0):
        conv(f'fpn.pred_layers.{i}.0.weight', f'p{i + 3}_1', f'p{i + 3}', 3, 1, relu=True)
    conv('fpn.downsample_layers.0.0.weight', 'p5', 'p6', 3, 2, relu=True)
    conv('fpn.downsample_layers.1.0.weight', 'p6', 'p7', 3, 2, relu=True)
    q = 'p3'
    for i in (0, 2, 4):
        conv(f'proto_net.proto1.{i}.weight', q, f'proto1.{i}', 3, 1, relu=True)
        q = f'proto1.{i}'
    ops.append(dict(kind='up2x', x=q, y='proto.up'))
    conv('proto_net.proto2.0.weight', 'proto.up', 'proto2.0', 3, 1, relu=True)
    conv('proto_net.proto2.2.weight', 'proto2.0', 'out.proto', 1, 1, relu=True, dense=True)
    for l, lv in enumerate(('p3', 'p4', 'p5', 'p6', 'p7')):
        conv('prediction_layers.upfeature.0.weight', lv, f'head.f{l}', 3, 1, relu=True)
        conv('head', f'head.f{l}', f'out.head{l}', 3, 1, bias=False, dense=True, name='head')     # (its bias: Run.weight)
    conv('semantic_seg_conv.weight', 'p3', 'out.seg', 1, 1, dense=True)
    for i, o in enumerate(ops):
        o['seq'] = i
    return ops


# ------------------------------------------------------------------------------------------------
# one engine run per configuration
# ------------------------------------------------------------------------------------------------
class Run:
    def __init__(self, key, dev):
        arch, S, B, prec, shift, blocks, config, nc = (CONFIGS[key] + (None, None))[:8]
        self.key, self.arch, self.S, self.B, self.prec, self.blocks, self.dev = key, arch, S, B, prec, blocks, dev
        self.u, self.dt = U[prec], DT[prec]
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        from oracle import synth
        net = tc.make_train_net(arch, S, B, dev, config, nc)
        net.cfg.train_precision = prec
        img = torch.from_numpy(synth.image_batch(11, B, S)).to(dev)
        if shift:
            with torch.no_grad():                 # stem channel 0: only the 2x2 taps that never touch the zero padding, all positive
                w = net.backbone.conv1.weight
                keep = torch.zeros(7, 7, device=dev)
                keep[3:5, 3:5] = 1
                w[0] = w[0].abs() * keep
            img = img + MEAN_SHIFT
        tg, mk = synth.train_targets(5, B, S, num_classes=net.cfg.num_classes - 1)
        self.tg, self.mk = tg, mk
        tgt = [torch.from_numpy(t).to(dev) for t in tg]
        mks = [torch.from_numpy(m).to(dev) for m in mk]
        t0 = time.time()
        for step in range(3):                     # step 3 replays the captured forward / backward graphs, as the benchmark does
            if step == 2:
                for p in net.parameters():
                    p.grad = None
                self.bn_before = {n: b.detach().clone() for n, b in net.named_buffers() if n.endswith(('running_mean', 'running_var'))}
            losses = net(img, tgt, mks)
            sum(losses).backward()
        torch.cuda.synchronize()
        self.train_s = time.time() - t0
        self.net = net
        self.eng = next(iter(net._train_engines.values()))
        self.img = img.double().to(self.dt).double()              # the engine's stem reads the image as 16-bit
        self.params = dict(net.named_parameters())
        self.buffers = dict(net.named_buffers())
        cfg = net.cfg
        self.R, self.NC, self.K = len(cfg.aspect_ratios), cfg.num_classes, net.coef_dim
        self.ops = graph(net.depth, self.R, self.NC, self.K)
        self.results = []                                         # (kind, tap, extent, worst err/bound, rel L2, rel bound)
        self.extents = {}
        self._loss_grads()

    def rd(self, name, grad=False):
        if name == 'img':
            return self.img
        return self.eng.read(name, grad=grad).double()

    def q(self, t):
        return t.to(self.dt).double()

    def weight(self, w):
        if w == 'head':
            names = ('prediction_layers.conf_layer', 'prediction_layers.bbox_layer', 'prediction_layers.coef_layer.0')
            W = torch.cat([self.params[n + '.weight'].detach() for n in names])
            b = torch.cat([self.params[n + '.bias'].detach() for n in names])
            return self.q(W.double()), b.double()
        b = w.rsplit('.', 1)[0] + '.bias'
        return self.q(self.params[w].detach().double()), (self.params[b].detach().double() if b in self.params else None)

    # ---- the dense outputs' gradients: the torch loss checker at the engine's own outputs ----
    def _loss_grads(self):
        eng, B = self.eng, self.B
        out = {k: eng.read_output(k) for k in ('cls', 'box', 'coef', 'proto', 'seg')}
        self.outs = out
        cfg = self.net.cfg
        anchors = self.net.anchors
        anchors = (anchors.detach().cpu().numpy() if isinstance(anchors, torch.Tensor) else np.asarray(anchors)).reshape(-1, 4).astype(np.float32)
        self.anchors = anchors
        seg = out['seg'][..., :self.NC - 1].permute(0, 3, 1, 2).contiguous()
        c = lambda t: t.cpu().numpy()
        _, g = tc.torch_losses_and_grads(cfg, anchors, self.tg, self.mk, c(out['cls']), c(out['box']), c(out['coef']), c(out['proto']), c(seg))
        g = {k: torch.from_numpy(v).to(self.dev).double() for k, v in g.items()}
        # the engine's scatter into the dense convs' dY (k_head_grad, k_dense_to_haloed) -- as NCHW fp32 before the 16-bit store
        A, R, NC, K = self.anchors.shape[0], self.R, self.NC, self.K
        coef = out['coef'].double()
        dcoef = g['d_coef'] * (1 - coef * coef)
        self.dY_dense, off = {}, 0
        for l, lv in enumerate(('p3', 'p4', 'p5', 'p6', 'p7')):
            H = eng.read(lv).shape[-1]
            n = H * H * R
            parts = [g['d_cls'][:, off:off + n].reshape(B, H, H, R * NC), g['d_box'][:, off:off + n].reshape(B, H, H, R * 4),
                     dcoef[:, off:off + n].reshape(B, H, H, R * K)]
            self.dY_dense[f'out.head{l}'] = torch.cat(parts, -1).permute(0, 3, 1, 2).contiguous()
            off += n
        assert off == A
        self.dY_dense['out.proto'] = (g['d_proto'] * (out['proto'] > 0)).permute(0, 3, 1, 2).contiguous()
        self.dY_dense['out.seg'] = g['d_seg']

    def dY(self, op):
        """(dY as the engine's conv backward consumed it, ambiguity of its 16-bit rounding or None)."""
        if not op['dense']:
            return self.rd(op['y'], grad=True), None
        g = self.dY_dense[op['y']]
        w = LOSS_GRAD_EPS * (g.abs() + g.pow(2).mean().sqrt())
        lo, hi = self.q(g - w), self.q(g + w)
        return self.q(g), (hi - lo).abs()

    def checked(self, op):
        return self.blocks is None or 'block' not in op or op['block'] in self.blocks

    # ---- the one error rule ----
    def check(self, kind, tap, eng, ref, rnd, ref_abs, n, u=None, extent=None, exact=False, nr=1):
        """u=None: a 16-bit result (nr roundings of the engine's type); u given: an fp32 result, rnd = ambiguity of its inputs / u."""
        eng, ref = eng.double(), ref.double()
        err = (eng - ref).abs()
        bound = (self.u if u is None else u) * rnd if rnd is not None else torch.zeros_like(ref)
        if rnd is not None and u is None:
            bound = bound + ETA[self.prec] * nr
        u = self.u
        if not exact:
            bound = bound + C_ACC * 2.0 ** -24 * n * ref_abs
        worst = float((err / bound.clamp_min(1e-300)).max()) if bool((bound > 0).any()) else 0.0
        if bool(((bound == 0) & (err > 0)).any()):
            worst = float('inf')
        nref = float(ref.norm())
        rel = float((eng - ref).norm()) / max(nref, 1e-300)
        rel_bound = L2_U * u * max(1.0, float(rnd.norm()) / max(nref, 1e-300) if rnd is not None else 1.0)
        self.results.append((kind, tap, extent, worst, rel, rel_bound))
        if extent is not None:
            self.extents.setdefault(kind, set()).add(extent)

    def report(self):
        lines, bad = [], []
        for kind in sorted({r[0] for r in self.results}):
            rs = [r for r in self.results if r[0] == kind]
            w = max(rs, key=lambda r: r[3])
            lines.append(f'{self.key} {kind:14s} n={len(rs):3d} extents={sorted(self.extents.get(kind, []), key=str)} worst err/bound {w[3]:.3f} ({w[1]}) '
                         f'max rel L2 {max(r[4] for r in rs):.2e}')
            bad += [r for r in rs if not (r[3] <= 1.0 and r[4] <= r[5] + 1e-300 or (r[4] == 0 and r[3] <= 1.0))]
        return lines, bad


@pytest.fixture(scope='module', params=list(CONFIGS))
def run(request, cuda):
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    r = Run(request.param, cuda)
    yield r
    print(f'\n{r.key}: engine steps {r.train_s:.1f} s, total {time.time() - t0:.1f} s, peak memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB')
    del r
    gc.collect()
    torch.cuda.empty_cache()


def finish(r, kinds):
    lines, bad = r.report()
    for ln in lines:
        if ln.split()[1] in kinds:
            print(ln)
    bad = [b for b in bad if b[0] in kinds]
    assert not bad, 'over the bound (kind, tap, extent, err/bound, rel L2, rel L2 bound): ' + repr(bad[:12])


def interp_matrix(Hc, Hf, align, dev):
    """[Hf, Hc] bilinear weights with the kernels' fp32 arithmetic (src_index in kernels_simt.cu / train_kernels.cu)."""
    f32 = lambda v: torch.tensor(v, dtype=torch.float32)
    scale = f32((Hc - 1) / (Hf - 1)) if align else f32(Hc) / f32(Hf)
    M = torch.zeros(Hf, Hc, dtype=torch.float64)
    for j in range(Hf):
        if align:
            src = scale * f32(j)
        else:                                        # fmaf(scale, j + 0.5, -0.5): one rounding (the product is exact in fp64)
            src = torch.clamp((scale.double() * (j + 0.5) - 0.5).float(), min=0.0)
        i0 = min(int(src), Hc - 1)
        i1 = min(i0 + 1, Hc - 1)
        l1 = src - f32(i0)
        l0 = f32(1.0) - l1
        M[j, i0] += float(l0)
        M[j, i1] += float(l1)
    return M.to(dev)


def interp(x, Hf, align, absolute=False):
    M = interp_matrix(x.shape[-1], Hf, align, x.device)
    return torch.einsum('yi,bcij,xj->bcyx', M, x.abs() if absolute else x, M)


def interp_bwd(df, Hc, align):
    M = interp_matrix(Hc, df.shape[-1], align, df.device)
    return torch.einsum('yi,bcyx,xj->bcij', M, df, M)


def conv_ref(x, W, b, k, s, absolute=False):
    if absolute:
        x, W, b = x.abs(), W.abs(), (b.abs() if b is not None else None)
    return F.conv2d(x, W, b, stride=s, padding=k // 2)


# ------------------------------------------------------------------------------------------------
def test_conv_forward(run):
    r = run
    up_of = {o['y']: o['x'] for o in r.ops if o['kind'] == 'upadd'}
    for op in r.ops:
        if op['kind'] != 'conv' or not r.checked(op):
            continue
        W, b = r.weight(op['w'])
        k, s = op['k'], op['s']
        n = W.shape[1] * k * k
        for_dense = op['dense']
        if for_dense and op['y'] != 'out.proto' and op['y'] != 'out.seg' and op['y'] != 'out.head0':
            continue
        x = r.rd(op['x'])
        ref = conv_ref(x, W, b, k, s)
        ref_abs = conv_ref(x, W, b, k, s, absolute=True)
        if op['relu']:
            ref = ref.clamp_min(0)
        extent = (x.shape[-1], ref.shape[-1], k, s)
        if for_dense:                              # fp32 outputs, no 16-bit rounding
            o = r.outs[op['y'][4:]] if op['y'] != 'out.head0' else None
            if op['y'] == 'out.head0':
                H, R, NC = ref.shape[-1], r.R, r.NC
                n_a = H * H * R
                eng = torch.cat([r.outs['cls'][:, :n_a].reshape(r.B, H, H, R * NC), r.outs['box'][:, :n_a].reshape(r.B, H, H, R * 4)], -1)
                ref, ref_abs = ref[:, :R * (NC + 4)], ref_abs[:, :R * (NC + 4)]
            else:
                eng = o[..., :ref.shape[1]]
            r.check('conv_fwd_dense', op['y'], eng.permute(0, 3, 1, 2), ref, None, ref_abs, n, u=0.0, extent=extent)
            continue
        eng = r.rd(op['y'])
        rnd = ref.abs()
        if op['y'] in up_of:                       # FPN: the lateral conv output is overwritten in place by  + up(coarse)
            c = r.rd(up_of[op['y']])
            ref = ref + interp(c, ref.shape[-1], False)
            ref_abs = ref_abs + interp(c, ref.shape[-1], False, absolute=True)
            rnd = rnd + ref.abs()
            r.check('fpn_upadd_fwd', op['y'], eng, ref, rnd, ref_abs, n, extent=(c.shape[-1], ref.shape[-1]))
            continue
        r.check('conv_fwd', op['y'], eng, ref, rnd, ref_abs, n, extent=extent)
    finish(r, ('conv_fwd', 'conv_fwd_dense', 'fpn_upadd_fwd'))
    kinds = {(e[2], e[3]) for e in r.extents['conv_fwd']}
    assert {(1, 1), (3, 1), (1, 2), (3, 2), (7, 2)} <= kinds, kinds
    if r.S == 550:
        assert (550, 275, 7, 2) in r.extents['conv_fwd']
        assert {(18, 35), (35, 69)} <= r.extents['fpn_upadd_fwd']


# ------------------------------------------------------------------------------------------------
def contributions(r, name):
    """Every backward contribution to tensor `name`'s gradient, in the engine's order: (kind, value, |value|-op, n, separately
    rounded, exact copy, ambiguity term)."""
    out = []
    for op in sorted(r.ops, key=lambda o: -o['seq']):
        if op['kind'] == 'conv' and op['x'] == name:
            W, _ = r.weight(op['w'])
            dy, unc = r.dY(op)
            k, s = op['k'], op['s']
            args = dict(stride=s, padding=k // 2)
            shape = r.rd(name).shape
            v = torch.nn.grad.conv2d_input(shape, W, dy, **args)
            a = torch.nn.grad.conv2d_input(shape, W.abs(), dy.abs(), **args)
            amb = torch.nn.grad.conv2d_input(shape, W.abs(), unc, **args) if unc is not None else None
            out.append(dict(op=op, v=v, a=a, n=W.shape[0] * k * k, sep=s == 2 and bool(out), exact=False, amb=amb, extent=(shape[-1], dy.shape[-1], k, s)))
        elif op['kind'] == 'bn' and op['res'] == name:
            g = r.rd(op['z'], grad=True)
            if op['relu']:
                g = g * (r.rd(op['z']) > 0)
            out.append(dict(op=op, v=g, a=g.abs(), n=1, sep=False, exact=not out, amb=None, extent=None))
        elif op['kind'] in ('upadd', 'up2x') and op['x'] == name:
            Hc = r.rd(name).shape[-1]
            df = r.rd(op['y'], grad=True)
            ac = op['kind'] == 'up2x'
            out.append(dict(op=op, v=interp_bwd(df, Hc, ac), a=interp_bwd(df.abs(), Hc, ac), n=16, sep=False, exact=False, amb=None,
                            extent=(Hc, df.shape[-1], int(ac))))
    return out


def contrib_kind(op):
    if op['kind'] == 'conv':
        return 'dgrad_s2' if op['s'] == 2 else 'dgrad'
    return {'bn': 'dres', 'upadd': 'bilinear_bwd', 'up2x': 'bilinear_bwd_ac'}[op['kind']]


def test_dgrad(run):
    """Input gradients, summed over every consumer in the engine's order (conv dgrad incl. stride-2 parity planes + phase merge,
    the residual branch, bilinear backward of the FPN / proto up-samples), ReLU-masked where the engine masks in place."""
    r = run
    relu_out = {o['y'] for o in r.ops if o['kind'] == 'conv' and o['relu'] and not o['dense']}
    consumers = {}
    for o in r.ops:
        for key in ('x', 'res'):
            if o.get(key) and o[key] != 'img' and (o['kind'] != 'bn' or key == 'res'):
                consumers.setdefault(o[key], []).append(o)
    for name, cons in consumers.items():
        if name == 'stem.z' or not all(r.checked(o) for o in cons):
            continue                                               # stem.z: the max-pool backward, checked below
        contrib = contributions(r, name)
        S = torch.zeros_like(contrib[0]['v'])
        rnd = torch.zeros_like(S)
        ref_abs = torch.zeros_like(S)
        amb = torch.zeros_like(S)
        nr = 0
        for c in contrib:
            if c['sep']:
                rnd += c['v'].abs()                                 # stride-2 dgrad planes into a scratch buffer, then k_add16
                nr += 1
            S += c['v']
            if not c['exact']:
                rnd += S.abs()
                nr += 1
            ref_abs += c['n'] * c['a']
            if c['amb'] is not None:
                amb += c['amb']
            kind = contrib_kind(c['op'])
            if c['extent'] is not None:
                r.extents.setdefault(kind, set()).add(c['extent'][:2] if kind.startswith('bilinear') else c['extent'])
        eng = r.rd(name, grad=True)
        if name in relu_out:
            m = r.rd(name) > 0
            S, rnd, ref_abs, amb = S * m, rnd * m, ref_abs * m, amb * m
        kinds = sorted({contrib_kind(c['op']) for c in contrib})
        # ambiguity of the dense outputs' 16-bit dY: one ulp where the checker's fp32 value sits within LOSS_GRAD_EPS of a rounding
        # midpoint -- enters like a rounding of the input, hence with weight 1 in units of u: amb / u
        r.check('dgrad', name + ' <- ' + '+'.join(kinds), eng, S, rnd + amb / r.u, ref_abs, 1, extent=tuple(kinds), nr=max(nr, 1))
    finish(r, ('dgrad',))
    if r.S == 550:
        s2 = {e[0] for e in r.extents['dgrad_s2']}
        assert {138, 69, 35, 18, 9} <= s2, s2
        assert {(18, 35), (35, 69)} <= r.extents['bilinear_bwd'] and (69, 138) in r.extents['bilinear_bwd_ac'], r.extents


# ------------------------------------------------------------------------------------------------
def test_weight_and_bias_grads(run):
    r = run
    wg, bg = {}, {}
    for op in r.ops:
        if op['kind'] != 'conv' or not r.checked(op):
            continue
        W, b = r.weight(op['w'])
        k, s = op['k'], op['s']
        x = r.rd(op['x'])
        dy, unc = r.dY(op)
        args = dict(stride=s, padding=k // 2)
        e = wg.setdefault(op['w'], [0, 0, 0, 0, (x.shape[-1], dy.shape[-1], k, s)])
        e[0] = e[0] + torch.nn.grad.conv2d_weight(x, W.shape, dy, **args)
        e[1] = e[1] + torch.nn.grad.conv2d_weight(x.abs(), W.shape, dy.abs(), **args)
        e[3] += dy.shape[0] * dy.shape[2] * dy.shape[3]
        if unc is not None:
            e[2] = e[2] + torch.nn.grad.conv2d_weight(x.abs(), W.shape, unc, **args)
        if op['b'] is not None or op['w'] == 'head':
            f = bg.setdefault(op['b'] or 'head', [0, 0, 0, 0])
            f[0] = f[0] + dy.sum((0, 2, 3))                      # VALID pixels only: the engine sums haloed rows
            f[1] = f[1] + dy.abs().sum((0, 2, 3))
            f[3] += dy.shape[0] * dy.shape[2] * dy.shape[3]
            if unc is not None:
                f[2] = f[2] + unc.sum((0, 2, 3))
    names = ('prediction_layers.conf_layer', 'prediction_layers.bbox_layer', 'prediction_layers.coef_layer.0')

    def split(name, sfx, *ts):
        """(parameter name, its rows of each t): the fused head's rows are conf | bbox | coef."""
        if name != 'head':
            return [(name,) + ts]
        sz = [r.params[n + '.bias'].numel() for n in names]
        return list(zip([n + sfx for n in names], *[torch.split(t, sz) for t in ts]))

    # fp32 gradients: no 16-bit rounding (u * rnd = 0) except the ambiguity of a dense output's 16-bit dY (amb: one ulp per ambiguous
    # term, passed as rnd = amb / u)
    u16 = r.u
    n_w = 0
    for name, (ref, ref_abs, amb, n, ext) in wg.items():
        amb = amb if torch.is_tensor(amb) else torch.zeros_like(ref)
        for pn, rv, ra, am in split(name, '.weight', ref, ref_abs, amb):
            r.check('wgrad', pn, r.params[pn].grad, rv, am / u16, ra, n, u=u16, extent=ext)
            n_w += 1
    for name, (ref, ref_abs, amb, n) in bg.items():
        amb = amb if torch.is_tensor(amb) else torch.zeros_like(ref)
        for pn, rv, ra, am in split(name, '.bias', ref, ref_abs, amb):
            r.check('bgrad', pn, r.params[pn].grad, rv, am / u16, ra, n, u=u16, extent=n)
    finish(r, ('wgrad', 'bgrad'))
    if r.blocks is None:
        n_conv = sum(1 for n, p in r.net.named_parameters() if n.endswith('.weight') and p.dim() == 4)
        assert n_w == n_conv, (n_w, n_conv)
    if r.S == 550:
        assert (550, 275, 7, 2) in r.extents['wgrad'] and (138, 138, 1, 1) in r.extents['wgrad'], r.extents['wgrad']


# ------------------------------------------------------------------------------------------------
def stats_chain(rows, C):
    """Longest fp32 accumulation chain of a per-channel reduction over `rows` (launch_colstats / launch_bn_bwd_reduce geometry:
    a row lane's serial sum, the block's shared-memory adds, the grid's global adds)."""
    cvb = min(C // 8, 256)
    bx = -(-(C // 8) // cvb)
    rpb = max(64, -(-rows // max(1, 132 * 8 // bx)))
    return -(-rpb // (256 // cvb)) + 256 // cvb + -(-rows // rpb)


def bn_stats(y):
    m = y.mean((0, 2, 3))
    var = (y - m[None, :, None, None]).pow(2).mean((0, 2, 3))
    return m, var


def test_batchnorm(run):
    """Forward vs two-pass fp64 batch statistics of the engine's y (+ residual, ReLU), the running statistics of the checked step
    (momentum 0.1, unbiased variance), and the backward: y.grad, the residual gradient, dgamma, dbeta."""
    r = run
    eps, mom = 1e-5, 0.1
    ratio_max = 0.0
    for op in r.ops:
        if op['kind'] != 'bn' or not r.checked(op):
            continue
        p = op['p']
        y = r.rd(op['y'])
        N = y.shape[0] * y.shape[2] * y.shape[3]
        m, var = bn_stats(y)
        if op['y'] == 'stem.y':
            ratio_max = float((m.abs() / var.sqrt()).max())
        inv = (var + eps).rsqrt()
        n = stats_chain(y.shape[0] * (y.shape[2] + 2) ** 2, y.shape[1])
        # k_colstats sums d = y - pivot (pivot = the channel's first interior value) and k_bn_finalize takes var = E[d^2] - E[d]^2:
        # the fp32 sums err by gamma_n * E[d^2] and gamma_n * E|d|, so var errs by gamma_n * (E[d^2] + 2 |E d| E|d|) <= 3 kappa
        # gamma_n var with kappa = E[d^2] / var = 1 + (mean - pivot)^2 / var.  kappa scales every term that depends on the
        # statistics.  (Without the pivot, kappa = 1 + mean^2 / var: the big-mean stem channel then misses the L2 rule in fp16.)
        kappa = 3 * (1 + (m - y[0, :, 0, 0]).pow(2) / var.clamp_min(1e-300))
        ma = m.abs() + (m - y[0, :, 0, 0]).abs()                 # the mean errs by gamma_n * E|d| <= gamma_n * (|mean - pivot| + std)
        gam, bet = r.params[p + '.weight'].detach().double(), r.params[p + '.bias'].detach().double()
        c = lambda v: v[None, :, None, None]
        xh = (y - c(m)) * c(inv)
        ref = xh * c(gam) + c(bet)
        ref_abs = (xh.abs() * c(kappa) + c(ma * inv) + y.abs() * c(inv)) * c(gam.abs()) + c(bet.abs())
        if op['res']:
            res = r.rd(op['res'])
            ref, ref_abs = ref + res, ref_abs + res.abs()
        if op['relu']:
            ref = ref.clamp_min(0)
        extent = N
        r.check('bn_fwd', op['z'], r.rd(op['z']), ref, ref.abs(), ref_abs, n, extent=extent)
        # running statistics of the checked step
        rm0, rv0 = r.bn_before[p + '.running_mean'].double(), r.bn_before[p + '.running_var'].double()
        rm_ref = (1 - mom) * rm0 + mom * m
        rv_ref = (1 - mom) * rv0 + mom * var * N / (N - 1)
        r.check('bn_running', p + '.running_mean', r.buffers[p + '.running_mean'], rm_ref, None,
                (1 - mom) * rm0.abs() + mom * (ma + var.sqrt()), n, extent=extent)
        r.check('bn_running', p + '.running_var', r.buffers[p + '.running_var'], rv_ref, None, (1 - mom) * rv0.abs() + mom * var * kappa, n, extent=extent)
        # backward
        dz = r.rd(op['z'], grad=True)
        g = dz * (r.rd(op['z']) > 0) if op['relu'] else dz
        sg, sgx = g.sum((0, 2, 3)), (g * xh).sum((0, 2, 3))
        dy_ref = c(gam * inv) * (g - c(sg) / N - xh * c(sgx) / N)
        gx_abs = (g * xh).abs().sum((0, 2, 3))
        dy_abs = c(gam.abs() * inv * kappa) * (g.abs() + c(g.abs().sum((0, 2, 3))) / N + (xh.abs() + c(ma * inv)) * c(gx_abs + g.abs().sum((0, 2, 3)) * ma * inv) / N)
        r.check('bn_bwd', op['y'] + '.grad', r.rd(op['y'], grad=True), dy_ref, dy_ref.abs(), dy_abs, n, extent=extent)
        r.check('bn_dgamma', p + '.weight', r.params[p + '.weight'].grad, sgx, None, (gx_abs + (g.abs() * (y.abs() + c(ma)) * c(inv)).sum((0, 2, 3))) * kappa, n, extent=extent)
        r.check('bn_dbeta', p + '.bias', r.params[p + '.bias'].grad, sg, None, g.abs().sum((0, 2, 3)), n, extent=extent)
        if op['res'] and op['res'].endswith('downsample.z'):        # dres is written straight into the branch's gradient: a copy
            r.check('bn_dres', op['res'], r.rd(op['res'], grad=True), g, None, None, 0, exact=True, extent=extent)
    finish(r, ('bn_fwd', 'bn_running', 'bn_bwd', 'bn_dgamma', 'bn_dbeta', 'bn_dres'))
    print(f'{r.key} stem.y max |mean|/std over channels: {ratio_max:.1f}')
    if CONFIGS[r.key][4]:
        assert ratio_max >= 50, ratio_max
    if r.S == 550:
        assert r.B * 275 ** 2 in r.extents['bn_fwd']


# ------------------------------------------------------------------------------------------------
def test_pool_and_upsample(run):
    r = run
    z = r.rd('stem.z')
    pool = r.rd('pool')
    ref = F.max_pool2d(z, 3, 2, 1)
    ext = (z.shape[-1], pool.shape[-1])
    r.check('maxpool_fwd', 'pool', pool, ref, None, None, 0, exact=True, extent=ext)
    zz = z.clone().requires_grad_(True)
    dpool = r.rd('pool', grad=True)
    dz_ref, = torch.autograd.grad(F.max_pool2d(zz, 3, 2, 1), zz, dpool)      # to the FIRST maximum of each window (row-major)
    dz_abs, = torch.autograd.grad(F.max_pool2d(zz, 3, 2, 1), zz, dpool.abs())
    r.check('maxpool_bwd', 'stem.z', r.rd('stem.z', grad=True), dz_ref, dz_ref.abs(), dz_abs, 4, extent=ext)
    ties = float(((z == 0).float().mean()))
    q14 = r.rd('proto1.4')
    upr = interp(q14, 2 * q14.shape[-1], True)
    r.check('up2x_ac_fwd', 'proto.up', r.rd('proto.up'), upr, upr.abs(), interp(q14, 2 * q14.shape[-1], True, absolute=True), 4,
            extent=(q14.shape[-1], upr.shape[-1]))
    finish(r, ('maxpool_fwd', 'maxpool_bwd', 'up2x_ac_fwd'))
    print(f'{r.key} stem.z zero fraction (max-pool ties) {ties:.2f}')
    if r.S == 550:
        assert (275, 138) in r.extents['maxpool_bwd'] and (69, 138) in r.extents['up2x_ac_fwd']


# ------------------------------------------------------------------------------------------------
def test_losses_at_550(cuda):
    """yb_losses at the benchmarked shape (A = 19248 anchors, P = 138, Hs = 69) on synthetic predictions vs the torch checker."""
    from oracle import synth, train_torch as tt
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    S, B = 550, 2
    cfg = make_config('res50_coco', S, mode='train', train_bs=B)
    anchors = Yolact(cfg).anchors
    anchors = (anchors.detach().cpu().numpy() if isinstance(anchors, torch.Tensor) else np.asarray(anchors)).reshape(-1, 4).astype(np.float32)
    A, P, Hs, NC = anchors.shape[0], 138, 69, 81
    assert A == 19248
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    tg, mk = synth.train_targets(9, B, S, n=4)
    class_p = f32(synth.normal(21, 1, (B, A, NC)) * 2)
    box_p = f32(synth.normal(21, 2, (B, A, 4)) * 0.5)
    coef_p = np.tanh(f32(synth.normal(21, 3, (B, A, 32))))
    proto_p = np.maximum(f32(synth.normal(21, 4, (B, P, P, 32))), 0)
    seg_p = f32(synth.normal(21, 5, (B, NC - 1, Hs, Hs)))
    r = tc.run_native_losses(cuda, cfg, anchors, tg, mk, class_p, box_p, coef_p, proto_p, seg_p)
    labels, idx = [], []
    anc = torch.from_numpy(anchors).float()
    for i in range(B):
        _, lab, _, ix = tt.assign_targets(cfg, torch.from_numpy(tg[i][:, :4]).float(), anc, torch.from_numpy(tg[i][:, 4]).long())
        labels.append(lab.numpy()); idx.append(ix.numpy())
    labels, idx = np.stack(labels), np.stack(idx)
    pos = labels > 0
    assert np.array_equal(r['labels'], labels)
    assert np.array_equal(r['matched_idx'][pos], idx[pos])
    assert int(pos.sum(1).max()) <= cfg.masks_to_train             # no random subset: the checker sees the same masks
    _, g = tc.torch_losses_and_grads(cfg, anchors, tg, mk, class_p, box_p, coef_p, proto_p, seg_p)
    for k in ('d_cls', 'd_box', 'd_coef', 'd_proto', 'd_seg'):
        e = tc.rel(r[k], g[k])
        print(f'losses@550 {k}: rel L2 {e:.2e}  (A={A} P={P} Hs={Hs})')
        assert e < 1e-5, (k, e)
