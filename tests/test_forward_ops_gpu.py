"""GPU: the inference forward op by op against fp64, at the engine's own operands, at the benchmarked shapes.

Each configuration builds one net from `synth_state_dict(arch, seed=0)`, runs a warm-up forward of a different full batch (so the
activation arena holds stale data behind every tensor), then steps through the finalized program with yb_net_forward_range: the
op's operands are read exactly as stored (yb_net_read_act_raw: halos, parity planes, dense rows), the op runs alone, its outputs
are read, and the op is recomputed in fp64 with torch on the GPU from exactly those operands and the engine's own packed weights
(which are checked bitwise against a numpy restatement of the BN fold and the packing).  Every element of every image is compared
under ONE error model, the one of test_train_ops_gpu.py:

    |eng - ref| <= u * rnd  +  eta * nr  +  C_ACC * 2^-24 * n * ref_abs  (+ extra, for the intrinsics below)

  u        unit roundoff of the 16-bit type (2^-8 bf16, 2^-11 fp16); 0 for fp32 results (the dense head / proto rows, the outputs)
  eta, nr  absolute rounding error of a subnormal (2^-25 fp16), times the number of such roundings
  rnd      magnitude of every value rounded to 16 bits on the way: |ref| for one store
  ref_abs  the same op on absolute values (|x| * |W| + |b| + |res| ...), computed in fp32 without TF32 (it is only a bound)
  n        terms per output (Cin * k * k + bias + residual), or the number of fp32 operations of an elementwise op
  C_ACC    2: any fp32 sum of n terms errs by at most gamma_n * sum|terms| (Higham 4.2); 2^-23 per step covers a truncating
           accumulator.  Exact GELU: |gelu'| <= 1.13 and erff errs by 2 ulp, both inside C_ACC for n >= 2.

and each tensor's relative L2 error must stay below L2_U * u * max(1, |rnd| / |ref|).  The intrinsics add their documented
errors (CUDA C Programming Guide, "Mathematical Functions", maximum ulp errors):

  __expf(x)  2 + floor(|1.173 x|) ulp (flushes results below 2^-126 to zero).  A softmax p_j = e_j / sum e with relative errors
             r_j on e_j errs by p_j * (r_j + sum_i p_i r_i) + the divide / sum roundings; x = s - max, whose subtraction adds
             2^-24 |x|.  So r_j = (2 + 2 |x_j|) 2^-23 (+ the score's own absolute error in attention), plus 2^-126.
  tanhf      2 ulp: 2^-22 |tanh|.
  rsqrtf     2 ulp: 2^-22 relative on LayerNorm's 1/std.  LayerNorm y = (a - mean) r g + b with fp32 sums over C channels:
             mean errs by C_ACC C 2^-24 mean|a| (+ the input's own error da), d = a - mean by da + that + 2^-24 |d|, the variance
             relatively by C_ACC (C + 2) 2^-24 + 2 mean(|d| |dd|) / var, r by 2^-22 + half of that + 2^-24, and y by
             |g| r (|dd| + |d| |dr/r|) + 3 2^-24 (|d r g| + |b|).
  window attention: P is rounded to 16 bits before P.V, which adds u * sum_j p_j |v_j| / l to the output (and eta * sum |v_j| for
             subnormal p); the score s = q.k * scale + table + mask errs by C_ACC 32 2^-24 |q|.|k| scale + 3 2^-24 (|s| + |table|
             + 100); the fp32 P.V accumulation (64 terms) by C_ACC 64 2^-24 sum p |v|, l by 64 2^-24, and 1/l and the product by
             2^-24 each.

Exact ops (max-pool, phase split, the stem's space-to-depth image, the head's box copy) must match exactly, halos and padding
included.  16-bit results must stay below the fp16 saturation (65504) so the bound means something.  Structural checks: every
haloed output except the attention output (whose halo is untouched by contract: the projection's epilogue zeroes its own) has
an all-zero halo; the census of checked ops equals the program's; and at the pipelined configurations the stepped outputs
equal a normal yb_net_forward bit for bit (k_conv_tc / k_bneck_tc launch with programmatic dependent launch).  The class-count
configurations run the head at 21 (Pascal), 5 (the custom set) and the bounds 2 and 129.
"""
import collections
import ctypes
import gc
import math
import os
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import forward_torch as ft

pytestmark = pytest.mark.gpu

C_ACC = 2.0
L2_U = 2.0
E24 = 2.0 ** -24
U = {1: 2.0 ** -8, 2: 2.0 ** -11}
ETA = {1: 2.0 ** -134, 2: 2.0 ** -25}
TDT = {0: torch.float32, 1: torch.bfloat16, 2: torch.float16}
R, K = 3, 32
KINDS = ['stem', 'pool', 'split', 'conv', 'upadd', 'up2x', 'headfin', 'patch_embed', 'ln', 'attn', 'merge_ln', 'bneck']
DEPTH = {'res50': 50, 'res101': 101, 'swin_tiny': 0}
BNECK_TRIPLES = {(64, 256, 64), (128, 512, 128), (256, 1024, 256), (64, 256, 128), (128, 512, 256)}
ELEMS = 1.2e8                                   # fp64 elements per reference chunk

CONFIGS = {
    'res101-550-B64-fp16': dict(arch='res101', S=550, B=64, prec='fp16', max_batch=64, pipelined=True),
    'res101-544-B4-fp16': dict(arch='res101', S=544, B=4, prec='fp16', max_batch=4),
    'res50-550-B5-bf16': dict(arch='res50', S=550, B=5, prec='bf16', max_batch=8),
    'swin-550-B32-fp16': dict(arch='swin_tiny', S=550, B=32, prec='fp16', max_batch=32, pipelined=True),
    'swin-544-B2-fp16': dict(arch='swin_tiny', S=544, B=2, prec='fp16', max_batch=2),
    'res50-550-B3-fp16-stemwide': dict(arch='res50', S=550, B=3, prec='fp16', max_batch=3, stem_only=True,
                                       env={'YOLACT_B200_STEM_WIDE': '1'}),
    # the class count (nc, background included; 81 when absent) sets the head conv's width, and with it the tile width
    # conv_tc.cu's pick_bn gives it, and how many logits each lane of k_head_finalize holds
    'res50-550-B2-bf16-nc21': dict(arch='res50', S=550, B=2, prec='bf16', max_batch=2, nc=21),
    'res101-550-B2-fp16-nc5': dict(arch='res101', S=550, B=2, prec='fp16', max_batch=2, nc=5),
    'res50-128-B2-fp16-nc2': dict(arch='res50', S=128, B=2, prec='fp16', max_batch=2, nc=2),
    'res50-128-B2-bf16-nc129': dict(arch='res50', S=128, B=2, prec='bf16', max_batch=2, nc=129, pipelined=True),
}
# the head conv's row stride, R * (nc + 4 + K) rounded up to 16: 176 is one 176-wide tile with 5 padding columns, 496 is
# 31 tiles of width 16
HEAD_LD = {81: 352, 21: 176, 5: 128, 2: 128, 129: 496}


def chunks(B, per_image):
    cb = max(1, min(B, int(ELEMS // max(1, per_image))))
    return [(b0, min(B, b0 + cb)) for b0 in range(0, B, cb)]


def conv_nhwc(x, taps, k, s, bias=None):
    """y[b, y, x] = bias + sum_(r,q) xpad[b, s y + r, s x + q] @ taps[r k + q]  (zero padding k // 2, NHWC, GEMMs per tap)."""
    b_, H, _, Cin = x.shape
    p = k // 2
    Ho = (H + 2 * p - k) // s + 1
    xp = F.pad(x, (0, 0, p, p, p, p))
    Cout = taps[0].shape[1]
    out = torch.zeros(b_ * Ho * Ho, Cout, dtype=x.dtype, device=x.device)
    if bias is not None:
        out += bias.to(x.dtype)
    for r in range(k):
        for q in range(k):
            if taps[r * k + q] is None:
                continue
            sl = xp[:, r:r + s * (Ho - 1) + 1:s, q:q + s * (Ho - 1) + 1:s, :]
            out.addmm_(sl.reshape(-1, Cin), taps[r * k + q].to(x.dtype))
    return out.view(b_, Ho, Ho, Cout)


def interp_matrix(Hc, Hf, align):
    """[Hf, Hc] bilinear weights with the kernels' fp32 source-coordinate arithmetic (src_index, kernels_simt.cu)."""
    f = np.float32
    scale = f(Hc - 1) / f(Hf - 1) if align else f(Hc) / f(Hf)
    M = np.zeros((Hf, Hc))
    for j in range(Hf):
        src = scale * f(j) if align else max(f(float(scale) * (j + 0.5) - 0.5), f(0))   # fmaf: one rounding
        i0 = min(int(src), Hc - 1)
        i1 = min(i0 + 1, Hc - 1)
        l1 = f(src - f(i0))
        l0 = f(f(1) - l1)
        M[j, i0] += float(l0)
        M[j, i1] += float(l1)
    return M


def interp_nhwc(x, M):
    return torch.einsum('yi,bijc,xj->byxc', M, x, M)


def ln_ref(a, g, b, da=None):
    """LayerNorm over the last axis in fp64 and the absolute error bound of the kernels' fp32 evaluation (module docstring)."""
    C = a.shape[-1]
    mean = a.mean(-1, keepdim=True)
    d = a - mean
    var = (d * d).mean(-1, keepdim=True)
    r = (var + 1e-5).rsqrt()
    y = d * r * g + b
    da_max = da.amax(-1, keepdim=True) if da is not None else 0.0
    dm = C_ACC * C * E24 * a.abs().mean(-1, keepdim=True) + da_max
    dd = (da if da is not None else 0.0) + dm + E24 * d.abs()
    dvar = C_ACC * (C + 2) * E24 + 2 * (d.abs() * dd).mean(-1, keepdim=True) / var
    dr = 2.0 ** -22 + 0.5 * dvar * var / (var + 1e-5) + E24
    extra = g.abs() * r * (dd + d.abs() * dr) + 3 * E24 * ((d * r * g).abs() + b.abs())
    return y, extra


class Stat:
    """Worst err / bound and relative L2 error of one op's output, accumulated over image chunks."""

    def __init__(self, u):
        self.u, self.worst, self.e2, self.r2, self.d2, self.sat, self.where = u, 0.0, 0.0, 0.0, 0.0, 0.0, None

    def add(self, eng, ref, bound, rnd=None):
        eng, ref = eng.double(), ref.double()
        if not bool(torch.isfinite(eng).all()):
            self.worst = math.inf
            return
        err = (eng - ref).abs()
        if bool(((bound <= 0) & (err > 0)).any()):
            self.worst = math.inf
        if bool((bound > 0).any()):
            ratio = err / bound.clamp_min(1e-300)
            w = float(ratio.max())
            if w > self.worst:
                j = int(ratio.argmax())
                self.where = (tuple(int(v) for v in np.unravel_index(j, tuple(ratio.shape))), float(eng.flatten()[j]), float(ref.flatten()[j]))
                self.worst = w
        self.e2 += float((err * err).sum())
        self.r2 += float((ref * ref).sum())
        self.d2 += float((rnd * rnd).sum()) if rnd is not None else 0.0
        self.sat = max(self.sat, float(ref.abs().max()))

    def rel(self):
        return math.sqrt(self.e2) / max(math.sqrt(self.r2), 1e-300)

    def ok(self):
        rel_bound = L2_U * self.u * max(1.0, math.sqrt(self.d2) / max(math.sqrt(self.r2), 1e-300))
        return self.worst <= 1.0 and self.rel() <= rel_bound


# ------------------------------------------------------------------------------------------------
class Stepped:
    def __init__(self, key, dev):
        c = CONFIGS[key]
        self.key, self.dev = key, dev
        self.arch, self.S, self.B, self.prec, self.mb = c['arch'], c['S'], c['B'], c['prec'], c['max_batch']
        self.nc = c.get('nc', 81)
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = False
        from yolact_minimal_b200 import _lib
        from yolact_minimal_b200.engine import Engine
        self.lib_ = _lib
        old = {k: os.environ.get(k) for k in c.get('env', {})}
        os.environ.update(c.get('env', {}))
        try:
            self.eng = Engine(DEPTH[self.arch], self.S, self.nc, R, K)
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        self.sd = ft.synth_state_dict(self.arch, num_classes=self.nc, seed=0)
        self.eng.load_state(self.sd)
        with torch.cuda.device(dev):
            self.eng.finalize(self.mb, self.prec)
        self.eng.device = dev
        self.L, self.h = self.eng.L, self.eng.h
        self.dcode = {'bf16': 1, 'fp16': 2}[self.prec]
        self.dt, self.u = TDT[self.dcode], U[self.dcode]
        self.n_ops = self.L.yb_net_num_ops(self.h)
        self.ops = [self.op_info(i) for i in range(self.n_ops)]
        self.producer = {o['out']: i for i, o in enumerate(self.ops) if o['out'] >= 0}
        self.stats, self.exact_fail, self.halo_fail, self.weight_fail = [], [], [], []
        self.census = collections.Counter()
        self.extents = collections.defaultdict(set)

    # ---- ABI helpers ----
    def check(self, st, what):
        self.lib_.check(st, what)

    def stream(self):
        return torch.cuda.current_stream().cuda_stream

    def op_info(self, i):
        oi = self.lib_.OpInfo()
        self.check(self.L.yb_net_op_info(self.h, i, ctypes.byref(oi)), 'yb_net_op_info')
        d = {n: getattr(oi, n) for n, _ in oi._fields_}
        d['in'] = d.pop('in_')
        for n in ('w0', 'b0', 'bn0', 'w1', 'bn1', 'wd', 'bnd', 'p0', 'p1'):
            d[n] = d[n].decode()
        d['kind'] = KINDS[d['kind']]
        return d

    def act(self, a):
        ai = self.lib_.ActInfo()
        self.check(self.L.yb_net_act_info(self.h, a, ctypes.byref(ai)), 'yb_net_act_info')
        return ai

    def raw(self, a):
        """(planes [P, B, H+2, H+2, C] or dense [B, H, H, C], pad rows or None) as stored."""
        ai, B = self.act(a), self.B
        if ai.dense:
            t = torch.empty(B * ai.H * ai.H, ai.C, dtype=torch.float32, device=self.dev)
        else:
            t = torch.empty(ai.planes * B * (ai.H + 2) ** 2 + ai.pad_rows, ai.C, dtype=TDT[ai.dtype], device=self.dev)
        self.check(self.L.yb_net_read_act_raw(self.h, a, B, t.data_ptr(), t.numel() * t.element_size(), self.stream()), 'yb_net_read_act_raw')
        if ai.dense:
            return t.view(B, ai.H, ai.H, ai.C), None
        n = ai.planes * B * (ai.H + 2) ** 2
        return t[:n].view(ai.planes, B, ai.H + 2, ai.H + 2, ai.C), (t[n:] if ai.pad_rows else None)

    def interior(self, a):
        x, _ = self.raw(a)
        return x[0, :, 1:-1, 1:-1]

    def weights(self, i, which):
        rows, cols = ctypes.c_int(), ctypes.c_int()
        self.check(self.L.yb_net_read_op_weights(self.h, i, which, None, 0, None, 0, ctypes.byref(rows), ctypes.byref(cols), None), 'weights')
        w = torch.empty(rows.value, cols.value, dtype=self.dt, device=self.dev)
        b = torch.empty(rows.value, dtype=torch.float32, device=self.dev)
        self.check(self.L.yb_net_read_op_weights(self.h, i, which, w.data_ptr(), w.numel() * 2, b.data_ptr(), b.numel() * 4, ctypes.byref(rows),
                                                 ctypes.byref(cols), self.stream()), 'yb_net_read_op_weights')
        return w, b

    def forward(self, img, first, last, outs):
        self.check(self.L.yb_net_forward_range(self.h, img.data_ptr(), img.shape[0], first, last, *[t.data_ptr() for t in outs], self.stream()),
                   'yb_net_forward_range')

    # ---- bookkeeping ----
    def stat(self, kind, label):
        s = Stat(self.u)                       # the relative L2 rule uses the 16-bit u for fp32 results too, as test_train_ops_gpu.py
        self.stats.append((kind, label, s))
        return s

    def exact(self, label, eng, ref):
        if not torch.equal(eng, ref):
            self.exact_fail.append(label)

    def halo(self, label, a):
        ai = self.act(a)
        if ai.dense or ai.planes > 1:
            return
        x = self.raw(a)[0][0]
        h = torch.cat([x[:, 0].flatten(), x[:, -1].flatten(), x[:, :, 0].flatten(), x[:, :, -1].flatten()])
        if bool((h != 0).any()):
            self.halo_fail.append((label, int((h != 0).sum())))

    # ---- the run ----
    def run(self, stem_only=False, pipelined=False):
        dev, B, S, A = self.dev, self.B, self.S, self.eng.num_anchors
        P = self.eng.proto_size
        gen = torch.Generator(device=dev)
        gen.manual_seed(7)
        warm = torch.randn(self.mb, 3, S, S, device=dev, generator=gen) * 2.0
        gen.manual_seed(1234)
        self.img = torch.randn(B, 3, S, S, device=dev, generator=gen)
        mk = lambda n: [torch.empty(n, A, self.nc, device=dev), torch.empty(n, A, 4, device=dev), torch.empty(n, A, K, device=dev),
                        torch.empty(n, P, P, K, device=dev)]
        self.forward(warm, 0, self.n_ops, mk(self.mb))                     # stale data in every arena slot
        self.outs = [t.fill_(float('nan')) for t in mk(B)]
        last = 1 if stem_only else self.n_ops
        for i in range(last):
            getattr(self, 'op_' + self.ops[i]['kind'])(i, self.ops[i])
            self.census[self.ops[i]['kind']] += 1
        torch.cuda.synchronize()
        if not stem_only:
            for name, t in zip(('cls', 'box', 'coef', 'proto'), self.outs):
                if not bool(torch.isfinite(t).all()):
                    self.exact_fail.append(f'{name}: unwritten (NaN) entries after the stepped run')
        if pipelined:
            ref = mk(B)
            self.forward(self.img, 0, self.n_ops, ref)
            torch.cuda.synchronize()
            self.pipelined_equal = all(torch.equal(a, b) for a, b in zip(self.outs, ref))

    def step(self, i, reads):
        """operands (read before), run op i alone"""
        pre = {a: self.raw(a) for a in reads if a >= 0}
        self.forward(self.img, i, i + 1, self.outs)
        return pre

    def report(self):
        lines = []
        for kind, label, s in self.stats:
            lines.append(f'{self.key} {kind:11s} {label:42s} worst err/bound {s.worst:7.3f}  rel L2 {s.rel():.2e}' +
                         (f'  at (chunk index, eng, ref) {s.where}' if s.worst > 1 else ''))
        return lines

    # ---- the ops ----
    def taps_of(self, w, k, cin, cout, cin_pad):
        w = w[:cout].view(cout, k * k, cin_pad)[:, :, :cin]
        return [w[:, t].t().contiguous() for t in range(k * k)]

    def check_conv(self, label, x_nhwc_fn, taps, k, s, bias, relu, res_fn, eng_fn, n, dense=False):
        """x_nhwc_fn(b0, b1) -> operand images (fp64, interior), res_fn likewise or None, eng_fn(b0, b1) -> engine output."""
        st = self.stat('conv' if not dense else 'conv_dense', label)
        x0 = x_nhwc_fn(0, 1)
        per = x0[0].numel() * 3 + (x0.shape[1] // s + 1) ** 2 * taps[0].shape[1] * 6
        taps_abs = [t.abs().float() if t is not None else None for t in taps]
        for b0, b1 in chunks(self.B, per):
            x = x_nhwc_fn(b0, b1)
            v = conv_nhwc(x, taps, k, s, bias)
            va = conv_nhwc(x.abs().float(), taps_abs, k, s, bias.abs().float() if bias is not None else None).double()
            if res_fn is not None:
                r = res_fn(b0, b1)
                v, va = v + r, va + r.abs()
            if relu == 1:
                v = v.clamp_min(0)
            elif relu == 2:
                v = 0.5 * v * (1 + torch.erf(v / math.sqrt(2)))
                va = va * 1.13
            eng = eng_fn(b0, b1)
            if dense:
                st.add(eng, v[..., :eng.shape[-1]], C_ACC * E24 * n * va[..., :eng.shape[-1]])
            else:
                bound = self.u * v.abs() + ETA[self.dcode] + C_ACC * E24 * n * va
                st.add(eng, v, bound, v.abs())
        if not dense and self.dcode == 2 and st.sat >= 65504:
            self.exact_fail.append(f'{label}: |ref| {st.sat} reaches the fp16 saturation')
        self.extents['conv'].add((x0.shape[1], k, s))

    def op_stem(self, i, o):
        self.forward(self.img, i, i + 1, self.outs)
        s2d, pad = self.raw(o['aux'])
        ai = self.act(o['aux'])
        Hp = ai.H + 2
        img16 = self.img.to(self.dt)
        Z = torch.zeros(self.B, 3, 2 * Hp + 8, 2 * Hp + 8, dtype=self.dt, device=self.dev)
        Z[:, :, 4:4 + self.S, 4:4 + self.S] = img16
        parts = torch.stack([Z[:, :, py::2, px::2][:, :, :Hp, :Hp] for py in (0, 1) for px in (0, 1)], 1)   # [B, 4, 3, Hp, Hp]
        e = F.pad(parts.permute(0, 3, 4, 1, 2).reshape(self.B, Hp, Hp, 12), (0, 4))
        if ai.C == 64:
            e = F.pad(e, (0, 0, 0, 3))
            e = torch.cat([e[:, :, d:d + Hp] for d in range(4)], -1)
        self.exact('stem s2d image', s2d[0].view(torch.int16), e.view(torch.int16))
        self.exact('stem s2d pad rows', pad.view(torch.int16), torch.zeros_like(pad).view(torch.int16))
        w, b = self.weights(i, 0)
        taps = [None] * 49
        for dy in range(4):
            for dx in range(4):
                for py in (0, 1):
                    for px in (0, 1):
                        r, q = 2 * dy + py - 1, 2 * dx + px - 1
                        if r >= 0 and q >= 0:
                            c0 = dy * 64 + dx * 16 + (py * 2 + px) * 3
                            taps[r * 7 + q] = w[:, c0:c0 + 3].t().double()
        taps = [t if t is not None else torch.zeros(3, 64, dtype=torch.float64, device=self.dev) for t in taps]
        out = self.interior(o['out'])
        imgn = img16.permute(0, 2, 3, 1)
        self.check_conv(f'stem {self.S}->{out.shape[1]} 7x7 s2', lambda b0, b1: imgn[b0:b1].double(), taps, 7, 2, b.double(), 1, None,
                        lambda b0, b1: out[b0:b1], 148)
        self.halo('stem', o['out'])
        self.extents['stem'].add((ai.C, self.S))

    def op_pool(self, i, o):
        self.forward(self.img, i, i + 1, self.outs)
        x = self.interior(o['in']).float().permute(0, 3, 1, 2)
        y = self.interior(o['out']).float().permute(0, 3, 1, 2)
        self.exact('maxpool', y, F.max_pool2d(x, 3, 2, 1))
        self.halo('maxpool', o['out'])

    def op_split(self, i, o):
        self.forward(self.img, i, i + 1, self.outs)
        x = self.interior(o['in'])
        planes, _ = self.raw(o['out'])
        Ho, Hin = planes.shape[2] - 2, x.shape[1]
        Z = torch.zeros(self.B, 2 * Ho + 4, 2 * Ho + 4, x.shape[-1], dtype=x.dtype, device=self.dev)
        Z[:, 2:2 + Hin, 2:2 + Hin] = x
        ref = torch.stack([Z[:, p::2, q::2][:, :Ho + 2, :Ho + 2] for p in (0, 1) for q in (0, 1)][:planes.shape[0]])
        self.exact(f'split {Hin}->{Ho} x{planes.shape[0]}', planes.view(torch.int16), ref.view(torch.int16))
        self.extents['split'].add(planes.shape[0])

    def op_upadd(self, i, o):
        pre = self.step(i, [o['in'], o['out']])
        coarse, fine = pre[o['in']][0][0, :, 1:-1, 1:-1], pre[o['out']][0][0, :, 1:-1, 1:-1]
        out = self.interior(o['out'])
        M = torch.from_numpy(interp_matrix(coarse.shape[1], fine.shape[1], False)).to(self.dev)
        st = self.stat('upadd', f'upadd {coarse.shape[1]}->{fine.shape[1]}')
        for b0, b1 in chunks(self.B, fine[0].numel() * 4):
            c = coarse[b0:b1].double()
            ref = fine[b0:b1].double() + interp_nhwc(c, M)
            ra = fine[b0:b1].double().abs() + interp_nhwc(c.abs(), M)
            st.add(out[b0:b1], ref, self.u * ref.abs() + ETA[self.dcode] + C_ACC * E24 * 8 * ra, ref.abs())
        self.halo('upadd', o['out'])
        self.extents['upadd'].add((coarse.shape[1], fine.shape[1]))

    def op_up2x(self, i, o):
        self.forward(self.img, i, i + 1, self.outs)
        x, out = self.interior(o['in']), self.interior(o['out'])
        M = torch.from_numpy(interp_matrix(x.shape[1], out.shape[1], True)).to(self.dev)
        st = self.stat('up2x', f'up2x {x.shape[1]}->{out.shape[1]}')
        for b0, b1 in chunks(self.B, out[0].numel() * 3):
            xx = x[b0:b1].double()
            ref, ra = interp_nhwc(xx, M), interp_nhwc(xx.abs(), M)
            st.add(out[b0:b1], ref, self.u * ref.abs() + ETA[self.dcode] + C_ACC * E24 * 8 * ra, ref.abs())
        self.halo('up2x', o['out'])

    def conv_input(self, planes, a, stride):
        """operand images of a convolution as fp64 NHWC interiors; stride 2: the full-resolution tensor rebuilt from its parity planes
        (which the split op is checked against bitwise, padding included)."""
        if stride == 1:
            return lambda b0, b1: planes[0, b0:b1, 1:-1, 1:-1].double()
        Hin = self.act(self.ops[self.producer[a]]['in']).H

        def full(b0, b1):
            X = torch.zeros(b1 - b0, Hin, Hin, planes.shape[-1], dtype=torch.float64, device=self.dev)
            for pl in range(planes.shape[0]):
                p, q = pl >> 1, pl & 1
                ny, nx = len(range(p, Hin, 2)), len(range(q, Hin, 2))
                X[:, p::2, q::2] = planes[pl, b0:b1, 1:1 + ny, 1:1 + nx].double()
            return X
        return full

    def op_conv(self, i, o):
        pre = self.step(i, [o['in'], o['res']])
        w, b = self.weights(i, 0)
        k, cin, cout = o['k'], o['cin'], o['cout']
        taps = self.taps_of(w, k, cin, cout, w.shape[1] // (k * k))
        taps = [t.double() for t in taps]
        xf = self.conv_input(pre[o['in']][0], o['in'], o['stride'])
        resf = None
        if o['res'] >= 0:
            rr = pre[o['res']][0]
            resf = lambda b0, b1: rr[0, b0:b1, 1:-1, 1:-1].double()
        n = cin * k * k + 1 + (o['res'] >= 0)
        head = o['out_mode'] == 1 and not o['ext_proto']
        name = o['w0'].rsplit('.', 1)[0] if o['w0'] else 'head'
        if o['ext_proto']:
            out = self.outs[3]
            self.check_conv(f'{name} (proto out)', xf, taps, k, 1, b[:cout].double(), o['relu'], None, lambda b0, b1: out[b0:b1], n, dense=True)
        elif head:
            out = self.raw(o['out'])[0]
            ncol = R * (self.nc + 4 + K)
            self.extents['head_ld'].add(out.shape[-1])
            self.check_conv(f'head conv {out.shape[1]}', xf, taps, k, 1, b[:cout].double(), o['relu'], None,
                            lambda b0, b1: out[b0:b1, ..., :ncol], n, dense=True)
        else:
            out = self.interior(o['out'])
            self.check_conv(f'{name} {out.shape[1]}', xf, taps, k, o['stride'], b[:cout].double(), o['relu'], resf,
                            lambda b0, b1: out[b0:b1], n)
            self.halo(name, o['out'])

    def op_bneck(self, i, o):
        pre = self.step(i, [o['in'], o['res'], o['in2']])
        w3, b3 = self.weights(i, 0)
        w1, b1 = self.weights(i, 1)
        cin, cexp = o['cin'], o['cout']
        cd = w3.shape[1] - cin if o['convd'] else 0
        cout1 = w1.shape[0]
        t2 = pre[o['in']][0][0, :, 1:-1, 1:-1]
        x = pre[o['res']][0][0, :, 1:-1, 1:-1] if o['res'] >= 0 else None
        xd = pre[o['in2']][0][0, :, 1:-1, 1:-1] if o['convd'] else None
        xo, t1 = self.interior(o['out']), self.interior(o['out2'])
        H = t2.shape[1]
        W3, Wd, W1 = w3[:, :cin].t().double(), (w3[:, cin:].t().double() if cd else None), w1.t().double()
        s1 = self.stat('bneck', f'bneck x\' {cin}->{cexp}{" +down" if cd else ""} {H}')
        s2 = self.stat('bneck', f'bneck t1 {cexp}->{cout1} {H}')
        for c0, c1 in chunks(self.B, H * H * (cexp * 3 + cin + cd)):
            a = t2[c0:c1].reshape(-1, cin).double()
            v = a @ W3 + b3.double()
            va = a.abs().float() @ W3.abs().float() + b3.abs()
            if cd:
                d = xd[c0:c1].reshape(-1, cd).double()
                v, va = v + d @ Wd, va + d.abs().float() @ Wd.abs().float()
            else:
                r = x[c0:c1].reshape(-1, cexp).double()
                v, va = v + r, va + r.abs().float()
            v = v.clamp_min(0)
            n1 = cin + cd + 2
            s1.add(xo[c0:c1].reshape(-1, cexp), v, self.u * v.abs() + ETA[self.dcode] + C_ACC * E24 * n1 * va.double(), v.abs())
            e = xo[c0:c1].reshape(-1, cexp).double()                      # t1 from the engine's stored x'
            t = (e @ W1 + b1.double()).clamp_min(0)
            ta = (e.abs().float() @ W1.abs().float() + b1.abs()).double()
            s2.add(t1[c0:c1].reshape(-1, cout1), t, self.u * t.abs() + ETA[self.dcode] + C_ACC * E24 * (cexp + 1) * ta, t.abs())
        for s in (s1, s2):
            if self.dcode == 2 and s.sat >= 65504:
                self.exact_fail.append(f'bneck op {i}: |ref| reaches the fp16 saturation')
        self.halo(f'bneck x\' op {i}', o['out'])
        self.halo(f'bneck t1 op {i}', o['out2'])
        self.extents['bneck'].add((cin, cexp, cout1))
        if cd:
            self.extents['bneck_fold'].add((cin, cd, cexp))

    def op_headfin(self, i, o):
        self.forward(self.img, i, i + 1, self.outs)
        h = self.raw(o['in'])[0]
        H = h.shape[1]
        n_a, a0, NC = H * H * R, o['anchor_offset'], self.nc
        lg = h.reshape(self.B, H * H, -1)[..., :R * (NC + 4 + K)]                # per pixel: conf R*NC | box R*4 | coef R*K
        conf = lg[..., :R * NC].reshape(self.B, n_a, NC).double()
        box = lg[..., R * NC:R * (NC + 4)].reshape(self.B, n_a, 4)
        coef = lg[..., R * (NC + 4):].reshape(self.B, n_a, K).double()
        x = conf - conf.amax(-1, keepdim=True)
        p = x.softmax(-1)
        rj = (2 + 2 * x.abs()) * 2.0 ** -23
        bound = p * (rj + (p * rj).sum(-1, keepdim=True) + 12 * E24) + 2.0 ** -126
        st = self.stat('headfin', f'head softmax level {o["level"]} ({H}x{H})')
        st.add(self.outs[0][:, a0:a0 + n_a], p, bound)
        self.exact(f'head box level {o["level"]}', self.outs[1][:, a0:a0 + n_a], box)
        t = torch.tanh(coef)
        st = self.stat('headfin', f'head tanh level {o["level"]}')
        st.add(self.outs[2][:, a0:a0 + n_a], t, 2.0 ** -22 * t.abs() + 2.0 ** -126)
        self.extents['headfin'].add(o['level'])

    # ---- Swin ----
    def p(self, name):
        return self.sd[name].to(self.dev).double()

    def ln_check(self, kind, label, a_fn, g, b, out, da_fn=None, per=1):
        st = self.stat(kind, label)
        for b0, b1 in chunks(self.B, per):
            a = a_fn(b0, b1)
            y, extra = ln_ref(a, g, b, da_fn(b0, b1) if da_fn else None)
            st.add(out[b0:b1], y, self.u * y.abs() + ETA[self.dcode] + extra, y.abs())
        if self.dcode == 2 and st.sat >= 65504:
            self.exact_fail.append(f'{label}: |ref| reaches the fp16 saturation')

    def op_patch_embed(self, i, o):
        self.forward(self.img, i, i + 1, self.outs)
        out = self.interior(o['out'])
        Hg = out.shape[1]
        pad = 4 * Hg - self.S
        W = self.p('backbone.patch_embed.proj.weight')
        bias = self.p('backbone.patch_embed.proj.bias')

        def conv(b0, b1, absolute=False):
            im = F.pad(self.img[b0:b1].double(), (0, pad, 0, pad))
            return F.conv2d(im.abs() if absolute else im, W.abs() if absolute else W, bias.abs() if absolute else bias, stride=4).permute(0, 2, 3, 1)
        self.ln_check('patch_embed', f'patch embed {self.S}->{Hg}', conv, self.p('backbone.patch_embed.norm.weight'),
                      self.p('backbone.patch_embed.norm.bias'), out, lambda b0, b1: C_ACC * E24 * 49 * conv(b0, b1, True), per=Hg * Hg * 96 * 6)
        self.halo('patch_embed', o['out'])

    def op_ln(self, i, o):
        self.forward(self.img, i, i + 1, self.outs)
        x, out = self.interior(o['in']), self.interior(o['out'])
        self.ln_check('ln', f'{o["p0"].rsplit(".", 1)[0]} {x.shape[1]}', lambda b0, b1: x[b0:b1].double(), self.p(o['p0']), self.p(o['p1']), out,
                      per=x[0].numel() * 6)
        self.halo(o['p0'], o['out'])

    def op_merge_ln(self, i, o):
        self.forward(self.img, i, i + 1, self.outs)
        x, out = self.interior(o['in']), self.interior(o['out'])
        Hin = x.shape[1]

        def gather(b0, b1):
            g = F.pad(x[b0:b1].double(), (0, 0, 0, Hin % 2, 0, Hin % 2))
            return torch.cat([g[:, 0::2, 0::2], g[:, 1::2, 0::2], g[:, 0::2, 1::2], g[:, 1::2, 1::2]], -1)
        self.ln_check('merge_ln', f'merge {Hin}->{out.shape[1]}', gather, self.p(o['p0']), self.p(o['p1']), out, per=x[0].numel() * 8)
        self.halo('merge_ln', o['out'])
        self.extents['merge_ln'].add((Hin, out.shape[1]))

    def op_attn(self, i, o):
        self.forward(self.img, i, i + 1, self.outs)
        qkv, out = self.interior(o['in']), self.interior(o['out'])
        H, C3 = qkv.shape[1], qkv.shape[-1]
        C, heads, shift, ws = C3 // 3, o['heads'], o['shift'], 7
        Hpad = -(-H // ws) * ws
        nW = Hpad // ws
        bias16 = self.sd[o['p0']].to(self.dev).to(self.dt).double()
        table = self.p(o['p1'])
        rel = table[ft._rel_index(ws).view(-1).to(self.dev)].view(49, 49, heads).permute(2, 0, 1)       # [heads, 49, 49]
        mask = ft._shift_mask(Hpad, Hpad, ws, shift).to(self.dev).double() if shift else torch.zeros(nW * nW, 49, 49, dtype=torch.float64,
                                                                                                    device=self.dev)
        scale = float(np.float32(32 ** -0.5))
        st = self.stat('attn', f'attn {H} shift {shift} heads {heads}')
        for b0, b1 in chunks(self.B, Hpad * Hpad * heads * 49 * 8):
            nb = b1 - b0
            g = bias16.view(1, 1, 1, -1).expand(nb, Hpad, Hpad, C3).clone()
            g[:, :H, :H] = qkv[b0:b1].double()
            if shift:
                g = torch.roll(g, shifts=(-shift, -shift), dims=(1, 2))
            win = g.view(nb, nW, ws, nW, ws, C3).permute(0, 1, 3, 2, 4, 5).reshape(-1, 49, 3, heads, 32).permute(2, 0, 3, 1, 4)
            q, k, v = win[0], win[1], win[2]                                                                # [B_, heads, 49, 32]
            sc = q @ k.transpose(-2, -1) * scale
            sa = q.abs() @ k.abs().transpose(-2, -1) * scale
            mw = mask.unsqueeze(1).repeat(nb, 1, 1, 1)                                                      # [B_, 1, 49, 49]
            s = sc + rel.unsqueeze(0) + mw
            ds = C_ACC * 32 * E24 * sa + 3 * E24 * (s.abs() + rel.abs().unsqueeze(0) + 100.0)
            x = s - s.amax(-1, keepdim=True)
            pr = x.softmax(-1)
            rj = ds + E24 * x.abs() + (2 + 1.173 * x.abs()) * 2.0 ** -23
            rl = (pr * rj).sum(-1, keepdim=True) + 64 * E24
            va = v.abs()
            o_ = pr @ v
            pv = pr @ va
            extra = (pr * rj) @ va + pv * (rl + C_ACC * 64 * E24) + 2 * E24 * o_.abs() + ETA[self.dcode] * va.sum(-2, keepdim=True)
            rnd = o_.abs() + pv

            def back(t):
                t = t.transpose(1, 2).reshape(-1, 49, C).view(nb, nW, nW, ws, ws, C).permute(0, 1, 3, 2, 4, 5).reshape(nb, Hpad, Hpad, C)
                if shift:
                    t = torch.roll(t, shifts=(shift, shift), dims=(1, 2))
                return t[:, :H, :H]
            ref, rnd, extra = back(o_), back(rnd), back(extra)
            st.add(out[b0:b1], ref, self.u * rnd + extra, rnd)
        self.extents['attn'].add((H, shift))


# ------------------------------------------------------------------------------------------------
def restate_packed(r):
    """numpy float32 restatement of bn_fold + pack_conv (net.cu) for every GEMM of the program: {(op, which): (w f32, b f32)}."""
    sd = {k: v.numpy() for k, v in r.sd.items() if v.is_floating_point()}
    f = np.float32

    def fold(bn):
        s = sd[bn + '.weight'] / np.sqrt(sd[bn + '.running_var'] + f(1e-5))
        return s, sd[bn + '.bias'] - sd[bn + '.running_mean'] * s

    def pack(wname, bname, bnname, cat=None):
        if cat:
            ws = [sd[n + '.weight'] for n in cat]
            W, b = np.concatenate(ws), np.concatenate([sd[n + '.bias'] for n in cat])
        else:
            W = sd[wname]
            b = sd[bname] if bname else np.zeros(W.shape[0], f)
            if bnname:
                s, t = fold(bnname)
                W = W * s[:, None, None, None]
                b = b * s + t
        if W.ndim == 2:                                        # Swin linears: 1x1 convolutions
            W = W[:, :, None, None]
        cout, cin, k, _ = W.shape
        cin_pad, cout_pad = -(-cin // 64) * 64, (-(-cout // 16) * 16 if cat else cout)
        rows = -(-cout_pad // 64) * 64
        P = np.zeros((rows, k * k, cin_pad), f)
        P[:cout, :, :cin] = W.transpose(0, 2, 3, 1).reshape(cout, k * k, cin)
        B = np.zeros(rows, f)
        B[:cout] = b
        return P.reshape(rows, -1), B

    out = {}
    for i, o in enumerate(r.ops):
        if o['kind'] == 'stem':
            s, t = fold('backbone.bn1')
            src = sd['backbone.conv1.weight']
            W = np.zeros((64, 256), f)
            for dy in range(4):
                for dx in range(4):
                    for py in (0, 1):
                        for px in (0, 1):
                            rr, q = 2 * dy + py - 1, 2 * dx + px - 1
                            if rr >= 0 and q >= 0:
                                c0 = dy * 64 + dx * 16 + (py * 2 + px) * 3
                                W[:, c0:c0 + 3] = src[:, :, rr, q] * s[:, None]
            out[(i, 0)] = (W, t)
        elif o['kind'] in ('conv', 'bneck'):
            if o['w0']:
                w, b = pack(o['w0'], o['b0'], o['bn0'])
            else:
                w, b = pack(None, None, None, cat=('prediction_layers.conf_layer', 'prediction_layers.bbox_layer', 'prediction_layers.coef_layer.0'))
            if o['kind'] == 'bneck' and o['convd']:
                wd, bd = pack(o['wd'], '', o['bnd'])
                w, b = np.concatenate([w, wd], 1), (b, bd)
            out[(i, 0)] = (w, b)
            if o['kind'] == 'bneck':
                out[(i, 1)] = pack(o['w1'], '', o['bn1'])
    return out


def check_packed(r):
    def ulps(a, b):
        return np.abs(a.astype(np.float64) - b) / np.spacing(np.abs(b).astype(np.float32)).astype(np.float64)

    for (i, which), (w, b) in restate_packed(r).items():
        ew, eb = r.weights(i, which)
        ew, eb = ew.cpu(), eb.cpu().numpy()
        if not torch.equal(ew.view(torch.int16), torch.from_numpy(w).to(r.dt).view(torch.int16)):
            r.weight_fail.append((i, which, 'weights differ'))
        if isinstance(b, tuple):                               # b3 + bd in fp32, each within 2 ulps of the restatement
            tol = 2 * (np.spacing(np.abs(b[0])) + np.spacing(np.abs(b[1]))) + np.spacing(np.abs(b[0] + b[1]))
            if not bool((np.abs(eb.astype(np.float64) - (b[0] + b[1])) <= tol).all()):
                r.weight_fail.append((i, which, 'folded bias'))
        elif not bool((ulps(eb, b) <= 2).all()):
            r.weight_fail.append((i, which, f'bias off by {ulps(eb, b).max():.1f} ulp'))


@pytest.fixture(scope='module', params=list(CONFIGS))
def stepped(request, cuda):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    r = Stepped(request.param, cuda)
    c = CONFIGS[request.param]
    with torch.no_grad():
        r.run(stem_only=c.get('stem_only', False), pipelined=c.get('pipelined', False))
        check_packed(r)
    for ln in r.report():
        print(ln)
    print(f'{r.key}: {r.n_ops} ops, {time.time() - t0:.1f} s, peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB')
    yield r
    r.eng = None
    del r
    gc.collect()
    torch.cuda.empty_cache()


def test_ops_against_fp64(stepped):
    r = stepped
    bad = [(k, l, s.worst, s.rel()) for k, l, s in r.stats if not s.ok()]
    assert not bad, f'{len(bad)} op outputs over the bound (kind, op, worst err/bound, rel L2): {bad[:12]}'
    assert not r.exact_fail, r.exact_fail[:12]


def test_halos_are_zero(stepped):
    assert not stepped.halo_fail, f'producers left non-zero halos (op, nonzero count): {stepped.halo_fail[:12]}'


def test_packed_weights(stepped):
    assert not stepped.weight_fail, stepped.weight_fail[:12]


def test_every_op_is_checked(stepped):
    r = stepped
    c = CONFIGS[r.key]
    prog = collections.Counter(o['kind'] for o in r.ops[:1 if c.get('stem_only') else None])
    assert r.census == prog, (r.census, prog)
    if c.get('stem_only'):
        assert r.extents['stem'] == {(64, 550)}
        return
    if r.arch == 'res101' and r.S == 550:
        assert r.extents['bneck'] == BNECK_TRIPLES, r.extents['bneck']
        assert r.extents['bneck_fold'], 'the layer1 downsample fold'
        assert r.extents['split'] == {1, 4}
        assert {(35, 69), (18, 35)} <= r.extents['upadd']
    if r.arch != 'swin_tiny':
        assert r.extents['stem'] == {(16, r.S)}
    assert r.extents['headfin'] == {0, 1, 2, 3, 4}
    assert r.extents['head_ld'] == {HEAD_LD[r.nc]}, r.extents['head_ld']
    if r.arch == 'swin_tiny':
        Hs = {550: (138, 69, 35, 18), 544: (136, 68, 34, 17)}[r.S]
        assert r.extents['attn'] == {(h, s) for h in Hs for s in (0, 3)}, r.extents['attn']
        assert len(r.extents['merge_ln']) == 3


def test_stepped_equals_pipelined(stepped):
    if not CONFIGS[stepped.key].get('pipelined'):
        pytest.skip('checked at the pipelined configurations')
    assert stepped.pipelined_equal, 'the op-by-op run differs from yb_net_forward'
