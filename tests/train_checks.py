"""Shared by tests/test_train_gpu.py and tools/diag_train.py: run the native training kernels / engine and the checkers
(oracle/train_np.py, oracle/train_torch.py, reference-minted goldens) on the same seeded inputs and return the comparisons."""
import ctypes

import numpy as np
import torch

from conftest import load_golden
from oracle import synth, forward_torch as ft, train_torch as tt

S_ST, B_ST, NCLS = 128, 3, 81


def stage_inputs(g):
    A, P = g['anchors'].shape[0], S_ST // 4
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    tg, mk = synth.train_targets(9, B_ST, S_ST, n=4)
    class_p = f32(synth.normal(21, 1, (B_ST, A, NCLS)) * 2)
    box_p = f32(synth.normal(21, 2, (B_ST, A, 4)) * 0.5)
    coef_p = np.tanh(f32(synth.normal(21, 3, (B_ST, A, 32))))
    proto_p = np.maximum(f32(synth.normal(21, 4, (B_ST, P, P, 32))), 0)
    seg_p = f32(synth.normal(21, 5, (B_ST, NCLS - 1, S_ST // 8, S_ST // 8)))
    return tg, mk, class_p, box_p, coef_p, proto_p, seg_p


def run_native_losses(dev, cfg, anchors, tg, mk, class_p, box_p, coef_p, proto_p, seg_nchw, grads=True, grad_scale=None, seed=1,
                      pos_iou_thr=None, neg_iou_thr=None, masks_to_train=None, ld_seg=None, sentinel=None, check=True):
    """yb_losses through ctypes.  Returns dict(losses, labels, matched_idx, offsets, neg, d_cls, d_box, d_coef, d_proto, d_seg (NCHW)).
    pos_iou_thr / neg_iou_thr / masks_to_train override cfg; the coefficient dimension is coef_p's last.  ld_seg > C-1 pads every
    seg row with columns the kernels must neither read (they hold NaN) nor leave unwritten (d_seg_nhwc keeps them).  grad_scale is
    passed in device memory.  sentinel: fill every output with this value before the call (integer outputs with int(sentinel)).
    check=False returns dict(status=..., outputs) instead of raising when yb_losses refuses the call."""
    from yolact_minimal_b200 import _lib
    L = _lib.lib()
    t = lambda a, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(a)).to(dev, dt)
    B, A, C = class_p.shape
    K, P, Hs, S = coef_p.shape[-1], proto_p.shape[1], seg_nchw.shape[-1], mk[0].shape[-1]
    ld = C - 1 if ld_seg is None else ld_seg
    cls, box, coef, proto = t(class_p), t(box_p), t(coef_p), t(proto_p)
    seg = torch.full((B, Hs, Hs, ld), float('nan'), device=dev)            # the engine's layout: NHWC, row stride ld
    seg[..., :C - 1] = t(seg_nchw).permute(0, 2, 3, 1)
    gt = t(np.concatenate(tg).reshape(-1, 5)); masks = t(np.concatenate(mk))  # exactly total_gt rows
    counts = [len(x) for x in tg]
    gt_off = torch.tensor(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32), device=dev)
    thr = lambda v, d: float(d if v is None else v)
    p = _lib.LossParams(B, A, C, K, P, Hs, S, thr(pos_iou_thr, cfg.pos_iou_thre), thr(neg_iou_thr, cfg.neg_iou_thre), 3,
                        int(cfg.masks_to_train if masks_to_train is None else masks_to_train), float(cfg.conf_alpha),
                        float(cfg.bbox_alpha), float(cfg.mask_alpha), float(cfg.semantic_alpha))
    ws = torch.empty(max(1, int(L.yb_losses_workspace_bytes(ctypes.byref(p), int(gt.shape[0])))), dtype=torch.uint8, device=dev)
    fi = 0 if sentinel is None else int(sentinel)
    out = dict(losses=torch.full((4,), 0.0 if sentinel is None else float(sentinel), device=dev),
               labels=torch.full((B, A), fi, dtype=torch.int32, device=dev), matched_idx=torch.full((B, A), fi, dtype=torch.int32, device=dev),
               offsets=torch.full((B, A, 4), 0.0 if sentinel is None else float(sentinel), device=dev),
               neg=torch.full((B, A), fi & 255, dtype=torch.uint8, device=dev))
    if grads:
        fv = 7.0 if sentinel is None else float(sentinel)
        out.update(d_cls=torch.full_like(cls, fv), d_box=torch.full_like(box, fv), d_coef=torch.full_like(coef, fv), d_proto=torch.full_like(proto, fv),
                   d_seg=torch.full_like(seg, fv))
    ptr = lambda k: out[k].data_ptr() if k in out else None
    gs = None if grad_scale is None else t(np.asarray(grad_scale, np.float32))
    status = L.yb_losses(ctypes.byref(p), cls.data_ptr(), box.data_ptr(), coef.data_ptr(), proto.data_ptr(), seg.data_ptr(), ld, t(anchors).data_ptr(),
                         gt.data_ptr(), gt_off.data_ptr(), masks.data_ptr(), int(gt.shape[0]), max(counts), seed, None if gs is None else gs.data_ptr(),
                         out['losses'].data_ptr(), ptr('d_cls'), ptr('d_box'), ptr('d_coef'), ptr('d_proto'), ptr('d_seg'), out['labels'].data_ptr(),
                         out['matched_idx'].data_ptr(), out['offsets'].data_ptr(), out['neg'].data_ptr(), ws.data_ptr(), ws.numel(),
                         torch.cuda.current_stream().cuda_stream)
    if check:
        _lib.check(status, 'yb_losses')
    torch.cuda.synchronize()
    if grads:
        out['d_seg_nhwc'] = out['d_seg']
        out['d_seg'] = out['d_seg'][..., :C - 1].permute(0, 3, 1, 2).contiguous()
    res = {k: v.cpu().numpy() for k, v in out.items()}
    if not check:
        res['status'] = int(status)
    return res


def torch_losses_and_grads(cfg, anchors, tg, mk, class_p, box_p, coef_p, proto_p, seg_p, grad_scale=(1, 1, 1, 1)):
    """The checker: oracle/train_torch.py's four losses and torch-autograd gradients w.r.t. the five network outputs (fp32 on CPU)."""
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).float().requires_grad_(True)
    cls, box, coef, proto, seg = t(class_p), t(box_p), t(coef_p), t(proto_p), t(seg_p)
    anc = torch.from_numpy(anchors).float()
    B = class_p.shape[0]
    out = [tt.assign_targets(cfg, torch.from_numpy(tg[i][:, :4]).float(), anc, torch.from_numpy(tg[i][:, 4]).long()) for i in range(B)]
    offsets, labels, matched, idx = (torch.stack(x) for x in zip(*out))
    pos = labels > 0
    masks = [torch.from_numpy(m).float() for m in mk]
    losses = (tt.category_loss(cfg, cls, labels, pos), tt.box_loss(cfg, box, offsets, pos), tt.mask_loss(cfg, pos, idx, coef, proto, masks, matched),
              tt.semantic_loss(cfg, seg, masks, [torch.from_numpy(x[:, 4]).long() for x in tg]))
    sum(w * l for w, l in zip(grad_scale, losses)).backward()
    return [float(l) for l in losses], dict(d_cls=cls.grad.numpy(), d_box=box.grad.numpy(), d_coef=coef.grad.numpy(), d_proto=proto.grad.numpy(),
                                            d_seg=seg.grad.numpy())


def make_train_net(arch, S, B, dev, config=None, num_classes=None):
    """A training-mode Yolact with synthetic weights.  config: a config name (default arch + '_coco'); num_classes (background
    included) overrides the config's class count, for the counts no config has."""
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    cfg = make_config(config or arch + '_coco', S, mode='train', train_bs=B)
    if num_classes is not None:
        cfg.num_classes = num_classes
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict(arch, num_classes=cfg.num_classes, seed=0, train=True), strict=True)
    return net.to(dev).train()


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-30))


def cos(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(a @ b / (np.linalg.norm(a) * np.linalg.norm(b) + 1e-30))


TAPS = ('stem.y', 'stem.z', 'pool', 'c2', 'c3', 'c4', 'c5', 'p5_1', 'p4_1', 'p3_1', 'p3', 'p4', 'p5', 'p6', 'p7', 'proto1.4', 'proto.up')


def engine_vs_checker(arch, S, B, dev, precision='bf16', img_seed=11, tgt_seed=5, mode='fp32'):
    """One native training step and one checker step (torch autograd on the GPU, TF32 off) from identical parameters and inputs.
    mode 'fp32'      the reference's arithmetic: how far a 16-bit training step is from fp32 (losses, gradient direction)
         'emulate'   the checker's forward rounds where the engine rounds (oracle/train_torch.forward_train act=)
         'subst'     the checker is evaluated AT the engine's stored activations (forward_train subst=): identical ReLU masks and
                     batch statistics, so the comparison isolates the engine's BACKWARD arithmetic (dgrad / wgrad / BN / pooling / ...)
    Returns dict(losses, ref_losses, act={tap: rel err}, gact={tap: rel err of the gradient}, grads={param: (rel err, cosine, ref norm)},
    bn={buffer: max abs err}, launches)."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    img = torch.from_numpy(synth.image_batch(img_seed, B, S)).to(dev)
    tg, mk = synth.train_targets(tgt_seed, B, S)
    tgt = [torch.from_numpy(t).to(dev) for t in tg]
    mks = [torch.from_numpy(m).to(dev) for m in mk]
    net = make_train_net(arch, S, B, dev)
    net.cfg.train_precision = precision
    losses = net(img, tgt, mks)
    sum(losses).backward()
    torch.cuda.synchronize()
    eng = next(iter(net._train_engines.values()))
    ref = make_train_net(arch, S, B, dev)
    taps = {}
    act = (torch.bfloat16 if precision == 'bf16' else torch.float16) if mode in ('emulate', 'subst') else None
    cache = {}

    def subst(name):
        if name not in cache:
            try:
                if name.startswith('out.'):
                    v = eng.read_output(name[4:])
                    cache[name] = v[..., :net.cfg.num_classes - 1].permute(0, 3, 1, 2).contiguous() if name == 'out.seg' else v   # engine: NHWC; checker: NCHW
                else:
                    cache[name] = eng.read(name)
            except Exception:
                cache[name] = None
        return cache[name]
    ref_losses = tt.training_step_forward(ref, img, tgt, mks, taps, act, subst if mode == 'subst' else None)
    sum(ref_losses).backward()
    out = dict(losses=[float(l.detach()) for l in losses], ref_losses=[float(l.detach()) for l in ref_losses], act={}, gact={}, grads={}, bn={},
               launches=eng.launches_per_step(), substituted=sum(v is not None for v in cache.values()))
    relu_out = lambda n: n in ('p3', 'p4', 'p5', 'p6', 'p7', 'proto2.0') or n.startswith(('proto1.', 'head.f'))     # the engine masks these gradients in place
    for name in taps:
        if name.startswith('out.'):
            continue
        try:
            out['act'][name] = rel(eng.read(name).cpu().numpy(), taps[name].detach().cpu().numpy())
            if taps[name].grad is not None and not relu_out(name):
                out['gact'][name] = rel(eng.read(name, grad=True).cpu().numpy(), taps[name].grad.cpu().numpy())
        except Exception as e:                                        # a tap without a gradient buffer etc.
            out['act'].setdefault(name, repr(e)[:80])
    rp = dict(ref.named_parameters())
    for n, p in net.named_parameters():
        g, r = p.grad, rp[n].grad
        if g is None or r is None:
            out['grads'][n] = (float('nan'), float('nan'), 0.0)
            continue
        g, r = g.cpu().numpy(), r.cpu().numpy()
        out['grads'][n] = (rel(g, r), cos(g, r), float(np.linalg.norm(r)))
    rb = dict(ref.named_buffers())
    for n, b in net.named_buffers():
        out['bn'][n] = float((b.double() - rb[n].double()).abs().max())
    return out
