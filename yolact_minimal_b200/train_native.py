"""Training branch of `Yolact.forward` (reference: modules/yolact.py:159-161,:166-313, utils/box_utils.py:57-114) on the native
engine: train-mode forward, target assignment, the four losses and the whole backward pass run in libyolact_b200.so
(csrc/train.cu, losses.cu, train_kernels.cu; wgmma convolutions / weight-gradient GEMMs, CUDA-core BatchNorm and glue).

torch provides what it provides everywhere else in this package: device memory (the fp32 nn.Parameters ARE the master weights
-- the engine reads them and writes their gradients through bound device pointers), streams, and the autograd / DDP plumbing:
the step is ONE autograd.Function whose inputs are the parameters, so `loss.backward()` hands each parameter its gradient
and DistributedDataParallel's hooks (train.py:76) all-reduce them over NCCL exactly as they do for the reference.
ResNet and Swin-T backbones (Swin-T: LayerNorm, window attention, GELU, patch merging and stochastic depth in csrc/swin_train.cu,
its linear layers on the same convolution kernels); 16-bit tensor-core operands (bf16 by default: gradients need the exponent range), fp32 accumulation,
statistics, losses and parameter gradients.
"""
import ctypes
import math

import numpy as np
import torch

from . import _lib

PRECISIONS = {'bf16': 1, 'fp16': 2}


class TrainEngine:
    """One native training program (fixed batch size) bound to a Yolact module's parameters and BN buffers."""

    def __init__(self, module, batch, precision='bf16'):
        if module.depth not in (50, 101, 0):
            raise NotImplementedError('the native training engine covers the res50 / res101 / swin_tiny configs')
        if precision not in PRECISIONS:
            raise ValueError(f'training precision must be one of {list(PRECISIONS)}, got {precision!r}')
        self.L = _lib.lib()
        cfg = module.cfg
        self.device = next(module.parameters()).device
        if self.device.type != 'cuda':
            raise _lib.YolactB200Error('training runs on CUDA only (no CPU fallback): move the model to the GPU')
        self.batch, self.img_size = batch, cfg.img_size
        self.netcfg = _lib.NetConfig(module.depth, cfg.img_size, cfg.num_classes, len(cfg.aspect_ratios), module.coef_dim)
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self.L.yb_train_create(ctypes.byref(self.netcfg), batch, PRECISIONS[precision], ctypes.byref(h)), 'yb_train_create')
        self.h = h
        self.names = []
        for i in range(self.L.yb_train_num_tensors(h)):
            name, cnt, kind = ctypes.c_char_p(), ctypes.c_int64(), ctypes.c_int()
            _lib.check(self.L.yb_train_tensor_info(h, i, ctypes.byref(name), ctypes.byref(cnt), ctypes.byref(kind)), 'yb_train_tensor_info')
            self.names.append((name.value.decode(), cnt.value, kind.value))
        a = module.anchors
        a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a, dtype=np.float64)
        a = np.ascontiguousarray(a.reshape(-1, 4).astype(np.float32))
        _lib.check(self.L.yb_train_set_anchors(h, a.ctypes.data, a.shape[0]), 'yb_train_set_anchors')
        self.hp = _lib.TrainHparams(float(cfg.pos_iou_thre), float(cfg.neg_iou_thre), 3, int(cfg.masks_to_train), float(cfg.conf_alpha),
                                    float(cfg.bbox_alpha), float(cfg.mask_alpha), float(cfg.semantic_alpha), 0.1, 1e-5)
        self.param_names = [n for n, _, k in self.names if k == 0]
        total = sum(c for _, c, k in self.names if k == 0)
        self.grad_flat = torch.zeros(total, dtype=torch.float32, device=self.device)     # the engine writes every gradient here
        self._sig = None
        self.step = 0

    def __del__(self):
        try:
            if getattr(self, 'h', None):
                self.L.yb_train_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def bind(self, tensors):
        """tensors: name -> fp32 CUDA tensor (parameters and BN running statistics).  Re-binds only when a storage moved."""
        sig = tuple(tensors[n].data_ptr() for n, _, _ in self.names)
        if sig == self._sig:
            return
        off = 0
        for name, cnt, kind in self.names:
            t = tensors[name]
            if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() != cnt or t.device != self.device:
                raise ValueError(f'{name}: expected a contiguous float32 tensor of {cnt} elements on {self.device}')
            g = None
            if kind == 0:
                g = self.grad_flat.data_ptr() + 4 * off
                off += cnt
            _lib.check(self.L.yb_train_bind(self.h, name.encode(), t.data_ptr(), g), f'yb_train_bind({name})')
        self._sig = sig

    def grad_views(self, flat):
        out, off = [], 0
        for name, cnt, kind in self.names:
            if kind == 0:
                out.append(flat[off:off + cnt])
                off += cnt
        return out

    def forward(self, img, gt, gt_off, masks, total_gt, max_gt, seed):
        losses = torch.empty(4, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.L.yb_train_forward(self.h, img.data_ptr(), gt.data_ptr(), gt_off.data_ptr(), masks.data_ptr(), total_gt, max_gt,
                                               ctypes.byref(self.hp), seed, losses.data_ptr(), torch.cuda.current_stream().cuda_stream),
                       'yb_train_forward')
        return losses

    def backward(self, loss_grad):
        with torch.cuda.device(self.device):
            _lib.check(self.L.yb_train_backward(self.h, loss_grad.data_ptr(), torch.cuda.current_stream().cuda_stream), 'yb_train_backward')
        return self.grad_flat.clone()                      # autograd may keep / alias what it is handed: never the engine's own buffer

    def read(self, name, grad=False):
        """Debug / parity tap: a named activation (or its gradient) as an NCHW float32 tensor."""
        C, H = ctypes.c_int(), ctypes.c_int()
        _lib.check(self.L.yb_train_read(self.h, name.encode(), 1 if grad else 0, None, 0, ctypes.byref(C), ctypes.byref(H), None), 'yb_train_read')
        out = torch.empty(self.batch, C.value, H.value, H.value, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.L.yb_train_read(self.h, name.encode(), 1 if grad else 0, out.data_ptr(), out.numel(), ctypes.byref(C), ctypes.byref(H),
                                            torch.cuda.current_stream().cuda_stream), 'yb_train_read')
        return out

    def read_output(self, name):
        """Debug / parity tap: a network output as the losses saw it -- 'cls' [B,A,C] raw logits, 'box' [B,A,4], 'coef' [B,A,K] (tanh),
        'proto' [B,P,P,K], 'seg' [B,Hs,Hs,C-1] (NHWC); Swin-T: 'drop_path' [B,12,2], the last step's stochastic-depth masks (block,
        attention | MLP branch)."""
        C, H = ctypes.c_int(), ctypes.c_int()
        key = ('out.' + name).encode()
        _lib.check(self.L.yb_train_read(self.h, key, 0, None, 0, ctypes.byref(C), ctypes.byref(H), None), 'yb_train_read')
        shape = (self.batch, H.value, C.value) if name in ('cls', 'box', 'coef', 'drop_path') else (self.batch, H.value, H.value, C.value)
        out = torch.empty(shape, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.L.yb_train_read(self.h, key, 0, out.data_ptr(), out.numel(), ctypes.byref(C), ctypes.byref(H),
                                            torch.cuda.current_stream().cuda_stream), 'yb_train_read')
        return out

    def launches_per_step(self):
        return int(self.L.yb_train_launches_per_step(self.h))


class _NativeTrainStep(torch.autograd.Function):
    """losses[4] = f(parameters): forward and backward both run in the native engine."""

    @staticmethod
    def forward(ctx, eng, img, gt, gt_off, masks, total_gt, max_gt, seed, *params):
        ctx.eng = eng
        ctx.keep = (gt, gt_off, masks)                 # the backward pass re-reads the targets through the engine's raw pointers
        return eng.forward(img, gt, gt_off, masks, total_gt, max_gt, seed)

    @staticmethod
    def backward(ctx, grad_losses):
        eng = ctx.eng
        flat = eng.backward(grad_losses.to(torch.float32).contiguous())
        return (None,) * 8 + tuple(v.view_as(p) for v, p in zip(eng.grad_views(flat), eng._params))


def training_step(net, img, box_classes, masks_gt):
    """Yolact.forward in training mode: the reference's 4-tuple (category, box, mask, semantic) of losses."""
    if not img.is_cuda:
        raise RuntimeError('yolact_minimal_b200.Yolact trains on CUDA only (no CPU fallback): move the model and input to the GPU')
    B, S = img.shape[0], net.cfg.img_size
    if tuple(img.shape[1:]) != (3, S, S):
        raise ValueError(f'expected input [B,3,{S},{S}], got {tuple(img.shape)}')
    engines = net.__dict__.setdefault('_train_engines', {})
    precision = getattr(net.cfg, 'train_precision', None) or 'bf16'
    key = (B, precision, img.device.index)
    eng = engines.get(key)
    if eng is None:
        eng = engines[key] = TrainEngine(net, B, precision)
    cache = net.__dict__.get('_train_tensor_cache')
    if cache is None or any(t is not u for (_, t), u in zip(cache[1], cache[2]())):        # a parameter / buffer object was replaced
        tensors = dict(net.named_parameters())
        tensors.update(dict(net.named_buffers()))
        objs = [(n, tensors[n]) for n, _, _ in eng.names]
        holders = [(net.get_submodule(n.rsplit('.', 1)[0]) if '.' in n else net, n.rsplit('.', 1)[-1]) for n, _, _ in eng.names]
        getter = lambda: [m._parameters[a] if a in m._parameters else m._buffers[a] for m, a in holders]
        bns = [b for n, b in net.named_buffers() if n.endswith('num_batches_tracked')]
        cache = net.__dict__['_train_tensor_cache'] = (tensors, objs, getter, bns)
    tensors = cache[0]
    eng.bind(tensors)
    eng._params = [tensors[n] for n in eng.param_names]
    dev = img.device
    counts = [int(t.shape[0]) for t in box_classes]
    gt = torch.cat([t.to(dev, torch.float32).reshape(-1, 5) for t in box_classes]).contiguous()
    masks = torch.cat([m.to(dev, torch.float32).reshape(-1, S, S) for m in masks_gt]).contiguous()
    gt_off = torch.tensor(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32), device=dev)
    if gt.shape[0] == 0:
        raise ValueError('training needs at least one ground-truth box in the batch')
    seed = int(torch.randint(0, 2 ** 31 - 1, (1,)).item())             # host RNG (like the reference's torch.randperm, yolact.py:263)
    losses = _NativeTrainStep.apply(eng, img.detach().to(torch.float32).contiguous(), gt, gt_off, masks, int(gt.shape[0]), max(counts), seed,
                                    *eng._params)
    if cache[3]:
        torch._foreach_add_(cache[3], 1)
    return tuple(losses.unbind(0))
