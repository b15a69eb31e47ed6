"""torch.optim.SGD / AdamW as one CUDA launch per step (yb_optim, csrc/optim.cu): the arithmetic of torch's foreach path on CUDA,
bit for bit, over parameters whose gradient is ONE flat fp32 buffer -- the training engine's `grad_flat`, the parameters
concatenated in the engine's kind-0 order.  The optimizer owns its state and belongs to no engine: every engine bound to the same
parameters (one per batch size) steps it.

    opt = NativeOptimizer([tensors[n] for n in eng.param_names], 'sgd', momentum=0.9, weight_decay=5e-4)
    opt.step(eng.grad_flat, lr)                                    # after yb_train_backward; grad_scale = 1 / world after a summed all-reduce

The step writes the parameters through their device pointers: torch sees no in-place op and bumps no `_version`, so a module
whose inference engine caches packed weights needs `refresh_engine()` before it runs inference on the stepped weights.
"""
import ctypes

import torch

from . import _lib

KINDS = {'sgd': 0, 'adamw': 1}


class NativeOptimizer:
    def __init__(self, params, kind, momentum=0.0, weight_decay=0.0, betas=(0.9, 0.999), eps=1e-8):
        if kind not in KINDS:
            raise ValueError(f'optimizer kind must be one of {list(KINDS)}, got {kind!r}')
        params = list(params)
        if not params:
            raise ValueError('NativeOptimizer needs at least one parameter')
        self.device = params[0].device
        for i, p in enumerate(params):
            if p.dtype != torch.float32 or not p.is_contiguous() or p.device != self.device or p.device.type != 'cuda':
                raise ValueError(f'parameter {i}: expected a contiguous float32 CUDA tensor on {self.device}')
        if len({p.data_ptr() for p in params}) != len(params):
            raise ValueError('a parameter is listed twice')
        self.L = _lib.lib()
        self.kind = kind
        self.params = params                                 # keeps the storages the device table points into alive
        self.numel = sum(p.numel() for p in params)
        hp = _lib.OptimParams(KINDS[kind], float(momentum), 0.0, float(weight_decay), float(betas[0]), float(betas[1]), float(eps))
        ptrs = (ctypes.c_void_p * len(params))(*[p.data_ptr() for p in params])
        counts = (ctypes.c_int64 * len(params))(*[p.numel() for p in params])
        h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self.L.yb_optim_create(ctypes.byref(hp), len(params), ptrs, counts, ctypes.byref(h)), 'yb_optim_create')
        self.h = h
        self.steps = 0

    def __del__(self):
        try:
            if getattr(self, 'h', None):
                self.L.yb_optim_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def step(self, grad_flat, lr, grad_scale=1.0):
        """One step with learning rate `lr` on the gradient grad_scale * grad_flat, queued on the current stream."""
        if grad_flat.dtype != torch.float32 or not grad_flat.is_contiguous() or grad_flat.numel() != self.numel \
                or grad_flat.device != self.device:
            raise ValueError(f'grad_flat: expected a contiguous float32 tensor of {self.numel} elements on {self.device}')
        with torch.cuda.device(self.device):
            _lib.check(self.L.yb_optim_step(self.h, grad_flat.data_ptr(), float(lr), float(grad_scale),
                                            torch.cuda.current_stream().cuda_stream), 'yb_optim_step')
        self.steps += 1

    def read_state(self, which=0):
        """Debug / parity tap: the momentum buffer (SGD) or exp_avg (which=0) / exp_avg_sq (which=1, AdamW) in grad_flat's layout."""
        out = torch.empty(self.numel, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self.L.yb_optim_read_state(self.h, which, out.data_ptr(), out.numel(), torch.cuda.current_stream().cuda_stream),
                       'yb_optim_read_state')
        return out
