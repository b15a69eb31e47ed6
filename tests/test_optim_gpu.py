"""GPU: yb_optim_step (csrc/optim.cu) against torch.optim.SGD / AdamW on their foreach CUDA path, bit for bit.

Parameters are the training engine's kind-0 tensors in its order (res50 for SGD, Swin-T for AdamW), placed in one arena with a
sentinel gap of 1-7 floats before each, so that they start at every 16-byte phase.  Six steps, each at its own learning rate, on
gradients written straight into flat buffers: exact zeros (elements and whole tensors), magnitudes from 1e-8 to 1e3,
grad_scale 0.5 on some steps, and a second gradient buffer at an odd offset that stands in for a second engine (and is read with
scalar loads).  After every step the parameters and the optimizer state equal torch's bit for bit, and no sentinel moved."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SENTINEL = -7.25e33


def _engine_params(name, cuda):
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    from yolact_minimal_b200.train import optimizer_params
    from yolact_minimal_b200.train_native import TrainEngine
    net = Yolact(make_config(name, 128, mode='train', train_bs=1)).to(cuda).train()
    eng = TrainEngine(net, 1)
    params = optimizer_params(net, eng.param_names)      # raises unless the engine's kind-0 tensors are the module's parameters
    assert [p.numel() for p in params] == [c for _, c, k in eng.names if k == 0]
    assert eng.grad_flat.numel() == sum(p.numel() for p in params)
    return [p.detach() for p in params]


def _arena(values, cuda, seed):
    rng = np.random.RandomState(seed)
    gaps = rng.randint(1, 8, size=len(values))
    total = int(sum(v.numel() for v in values) + gaps.sum() + 8)
    arena = torch.full((total,), SENTINEL, dtype=torch.float32, device=cuda)
    views, off, inside = [], 0, torch.zeros(total, dtype=torch.bool, device=cuda)
    for v, g in zip(values, gaps):
        off += int(g)
        view = arena[off:off + v.numel()]
        view.copy_(v.reshape(-1))
        inside[off:off + v.numel()] = True
        views.append(view)
        off += v.numel()
    return arena, views, ~inside


def _gradient(n, seed, cuda, sizes):
    g = torch.Generator(device='cpu').manual_seed(seed)
    x = torch.randn(n, generator=g) * torch.pow(10.0, torch.empty(n).uniform_(-8, 3, generator=g))
    x[torch.rand(n, generator=g) < 0.05] = 0.0
    off = 0
    for i, s in enumerate(sizes):                         # whole tensors without a gradient (a head that was not used)
        if (i + seed) % 11 == 0:
            x[off:off + s] = 0.0
        off += s
    return x.to(cuda)


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize('name, kind', [('res50_coco', 'sgd'), ('swin_tiny_coco', 'adamw')])
def test_optimizer_step_is_torch_foreach_bit_for_bit(cuda, name, kind):
    from yolact_minimal_b200.optim import NativeOptimizer
    from yolact_minimal_b200.train import optimizer_settings
    torch.manual_seed(0)
    values = [v.clone() for v in _engine_params(name, cuda)]
    for v in values:                                      # biases start at zero; give every tensor non-trivial values
        v.add_(torch.randn_like(v) * 0.05)
    sizes = [v.numel() for v in values]
    n = sum(sizes)
    assert any(s % 4 for s in sizes), 'the parameter list should have ragged tensors'
    arena, views, outside = _arena(values, cuda, 1)
    sentinels = arena[outside].clone()
    settings = optimizer_settings(name)
    assert settings['kind'] == kind
    opt = NativeOptimizer(views, **settings)
    ref = [torch.nn.Parameter(v.clone().reshape(-1)) for v in values]
    if kind == 'sgd':
        topt = torch.optim.SGD(ref, lr=1.0, momentum=settings['momentum'], weight_decay=settings['weight_decay'], foreach=True)
    else:
        topt = torch.optim.AdamW(ref, lr=1.0, weight_decay=settings['weight_decay'], foreach=True)
    g1 = torch.empty(n, dtype=torch.float32, device=cuda)
    g2_store = torch.empty(n + 3, dtype=torch.float32, device=cuda)
    g2 = g2_store[1:n + 1]                                # a second engine's buffer, 4 bytes past a 16-byte boundary
    lrs = [1e-3, 2e-4, 5.5e-3, 1e-4, 3.3e-3, 7e-4] if kind == 'sgd' else [5e-5, 1e-5, 2.7e-4, 3e-6, 1e-4, 6.1e-5]
    scales = [1.0, 0.5, 1.0, 0.5, 0.5, 1.0]
    for step, (lr, scale) in enumerate(zip(lrs, scales)):
        buf = g1 if step % 2 == 0 else g2
        buf.copy_(_gradient(n, 100 + step, cuda, sizes))
        opt.step(buf, lr, scale)
        grads = (buf * scale).split(sizes)                # scale is 1 or 0.5: exact, as a summed all-reduce over 2 ranks then 1/world
        for p, g in zip(ref, grads):
            p.grad = g.clone()
        for group in topt.param_groups:
            group['lr'] = lr
        topt.step()
        torch.cuda.synchronize()
        for i, (v, p) in enumerate(zip(views, ref)):
            assert torch.equal(_bits(v), _bits(p.detach())), f'step {step}: parameter {i} ({sizes[i]} elements) differs'
        states = ['momentum_buffer'] if kind == 'sgd' else ['exp_avg', 'exp_avg_sq']
        for which, key in enumerate(states):
            mine = opt.read_state(which).split(sizes)
            for i, p in enumerate(ref):
                assert torch.equal(_bits(mine[i]), _bits(topt.state[p][key])), f'step {step}: {key} of parameter {i} differs'
        assert torch.equal(_bits(arena[outside]), _bits(sentinels)), f'step {step}: a sentinel was overwritten'


def test_optimizer_refuses_bad_arguments(cuda):
    from yolact_minimal_b200 import _lib
    from yolact_minimal_b200.optim import NativeOptimizer
    p = [torch.zeros(10, device=cuda), torch.zeros(3, device=cuda)]
    with pytest.raises(_lib.YolactB200Error):
        NativeOptimizer(p, 'sgd', momentum=0.0)
    with pytest.raises(_lib.YolactB200Error):
        NativeOptimizer(p, 'adamw', betas=(0.4, 0.999))
    with pytest.raises(ValueError):
        NativeOptimizer([p[0], p[0]], 'sgd', momentum=0.9)
    opt = NativeOptimizer(p, 'sgd', momentum=0.9)
    with pytest.raises(ValueError):
        opt.step(torch.zeros(12, device=cuda), 1e-3)
