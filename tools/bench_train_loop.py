"""Time `python -m yolact_minimal_b200.train`'s step against the reference-style step on this package, on one GPU:
    python tools/bench_train_loop.py [--size 550] [--bs 8] [--steps 20] [--rounds 4] [--out FILE]
Workloads: res101_coco (SGD) and swin_tiny_coco (AdamW) at size x size, bs images, one resident synthetic batch.
  native step    : NativeTrainer.step -- engine forward + backward into grad_flat, the optimizer as one yb_optim_step launch
  reference step : train-mode Yolact (the same engine behind autograd), loss.backward(), torch.optim foreach step
The two arms alternate in rounds within this one command and are timed with CUDA events.  The optimizer alone is timed the same
way: yb_optim_step against optimizer.step() on the same parameters, with its algorithmic bytes (fused: SGD reads p, g, buf and
writes p, buf = 20 B per parameter; AdamW 28 B) over 3.35 TB/s, the H100 SXM data-sheet HBM3 bandwidth."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from oracle import synth  # noqa: E402
from yolact_minimal_b200.config import make_config  # noqa: E402
from yolact_minimal_b200.modules.yolact import Yolact  # noqa: E402
from yolact_minimal_b200.train import NativeTrainer, optimizer_settings  # noqa: E402

HBM_BPS = 3.35e12
FUSED_BYTES = {'sgd': 20, 'adamw': 28}


def events(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def torch_optimizer(net, settings, lr):
    if settings['kind'] == 'sgd':
        return torch.optim.SGD(net.parameters(), lr=lr, momentum=settings['momentum'], weight_decay=settings['weight_decay'], foreach=True)
    return torch.optim.AdamW(net.parameters(), lr=lr, weight_decay=settings['weight_decay'], foreach=True)


def run(name, S, bs, steps, rounds, dev):
    cfg = make_config(name, S, mode='train', train_bs=bs)
    settings = optimizer_settings(name)
    img = torch.from_numpy(synth.image_batch(100, bs, S)).to(dev)
    tg, mk = synth.train_targets(1, bs, S)
    tgt = [torch.from_numpy(t).to(dev) for t in tg]
    mks = [torch.from_numpy(m).to(dev) for m in mk]
    torch.manual_seed(0)
    net_n = Yolact(cfg).to(dev).train()
    net_r = Yolact(cfg).to(dev).train()
    net_r.load_state_dict(net_n.state_dict())
    trainer = NativeTrainer(net_n, name)
    opt_r = torch_optimizer(net_r, settings, cfg.lr)

    def native():
        trainer.step(img, tgt, mks, cfg.lr)

    def reference():
        losses = net_r(img, tgt, mks)
        opt_r.zero_grad()
        sum(losses).backward()
        opt_r.step()

    for _ in range(3):
        native()
        reference()
    torch.cuda.synchronize()
    nat, ref = [], []
    for _ in range(rounds):
        nat.append(events(native, steps))
        ref.append(events(reference, steps))
    # the optimizer alone, on the gradients the last steps left
    eng = next(iter(net_n.__dict__['_train_engines'].values()))
    n_params = sum(p.numel() for p in net_n.parameters())
    o_nat, o_ref = [], []
    for _ in range(rounds):
        o_nat.append(events(lambda: trainer.opt.step(eng.grad_flat, cfg.lr), 50))
        o_ref.append(events(opt_r.step, 50))
    med = lambda xs: sorted(xs)[len(xs) // 2]
    fused_bytes = FUSED_BYTES[settings['kind']] * n_params
    return {'cfg': name, 'optimizer': settings['kind'], 'params': n_params,
            'native_step_ms': round(med(nat), 3), 'reference_step_ms': round(med(ref), 3),
            'native_step_ms_rounds': [round(x, 3) for x in nat], 'reference_step_ms_rounds': [round(x, 3) for x in ref],
            'step_speedup': round(med(ref) / med(nat), 3),
            'optim_native_ms': round(med(o_nat), 4), 'optim_torch_foreach_ms': round(med(o_ref), 4),
            'optim_native_ms_rounds': [round(x, 4) for x in o_nat], 'optim_torch_ms_rounds': [round(x, 4) for x in o_ref],
            'optim_fused_bytes': fused_bytes,
            'optim_native_tb_s': round(fused_bytes / (med(o_nat) * 1e-3) / 1e12, 3),
            'optim_native_share_of_3_35_tb_s': round(fused_bytes / HBM_BPS / (med(o_nat) * 1e-3), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--size', type=int, default=550)
    ap.add_argument('--bs', type=int, default=8)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=4)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    dev = torch.device('cuda:0')
    torch.cuda.set_device(dev)
    rows = [run(name, a.size, a.bs, a.steps, a.rounds, dev) for name in ('res101_coco', 'swin_tiny_coco')]
    smi = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader,nounits'],
                         capture_output=True, text=True).stdout.strip().split(', ')
    res = {'workload': f'training step at {a.size}x{a.size}, bs={a.bs}, one resident synthetic batch, {a.steps} steps x {a.rounds} '
                       'alternating rounds (medians)',
           'command': f'python tools/bench_train_loop.py --size {a.size} --bs {a.bs} --steps {a.steps} --rounds {a.rounds}',
           'native': 'NativeTrainer.step: engine forward + backward into grad_flat, yb_optim_step (one launch)',
           'reference': 'train-mode Yolact of this package under autograd, loss.backward(), torch.optim foreach step',
           'rows': rows, 'gpu': smi[0], 'gpu_power_limit_w': float(smi[1]), 'gpu_sm_max_mhz': int(smi[2])}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
