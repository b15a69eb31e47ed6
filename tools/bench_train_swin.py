"""Time one swin_tiny_coco training step on the native engine against the eager torch step on the same GPU:
    python tools/bench_train_swin.py [size] [per_gpu] [steps]
The step is Yolact.forward in train mode + loss.backward() + AdamW (train.py's optimizer for this config).  The eager step is the
torch-autograd checker of tests/swin_train_torch.py (fp32, TF32 and cudnn.benchmark at torch's defaults) on the same inputs."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch  # noqa: E402

import bench  # noqa: E402
from oracle import synth, forward_torch as ft  # noqa: E402
from yolact_minimal_b200.config import make_config  # noqa: E402
from yolact_minimal_b200.modules.yolact import Yolact  # noqa: E402
import swin_train_torch as st  # noqa: E402

S = int(sys.argv[1]) if len(sys.argv) > 1 else 550
per = int(sys.argv[2]) if len(sys.argv) > 2 else 8
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 20
dev = torch.device('cuda:0')
torch.backends.cudnn.benchmark = True


def make():
    cfg = make_config('swin_tiny_coco', S, mode='train', train_bs=per)
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict('swin_tiny', seed=0, train=True), strict=True)
    return net.to(dev).train()


img = torch.from_numpy(synth.image_batch(100, per, S)).to(dev)
tg, mk = synth.train_targets(1, per, S)
tgt = [torch.from_numpy(t).to(dev) for t in tg]
mks = [torch.from_numpy(m).to(dev) for m in mk]
rates = st.drop_rates()


def timed(net, fwd):
    opt = torch.optim.AdamW(net.parameters(), lr=net.cfg.lr, weight_decay=0.05)

    def step(_):
        losses = fwd(net)
        opt.zero_grad(set_to_none=True)
        sum(losses).backward()
        opt.step()
    for i in range(3):
        step(i)
    torch.cuda.synchronize()
    return bench.cuda_time(step, steps)


def eager(net):
    masks = torch.floor(1 - torch.tensor(rates, device=dev).view(1, -1, 1) + torch.rand(per, len(rates), 2, device=dev))
    return st.training_step_forward(net, img, tgt, mks, masks)


native_ms = timed(make(), lambda net: net(img, tgt, mks))
eager_ms = timed(make(), eager)
smi = subprocess.run(['nvidia-smi', '-i', str(dev.index or 0), '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader,nounits'],
                     capture_output=True, text=True).stdout.strip().split(', ')
print(json.dumps({'workload': f'swin_tiny_coco {S}x{S} training step, bs={per}, synthetic targets, AdamW', 'steps': steps,
                  'command': f'python tools/bench_train_swin.py {S} {per} {steps}',
                  'native': 'native engine: bf16 tensor-core operands, fp32 accumulation / statistics / master weights, CUDA-graph replay',
                  'eager': 'NOT the reference Yolact: the fp32 torch-autograd checker tests/swin_train_torch.py (with its tap hooks idle), '
                           'TF32 and cudnn.benchmark at torch defaults',
                  'native_step_ms': round(native_ms, 3), 'eager_torch_step_ms': round(eager_ms, 3),
                  'native_over_eager_checker': round(eager_ms / native_ms, 3),
                  'gpu': smi[0], 'gpu_power_limit_w': float(smi[1]), 'gpu_sm_max_mhz': int(smi[2])}))
