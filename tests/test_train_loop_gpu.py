"""GPU: `python -m yolact_minimal_b200.train` -- the native step (engine forward and backward, optimizer in one launch) on a
repeated batch, with no host synchronisation in steady state, and short runs through torchrun on a stub COCO: checkpoints under
the reference's names, the refresh of the inference engine (a fresh module loaded from latest_* evaluates to the in-loop rows bit
for bit), --resume, and two ranks that stay identical."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('arch, lr', [('res50', 1e-3), ('swin_tiny', 5e-4)])
def test_native_step_on_a_repeated_batch_never_syncs(cuda, arch, lr):
    from oracle import forward_torch as ft, synth
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    from yolact_minimal_b200.train import NativeTrainer
    torch.manual_seed(0)
    S, B = 128, 2
    net = Yolact(make_config(arch + '_coco', S, mode='train', train_bs=B))
    if arch == 'res50':                                                # BatchNorm statistics of a trained network: xavier alone diverges
        net.load_state_dict(ft.synth_state_dict(arch, seed=0, train=True), strict=True)
    net = net.to(cuda).train()
    img = torch.from_numpy(synth.image_batch(20, B, S)).to(cuda)
    tg, mk = synth.train_targets(1, B, S)
    tgt = [torch.from_numpy(t).to(cuda) for t in tg]
    mks = [torch.from_numpy(m).to(cuda) for m in mk]
    trainer = NativeTrainer(net, arch + '_coco')
    hist = [trainer.step(img, tgt, mks, lr) for _ in range(2)]          # creates the engine and the optimizer
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for _ in range(10):
            hist.append(trainer.step(img, tgt, mks, lr))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    total = torch.stack(hist).sum(1).tolist()
    assert np.isfinite(total).all() and min(total[6:]) < 0.9 * total[0], total
    nbt = [b for n, b in net.named_buffers() if n.endswith('num_batches_tracked')]
    assert all(int(b) == 12 for b in nbt)


def _torchrun(tmp_path, cfg, mode, nproc, port):
    out = tmp_path / f'{cfg}_{mode}.json'
    work = tmp_path / f'{cfg}_{mode}'
    work.mkdir()
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', str(nproc), '--master-addr', '127.0.0.1',
           '--master-port', str(port), os.path.join(ROOT, 'tests', 'train_loop_worker.py'), str(out), cfg, str(work), mode]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-5000:]
    return json.load(open(out))


@pytest.mark.parametrize('cfg, port', [('res50_coco', 29641), ('swin_tiny_coco', 29642)])
def test_short_run_through_torchrun(tmp_path, cuda, cfg, port):
    from yolact_minimal_b200.config import make_config
    res = _torchrun(tmp_path, cfg, 'run', 1, port)
    c = make_config(cfg, 128, mode='train', train_bs=2)
    lr0 = c.lr
    lrs = {int(k): v for k, v in res['lrs'].items()}
    assert sorted(lrs) == list(range(9))
    warm = [(lr0 - lr0 * 0.1) * (s / 2) + lr0 * 0.1 for s in range(3)]
    assert lrs[0] == lr0 and lrs[1] == warm[1] and lrs[2] == lrs[3] == lrs[4] == warm[2]
    assert lrs[5] == lrs[8] == lr0 * 0.1
    assert [e[0] for e in res['evals']] == [4, 8]
    files = res['files']
    assert f'latest_{cfg}_9.pth' in files, files
    best = [f for f in files if f.startswith('best_')]
    assert len(best) == 1 and best[0] in {f'best_{m[1]}_{cfg}_{s}.pth' for s, _, m in res['evals']}, (best, res['evals'])
    assert res['fresh_eval'] == res['evals'][-1], 'the in-loop evaluation did not see the stepped weights'
    assert res['resume_start'] == 9
    rl = {int(k): v for k, v in res['resume_lrs'].items()}
    assert rl == {9: lr0, 10: lr0, 11: lr0 * 0.1 ** 2, 12: lr0 * 0.1 ** 2}, rl
    assert f'latest_{cfg}_13.pth' in res['files_after_resume'] and f'latest_{cfg}_9.pth' not in res['files_after_resume']


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs >= 2 GPUs')
def test_two_ranks_stay_identical(tmp_path, cuda):
    res = _torchrun(tmp_path, 'res50_coco', 'ranks', 2, 29643)
    assert res['world'] == 2 and res['params_finite']
    assert res['params_equal'] and res['buffers_equal'] and res['buffers_numel'] > 0, res
