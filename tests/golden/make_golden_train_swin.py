#!/usr/bin/env python
"""Golden of one Swin-T training step (TEST INFRASTRUCTURE), minted by the UNMODIFIED reference on the CPU:

  YOLACT_REFERENCE=<checkout> python tests/golden/make_golden_train_swin.py      # writes tests/golden/train_swin.npz

swin_tiny_coco at S = 128, B = 2, synthetic weights synth_state_dict('swin_tiny', train=True), inputs from oracle/synth.py.
Stochastic depth: DropPath.forward is wrapped HERE (the reference is not modified) so that each call applies the mask the native
engine draws for the step's seed (swin_drop_masks below restates its counter hash, csrc/swin_train.cu).  The same masks can then be
handed to the checker on the CPU and are drawn by the engine on the GPU, so all three compute the same step.  Written: the seed,
the masks [B, 12, 2], the four losses, and per parameter its gradient norm and the gradient at a fixed sample of <= 512 elements
(every element for tensors of <= 4096)."""
import contextlib
import io
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from oracle import synth, forward_torch as ft, ref_loader  # noqa: E402
from swin_golden import S, B, SEED_STEP, swin_drop_masks, step_seed, grad_sample  # noqa: E402


def main():
    torch.set_num_threads(os.cpu_count())
    rcfg, ryolact, _, _ = ref_loader.load()
    rswin = sys.modules['modules.swin_transformer']
    seed = step_seed(SEED_STEP)
    masks = swin_drop_masks(seed, B)
    calls = []

    def drop_forward(self, x):                                    # DropPath.forward (:68-80) with the given draws
        k = len(calls)                                            # block 0 (rate 0) is nn.Identity: calls start at block 1
        calls.append(k)
        if self.drop_prob == 0. or not self.training:
            return x
        keep_prob = 1 - self.drop_prob
        m = torch.from_numpy(masks[:, 1 + k // 2, k % 2]).to(x.dtype).view((x.shape[0],) + (1,) * (x.ndim - 1))
        return x.div(keep_prob) * m
    rswin.DropPath.forward = drop_forward
    ns = types.SimpleNamespace(cfg='swin_tiny_coco', img_size=S, weight=None, traditional_nms=False, resume=None, train_bs=B,
                               val_interval=-1, val_num=-1, coco_api=False)
    with contextlib.redirect_stdout(io.StringIO()):
        cfg = rcfg.get_config(ns, 'train')
    net = ryolact.Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict('swin_tiny', seed=0, train=True), strict=True)
    net.train()
    img = torch.from_numpy(synth.image_batch(11, B, S))
    tg, mk = synth.train_targets(5, B, S)
    losses = net(img, [torch.from_numpy(t) for t in tg], [torch.from_numpy(m) for m in mk])
    assert len(calls) == 22, len(calls)                           # two DropPath calls per block, blocks 1..11
    sum(losses).backward()
    out = dict(seed=np.int64(seed), masks=masks, losses=np.asarray([float(l) for l in losses], np.float64))
    for n, p in net.named_parameters():
        out['norm/' + n] = np.float64(p.grad.double().norm())
        out['grad/' + n] = grad_sample(n, p.grad.numpy())
    np.savez_compressed(os.path.join(HERE, 'train_swin.npz'), **out)
    print('swin train golden: seed', seed, 'dropped', int((masks == 0).sum()), 'losses', out['losses'].tolist())


if __name__ == '__main__':
    main()
