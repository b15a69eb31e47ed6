"""CPU: the Swin-T training checker (tests/swin_train_torch.py) against the reference.

  * tests/golden/train_swin.npz, minted by the unmodified reference (tests/golden/make_golden_train_swin.py) with the stochastic-depth
    draws of the engine for the golden step's seed: the four losses and every parameter's gradient;
  * with nothing dropped, the checker's backbone equals oracle/forward_torch.swin_backbone (the reference's eval forward, restated)."""
import numpy as np
import torch

import swin_train_torch as st
import train_checks as tc
from conftest import load_golden
from oracle import synth, forward_torch as ft
from swin_golden import S, B, SEED_STEP, grad_sample, step_seed, swin_drop_masks


def _inputs():
    img = torch.from_numpy(synth.image_batch(11, B, S))
    tg, mk = synth.train_targets(5, B, S)
    return img, [torch.from_numpy(t) for t in tg], [torch.from_numpy(m) for m in mk]


def test_golden_draws_are_the_engines_for_its_seed():
    g = load_golden('train_swin.npz')
    assert int(g['seed']) == step_seed(SEED_STEP)
    assert np.array_equal(g['masks'], swin_drop_masks(int(g['seed']), B))
    assert (g['masks'][:, 0] == 1).all() and (g['masks'] == 0).any()          # block 0 never dropped; the golden step drops some paths


def test_swin_checker_matches_reference_training_step():
    g = load_golden('train_swin.npz')
    net = tc.make_train_net('swin_tiny', S, B, 'cpu')
    img, tgt, mks = _inputs()
    losses = st.training_step_forward(net, img, tgt, mks, torch.from_numpy(g['masks']))
    got = np.asarray([float(l.detach()) for l in losses])
    assert np.allclose(got, g['losses'], rtol=2e-3), (got, g['losses'])
    sum(losses).backward()
    named = dict(net.named_parameters())
    assert {k[len('grad/'):] for k in g.files if k.startswith('grad/')} == set(named)
    for n, p in named.items():
        gs = grad_sample(n, p.grad.numpy())
        want = g['grad/' + n]
        assert tc.rel(gs, want) < 1e-3 and (tc.cos(gs, want) > 0.999 or not want.any()), (n, tc.rel(gs, want), tc.cos(gs, want))
        assert abs(float(p.grad.double().norm()) / max(float(g['norm/' + n]), 1e-30) - 1) < 1e-3 or float(g['norm/' + n]) == 0, n


def test_swin_checker_without_drops_equals_the_eval_forward(monkeypatch):
    monkeypatch.setattr(st, 'drop_rates', lambda: [0.0] * 12)
    net = tc.make_train_net('swin_tiny', S, B, 'cpu')
    img, _, _ = _inputs()
    taps = {}
    with torch.no_grad():
        st.forward_train(net, img, torch.ones(B, 12, 2), taps)
        ref = ft.swin_backbone(img, net.state_dict())
    for name, i in (('c3', 1), ('c4', 2), ('c5', 3)):
        assert float((taps[name] - ref[i]).abs().max()) < 1e-5 * float(ref[i].abs().max()) + 1e-5, name
