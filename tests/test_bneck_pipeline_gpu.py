"""GPU: the pipelined fused bottleneck kernel k_bneck_tc at launch shapes tests/test_fused_bottleneck_gpu.py does not reach.

Each case is checked BIT FOR BIT against the unfused path (YOLACT_B200_NO_FUSE=1: conv3 + residual + ReLU and the next block's conv1
as two k_conv_tc launches) on the stage output c4 and all four network outputs, with the layer1 downsample branch unfolded
(YOLACT_B200_NO_FUSE_DOWN=1) so both paths round at the same points:
  - the bench shape, res101 550x550 at batch 64: 685 layer3 tiles, 5.2 waves on 132 SMs, more than one tile per CTA at every stage;
  - odd tile counts with a ragged last tile at every fused width (Cmid 64 / 128 / 256), where the last x buffer of a CTA is used
    an odd number of times and the TMA store of xo must stop at the last row;
  - batch 1 at a size where every fused launch has fewer tiles than SMs.
Run-to-run determinism is checked on the same network."""
import os

import pytest
import torch

from oracle import synth, forward_torch as ft

pytestmark = pytest.mark.gpu


def _stage_sizes(S):
    """Output side of layer1, layer2, layer3 (stem stride 2, max-pool stride 2, then layer2 / layer3 stride 2)."""
    h1 = (S - 1) // 2 + 1
    h2 = (h1 - 1) // 2 + 1
    h3 = (h2 - 1) // 2 + 1
    return h2, h3, (h3 - 1) // 2 + 1


def _tiles(B, H):
    rows = B * (H + 2) ** 2                          # haloed rows of one activation
    return (rows + 127) // 128, rows % 128


def _run(arch, S, B, precision, cuda, fuse):
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    saved = {k: os.environ.pop(k, None) for k in ('YOLACT_B200_NO_FUSE', 'YOLACT_B200_NO_FUSE_DOWN')}
    os.environ['YOLACT_B200_NO_FUSE_DOWN'] = '1'
    if not fuse:
        os.environ['YOLACT_B200_NO_FUSE'] = '1'
    try:
        cfg = make_config(arch + '_coco', S)
        cfg.precision, cfg.max_batch = precision, B
        net = Yolact(cfg)
        net.load_state_dict(ft.synth_state_dict(arch, seed=0), strict=True)
        net = net.to(cuda).eval()
        img = torch.from_numpy(synth.image_batch(21, B, S)).to(cuda)
        with torch.no_grad():
            out = [o.clone() for o in net(img)]
            again = [o.clone() for o in net(img)]
        c4 = net.engine(B).read_activation('c4', B).clone()
        torch.cuda.synchronize()
    finally:
        for k, v in saved.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v
    del net
    torch.cuda.empty_cache()
    return out, again, c4


def _check(arch, S, B, precision, cuda):
    fused, fused2, c4f = _run(arch, S, B, precision, cuda, True)
    plain, _, c4p = _run(arch, S, B, precision, cuda, False)
    assert c4f.shape[-1] == _stage_sizes(S)[2]
    assert torch.equal(c4f, c4p), float((c4f - c4p).abs().max())
    for name, a, b, c in zip(('cls', 'box', 'coef', 'proto'), fused, plain, fused2):
        assert torch.equal(a, c), name                                   # run to run
        assert torch.equal(a, b), (name, float((a - b).abs().max()))


def test_bench_shape_bitwise(cuda):
    assert [_tiles(64, h)[0] for h in _stage_sizes(550)] == [9800, 2521, 685]
    _check('res101', 550, 64, 'fp16', cuda)


@pytest.mark.parametrize('arch,S,B,precision', [('res101', 358, 7, 'fp16'), ('res50', 314, 5, 'bf16')])
def test_odd_ragged_tile_counts_bitwise(cuda, arch, S, B, precision):
    for H in _stage_sizes(S):                                            # every fused width: odd tile count, ragged last tile
        n, rem = _tiles(B, H)
        assert n % 2 == 1 and rem != 0, (H, n, rem)
    _check(arch, S, B, precision, cuda)


def test_batch1_fewer_tiles_than_sms_bitwise(cuda):
    assert all(_tiles(1, h)[0] < 132 for h in _stage_sizes(270))
    _check('res101', 270, 1, 'fp16', cuda)
