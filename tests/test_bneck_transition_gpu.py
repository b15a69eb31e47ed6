"""GPU: the fused bottleneck kernel k_bneck_tc at the two stage transitions, where the next block's conv1 is twice as wide as this
block's conv3 input: layer1.2 -> layer2.0 (64 -> 256 -> 128) and layer2.3 -> layer3.0 (128 -> 512 -> 256), in res50 and res101.
The planner fuses them; the layer3 -> layer4 transition (256 -> 1024 -> 512) stays two k_conv_tc launches.

The fused network is checked BIT FOR BIT against the unfused path (YOLACT_B200_NO_FUSE=1) on c2 / c3 / c4 -- c2 and c3 are the x'
the transition launches write -- and all four network outputs, with the layer1 downsample branch unfolded (YOLACT_B200_NO_FUSE_DOWN=1)
so both paths round at the same points:
  - the bench shape, res101 550x550 at batch 64;
  - an odd tile count with a ragged last tile at both transition resolutions, fp16 and bf16;
  - batch 1 with fewer tiles than SMs at both transition resolutions."""
import csv
import os

import pytest
import torch

from oracle import synth, forward_torch as ft

pytestmark = pytest.mark.gpu

OP_CONV, OP_BNECK = 3, 11      # net.cu OpKind


def _stage_sizes(S):
    """Output side of layer1, layer2, layer3 (stem stride 2, max-pool stride 2, then layer2 / layer3 stride 2)."""
    h1 = (S - 1) // 2 + 1
    h2 = (h1 - 1) // 2 + 1
    h3 = (h2 - 1) // 2 + 1
    return h2, h3, (h3 - 1) // 2 + 1


def _tiles(B, H):
    rows = B * (H + 2) ** 2                          # haloed rows of one activation
    return (rows + 127) // 128, rows % 128


def _net(arch, S, B, precision, cuda):
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    cfg = make_config(arch + '_coco', S)
    cfg.precision, cfg.max_batch = precision, B
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict(arch, seed=0), strict=True)
    return net.to(cuda).eval()


def _with_env(env, fn):
    keys = ('YOLACT_B200_NO_FUSE', 'YOLACT_B200_NO_FUSE_DOWN', 'YOLACT_B200_PROFILE_DUMP')
    saved = {k: os.environ.pop(k, None) for k in keys}
    os.environ.update(env)
    try:
        return fn()
    finally:
        for k, v in saved.items():
            os.environ.pop(k, None)
            if v is not None:
                os.environ[k] = v


def _run(arch, S, B, precision, cuda, fuse):
    def go():
        net = _net(arch, S, B, precision, cuda)
        img = torch.from_numpy(synth.image_batch(21, B, S)).to(cuda)
        with torch.no_grad():
            out = [o.clone() for o in net(img)]
            again = [o.clone() for o in net(img)]
        eng = net.engine(B)
        taps = {n: eng.read_activation(n, B).clone() for n in ('c2', 'c3', 'c4')}
        torch.cuda.synchronize()
        del net, eng
        torch.cuda.empty_cache()
        return out, again, taps
    env = {'YOLACT_B200_NO_FUSE_DOWN': '1'}
    if not fuse:
        env['YOLACT_B200_NO_FUSE'] = '1'
    return _with_env(env, go)


def _check(arch, S, B, precision, cuda):
    fused, fused2, tf = _run(arch, S, B, precision, cuda, True)
    plain, _, tp = _run(arch, S, B, precision, cuda, False)
    for n in ('c2', 'c3', 'c4'):
        assert torch.equal(tf[n], tp[n]), (n, float((tf[n] - tp[n]).abs().max()))
    for name, a, b, c in zip(('cls', 'box', 'coef', 'proto'), fused, plain, fused2):
        assert torch.equal(a, c), name                                   # run to run
        assert torch.equal(a, b), (name, float((a - b).abs().max()))


def _ops(arch, S, B, precision, cuda, tmp_path):
    """The engine's op list with each op's kind, widths and resolution (one profiled forward, YOLACT_B200_PROFILE_DUMP)."""
    path = str(tmp_path / f'{arch}_ops.csv')

    def go():
        net = _net(arch, S, B, precision, cuda)
        img = torch.from_numpy(synth.image_batch(21, B, S)).to(cuda)
        eng = net.engine(B)
        eng.set_profiling(True)
        with torch.no_grad():
            net(img)
        torch.cuda.synchronize()
        os.environ['YOLACT_B200_PROFILE_DUMP'] = path
        prof = eng.profile()
        eng.set_profiling(False)
        del net, eng
        return prof
    prof = _with_env({}, go)
    rows = [{k: int(v) for k, v in r.items() if k not in ('ms', 'gflop')} for r in csv.DictReader(open(path))]
    return prof, rows


@pytest.mark.parametrize('arch,fused,conv_tc', [('res101', 29, 67), ('res50', 12, 50)])
def test_transition_launch_counts(cuda, tmp_path, arch, fused, conv_tc):
    prof, rows = _ops(arch, 128, 1, 'fp16', cuda, tmp_path)
    assert prof['bneck_tc']['launches'] == fused
    assert prof['conv_tc']['launches'] == conv_tc
    h1, h2, _ = _stage_sizes(128)
    bn = [r for r in rows if r['kind'] == OP_BNECK]
    # layer1: 2 within the stage + layer1 -> layer2; layer2: 3 + layer2 -> layer3 (the fused op's row carries conv3's widths)
    assert sum(r['h_out'] == h1 and r['cin'] == 64 and r['cout'] == 256 for r in bn) == 3
    assert sum(r['h_out'] == h2 and r['cin'] == 128 and r['cout'] == 512 for r in bn) == 4


def test_layer3_to_layer4_stays_unfused(cuda, tmp_path):
    """(256, 1024, 512) is not a fused width (accB would need 256 registers per thread): layer3.22.conv3 + residual and layer4.0.conv1
    run as two k_conv_tc launches."""
    _, rows = _ops('res101', 128, 1, 'fp16', cuda, tmp_path)
    h3 = _stage_sizes(128)[2]
    pairs = [(a, b) for a, b in zip(rows, rows[1:]) if a['h_out'] == h3 and a['cin'] == 256 and a['cout'] == 1024 and a['res'] == 1
             and b['cin'] == 1024 and b['cout'] == 512 and b['k'] == 1]
    assert len(pairs) == 1, pairs
    a, b = pairs[0]
    assert a['kind'] == b['kind'] == OP_CONV and a['tc'] == b['tc'] == 1


def test_bench_shape_bitwise(cuda):
    _check('res101', 550, 64, 'fp16', cuda)


@pytest.mark.parametrize('arch,S,B,precision', [('res101', 358, 7, 'fp16'), ('res50', 314, 5, 'bf16')])
def test_odd_ragged_tile_counts_bitwise(cuda, arch, S, B, precision):
    for H in _stage_sizes(S)[:2]:                                         # both transition resolutions
        n, rem = _tiles(B, H)
        assert n % 2 == 1 and rem != 0, (H, n, rem)
    _check(arch, S, B, precision, cuda)


def test_batch1_fewer_tiles_than_sms_bitwise(cuda):
    assert all(_tiles(1, h)[0] < 132 for h in _stage_sizes(270)[:2])
    _check('res101', 270, 1, 'fp16', cuda)
