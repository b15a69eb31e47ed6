"""Per-launch timing of the fused bottleneck kernel k_bneck_tc at the bench shape, against the unfused path in the same process.

    python tools/bench_bneck.py [--arch res101] [--size 550] [--batch 64] [--precision fp16] [--forwards 5] [--json OUT]

Builds the network (synthetic weights, seeded input), runs the engine's per-op profiling pass (CUDA events around every op,
YOLACT_B200_PROFILE_DUMP) and prints one line per k_bneck_tc launch: stage (`layer1→2` / `layer2→3` for the launches that end
a stage and feed the next stage's first conv1), h_out, ms, the algorithmic bytes of the pair (t2 / block input read, x' and t1
written once, both weights) and the rate they imply as a share of the H100 SXM data sheet's 3.35 TB/s.  It then rebuilds the
network with YOLACT_B200_NO_FUSE=1 and prints the k_conv_tc launches that replace each fused launch (conv3 + residual + ReLU,
the next block's conv1 and, for the folded first block of layer1, the downsample convolution),
so the unfused path is the control measured on the same card in the same run.  The card's name, power limit and max SM clock
are read in the same run."""
import argparse
import csv
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HBM_GBS = 3350.0            # NVIDIA H100 SXM data sheet (700 W)
OP_CONV, OP_BNECK = 3, 11   # net.cu OpKind
# (Cin, Cexp, Cout) widths k_bneck_tc fuses (conv_tc.cu bneck_supported): within a stage, and into the next stage's first conv1
FUSED_WIDTHS = {(64, 256, 64), (128, 512, 128), (256, 1024, 256), (64, 256, 128), (128, 512, 256)}


def card():
    import torch
    info = {'gpu': torch.cuda.get_device_name(0), 'power_limit_w': None, 'sm_max_mhz': None}
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(',')
        info['power_limit_w'], info['sm_max_mhz'] = float(out[0]), float(out[1])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return info


def profile_rows(arch, size, batch, precision, forwards, fuse):
    """Per-op rows of the engine's profiling pass, each op's ms averaged over `forwards` forwards."""
    import torch
    from oracle import synth, forward_torch as ft
    from yolact_minimal_b200.config import make_config
    from yolact_minimal_b200.modules.yolact import Yolact
    if fuse:
        os.environ.pop('YOLACT_B200_NO_FUSE', None)
    else:
        os.environ['YOLACT_B200_NO_FUSE'] = '1'
    dev = torch.device('cuda:0')
    cfg = make_config(arch + '_coco', size)
    cfg.precision, cfg.max_batch = precision, batch
    net = Yolact(cfg)
    net.load_state_dict(ft.synth_state_dict(arch, seed=0), strict=True)
    net = net.to(dev).eval()
    img = torch.from_numpy(synth.image_batch(21, batch, size)).to(dev)
    eng = net.engine(batch)
    with torch.no_grad():
        for _ in range(3):
            net(img)
        torch.cuda.synchronize()
        eng.set_profiling(True)
        eng.profile()
        for _ in range(forwards):
            net(img)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, 'ops.csv')
        os.environ['YOLACT_B200_PROFILE_DUMP'] = path
        try:
            eng.profile()
        finally:
            os.environ.pop('YOLACT_B200_PROFILE_DUMP', None)
        rows = list(csv.DictReader(open(path)))
    eng.set_profiling(False)
    os.environ.pop('YOLACT_B200_NO_FUSE', None)
    ops = {}
    for r in rows:
        o = ops.setdefault(int(r['op']), dict({k: int(v) for k, v in r.items() if k not in ('forward', 'ms', 'gflop')}, gflop=float(r['gflop'])))
        o['ms'] = o.get('ms', 0.0) + float(r['ms']) / forwards
    del net, eng
    torch.cuda.empty_cache()
    return [ops[i] for i in sorted(ops)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--arch', default='res101')
    ap.add_argument('--size', type=int, default=550)
    ap.add_argument('--batch', type=int, default=64)
    ap.add_argument('--precision', default='fp16', choices=('fp16', 'bf16'))
    ap.add_argument('--forwards', type=int, default=5)
    ap.add_argument('--json', default=None, help='also write the result as JSON here')
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), 'bench_bneck.py needs a GPU'
    info = card()
    fused = [o for o in profile_rows(args.arch, args.size, args.batch, args.precision, args.forwards, True) if o['kind'] == OP_BNECK]
    plain = profile_rows(args.arch, args.size, args.batch, args.precision, args.forwards, False)

    # the unfused launches of each fused one, in network order: [downsample] conv3 (Cin -> Cexp, + residual) conv1 (Cexp -> Cout)
    groups = []
    for j in range(len(plain) - 1):
        a, b = plain[j], plain[j + 1]
        if (a['kind'] == b['kind'] == OP_CONV and a['k'] == b['k'] == 1 and a['stride'] == b['stride'] == 1 and a['res'] == 1
                and a['cout'] == b['cin'] and a['h_out'] == b['h_out'] and (a['cin'], a['cout'], b['cout']) in FUSED_WIDTHS):
            g = [a, b]
            d = plain[j - 1]
            if d['kind'] == OP_CONV and d['k'] == 1 and d['cout'] == a['cout'] and d['h_out'] == a['h_out']:
                g.insert(0, d)
            groups.append(g)
    assert len(groups) == len(fused), f'{len(fused)} fused launches but {len(groups)} unfused pairs'

    esz = 2
    layer = {h: i + 1 for i, h in enumerate(sorted({o['h_out'] for o in fused}, reverse=True))}
    print(json.dumps(dict(info, arch=args.arch, size=args.size, batch=args.batch, precision=args.precision, forwards=args.forwards)))
    print(f'{"#":>3} {"stage":8} {"h_out":>5} {"Cin":>4} {"Cout":>4} {"fold":>4} {"fused ms":>9} {"MB":>7} {"GB/s":>7} {"%HBM":>5} {"unfused ms":>10} '
          f'{"fused/unfused":>13}')
    launches, tot_f, tot_u, tot_b = [], 0.0, 0.0, 0.0
    for n, (f, g) in enumerate(zip(fused, groups)):
        cin, cexp, cout, px = f['cin'], f['cout'], g[-1]['cout'], float(args.batch) * f['h_out'] ** 2
        assert (g[-2]['cin'], g[-2]['cout'], g[-2]['h_out']) == (cin, cexp, f['h_out']), (f, g)
        stage = f'layer{layer[f["h_out"]]}' + (f'→{layer[f["h_out"]] + 1}' if cout != cin else '')
        fold = len(g) == 3
        nbytes = px * esz * (cin + 2.0 * cexp + cout) + cexp * (cin + cout) * esz           # net.cu yb_net_profile's formula
        if fold:
            cd = g[0]['cin']
            nbytes += px * esz * (cd - cexp) + cexp * cd * esz
        ms_u = sum(o['ms'] for o in g)
        gbs = nbytes / (f['ms'] * 1e-3) / 1e9
        rec = {'launch': n, 'stage': stage, 'h_out': f['h_out'], 'Cin': cin, 'Cout': cout, 'folded_downsample': fold, 'ms': f['ms'],
               'bytes': nbytes, 'gbs': gbs, 'hbm_frac': gbs / HBM_GBS, 'unfused_ms': ms_u, 'unfused_launches': [o['ms'] for o in g]}
        launches.append(rec)
        tot_f += f['ms']; tot_u += ms_u; tot_b += nbytes
        print(f'{n:3d} {stage:8} {f["h_out"]:5d} {cin:4d} {cout:4d} {"yes" if fold else "":>4} {f["ms"]:9.4f} {nbytes / 1e6:7.1f} {gbs:7.0f} '
              f'{100 * gbs / HBM_GBS:4.1f}% {ms_u:10.4f} {f["ms"] / ms_u:13.3f}')
    per_stage = {}
    for r in launches:
        s = per_stage.setdefault(r['stage'], {'launches': 0, 'ms': 0.0, 'unfused_ms': 0.0, 'bytes': 0.0})
        s['launches'] += 1; s['ms'] += r['ms']; s['unfused_ms'] += r['unfused_ms']; s['bytes'] += r['bytes']
    for name, s in sorted(per_stage.items()):
        s['gbs'] = s['bytes'] / (s['ms'] * 1e-3) / 1e9
        print(f'{name}: {s["launches"]} launches, fused {s["ms"]:.3f} ms ({s["gbs"]:.0f} GB/s, {100 * s["gbs"] / HBM_GBS:.1f}% of {HBM_GBS:.0f}), '
              f'unfused {s["unfused_ms"]:.3f} ms, fused/unfused {s["ms"] / s["unfused_ms"]:.3f}')
    summary = {'fused_ms': tot_f, 'unfused_ms': tot_u, 'fused_over_unfused': tot_f / tot_u, 'gbs': tot_b / (tot_f * 1e-3) / 1e9}
    print(json.dumps(summary))
    if args.json:
        with open(args.json, 'w') as fh:
            config = {k: v for k, v in vars(args).items() if k != 'json'}          # the workload, not where the result went
            json.dump(dict(info, config=config, launches=launches, per_stage=per_stage, summary=summary), fh, indent=1)


if __name__ == '__main__':
    main()
