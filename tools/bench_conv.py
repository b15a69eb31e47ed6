"""Per-launch timing of the tensor-core convolution k_conv_tc at the bench shape.

    python tools/bench_conv.py [--arch res101] [--size 550] [--batch 64] [--precision fp16] [--forwards 5] [--json OUT]

Builds the network (synthetic weights, seeded input), runs the engine's per-op profiling pass (CUDA events around every op,
YOLACT_B200_PROFILE_DUMP) and prints one line per k_conv_tc launch, the stem included (its row also holds the space-to-depth
repack launch): op index, layer shape, tile width BN, tiles and tiles per CTA, ms, the algorithmic FLOP and bytes (net.cu
yb_net_profile's formulas), the rates they imply, and the share of the larger of the two H100 SXM data-sheet bounds (989 TFLOP/s
dense fp16 / bf16, 3.35 TB/s HBM3) that the launch reaches.  The card's name, power limit and max SM clock are read in the same run."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_bneck import card, profile_rows  # noqa: E402

TFLOPS, HBM_GBS = 989.0, 3350.0          # NVIDIA H100 SXM data sheet (700 W)
OP_STEM, OP_CONV = 0, 3                  # net.cu OpKind
TILE_WIDTHS = (256, 192, 176, 128, 96, 64, 32, 16)      # conv_tc.cu kTileWidths, widest first
BM = 128


def launch_row(o, batch, sms, esz):
    stem = o['kind'] == OP_STEM
    cin, cout, k = (64, 64, 2) if stem else (o['cin'], o['cout'], o['k'])     # the stem runs as a 4-tap K = 64 GEMM
    h = (o['img'] - 1) // 2 + 1 if stem else o['h_out']
    bn = next(w for w in TILE_WIDTHS if cout % w == 0)
    tiles = -(-batch * (h + 2) ** 2 // BM) * (cout // bn)
    px = float(batch) * h * h
    if stem:
        nbytes = batch * 3.0 * o['img'] ** 2 * 4 + px * 64 * esz
    else:
        nbytes = (px * cin * esz * (4 if o['stride'] == 2 and k == 3 else 1) + float(cout) * cin * k * k * esz
                  + px * cout * (4 if o['out_mode'] == 1 else esz) + (px * cout * esz if o['res'] else 0))
    flop = o['gflop'] * 1e9
    s = o['ms'] * 1e-3
    tf, gbs = flop / s / 1e12, nbytes / s / 1e9
    bound = 'tensor' if flop / (TFLOPS * 1e12) >= nbytes / (HBM_GBS * 1e9) else 'hbm'
    return {'op': o['op'], 'layer': 'stem' if stem else f'{k}x{k} s{o["stride"]} {cin}->{cout} @{h}', 'cin': cin, 'cout': cout, 'k': k,
            'stride': o['stride'], 'h_out': h, 'residual': bool(o.get('res', 0)), 'out_mode': o.get('out_mode', 0), 'BN': bn,
            'tiles': tiles, 'tiles_per_cta': tiles / min(tiles, sms), 'ms': o['ms'], 'flop': flop, 'bytes': nbytes, 'tflops': tf,
            'gbs': gbs, 'bound': bound, 'frac_of_bound': (tf / TFLOPS) if bound == 'tensor' else (gbs / HBM_GBS)}


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
    assert torch.cuda.is_available(), 'bench_conv.py needs a GPU'
    info = card()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ops = profile_rows(args.arch, args.size, args.batch, args.precision, args.forwards, True)
    launches = []
    for o in ops:
        if o['tc'] and o['kind'] in (OP_STEM, OP_CONV):
            o['img'] = args.size
            launches.append(launch_row(o, args.batch, sms, 2))
    print(json.dumps(dict(info, arch=args.arch, size=args.size, batch=args.batch, precision=args.precision, forwards=args.forwards)))
    print(f'{"op":>4} {"layer":28} {"res":>3} {"out":>3} {"BN":>3} {"tiles":>6} {"/CTA":>6} {"ms":>8} {"GFLOP":>8} {"MB":>7} '
          f'{"TFLOP/s":>7} {"GB/s":>6} {"bound":>6} {"%":>5}')
    for r in launches:
        print(f'{r["op"]:4d} {r["layer"]:28} {"yes" if r["residual"] else "":>3} {r["out_mode"]:3d} {r["BN"]:3d} {r["tiles"]:6d} '
              f'{r["tiles_per_cta"]:6.1f} {r["ms"]:8.4f} {r["flop"] / 1e9:8.1f} {r["bytes"] / 1e6:7.1f} {r["tflops"]:7.1f} {r["gbs"]:6.0f} '
              f'{r["bound"]:>6} {100 * r["frac_of_bound"]:4.1f}%')
    conv = [r for r in launches if r['layer'] != 'stem']
    summary = {'launches': len(conv), 'conv_ms': sum(r['ms'] for r in conv), 'stem_ms': sum(r['ms'] for r in launches if r['layer'] == 'stem'),
               'conv_tflops': sum(r['flop'] for r in conv) / (sum(r['ms'] for r in conv) * 1e-3) / 1e12,
               'conv_gbs': sum(r['bytes'] for r in conv) / (sum(r['ms'] for r in conv) * 1e-3) / 1e9}
    print(json.dumps(summary))
    if args.json:
        with open(args.json, 'w') as fh:
            config = {k: v for k, v in vars(args).items() if k != 'json'}          # the workload, not where the result went
            json.dump(dict(info, config=config, sms=sms, launches=launches, summary=summary), fh, indent=1)


if __name__ == '__main__':
    main()
