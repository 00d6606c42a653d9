#!/usr/bin/env python
"""Per-family time of the SD v1-4 U-Net and the KL-f8 decoder at image sizes other than 512 x 512 (in-engine profiler, CUDA events).

    python tools/bench_sizes.py [--reps N] [--root DIR]

One CFG batch-8 U-Net call (B = 16) at latents 64x64, 64x96 and 96x96 (512x512, 512x768, 768x768 images) and one VAE decode of a
64x96 latent (512x768 image).  Per family: ms per call, launches per call and TFLOP/s from the shapes' operation counts.  Also printed,
computed on the CPU from the conv3x3 tile planner's rule: which share of the 128 rows of the conv3x3 tiles are real pixels at each
map size of the call.  --root imports the engine from another checkout (two versions compared in one run).
"""
import argparse
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument('--reps', type=int, default=3)
ap.add_argument('--root', default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))
import torch  # noqa: E402

from cycle_diffusion_b200 import specs  # noqa: E402
from cycle_diffusion_b200.engine import VAE, Engine, UNet  # noqa: E402


def pow2(v):
    return v > 0 and v & (v - 1) == 0


def cdiv(a, b):
    return -(-a // b)


def conv_box(W, H, B, stride=1):
    """The pixel box (bw, bh, bn) of a conv3x3 M tile, as csrc/kernels_tc.cu gemm_tc / conv_ragged_tile choose it."""
    if pow2(H) and pow2(W):
        bw = min(W, 16)
        bh = min(H, 128 // bw)
        return bw, bh, 128 // (bw * bh)
    best = None
    bw = 128
    while bw >= 1:
        bh = 128 // bw
        while bh >= 1:
            bn = 128 // (bw * bh)
            if bw * stride <= 256 and bh * stride <= 256:
                key = (cdiv(W, bw) * cdiv(H, bh) * cdiv(B, bn), bn * (bw + 2) * (bh + 2))
                if best is None or key < best[0]:
                    best = (key, (bw, bh, bn))
            bh //= 2
        bw //= 2
    return best[1]


def row_use(W, H, B, stride=1):
    bw, bh, bn = conv_box(W, H, B, stride)
    tiles = cdiv(W, bw) * cdiv(H, bh) * cdiv(B, bn)
    return (bw, bh, bn), tiles, B * H * W / (tiles * 128.0)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        lim = r.stdout.strip() or 'unknown'
    except (OSError, subprocess.SubprocessError):
        lim = 'unknown'
    return f'{name}, power limit / max SM clock: {lim}'


def report(title, eng, fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for _ in range(reps):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    print(f'\n== {title}: {ev0.elapsed_time(ev1) / reps:.3f} ms per call (unprofiled)')
    eng.profile(True)
    for _ in range(reps):
        fn()
    fam = eng.profile_read()
    eng.profile(False)
    for k, v in sorted(fam.items(), key=lambda kv: -kv[1]['ms']):
        tf = v['flops'] / (v['ms'] * 1e-3) / 1e12 if v['flops'] > 0 and v['ms'] > 0 else 0.0
        print(f'   {k:14s} {v["ms"] / reps:9.3f} ms  {v["launches"] // reps:5d} launches  {tf:7.1f} TFLOP/s')


def main():
    eng = Engine(0)
    print(f'card: {card()}')
    print(f'engine from: {os.path.abspath(args.root)}')
    cfg = specs.sd_unet_config(768)
    unet = UNet(eng, cfg, 'openai').load_state_dict(specs.synth_state_dict(specs.openai_unet_params(cfg), 1234))
    B = 16                                           # CFG batch 8: [conditional | unconditional]
    for h, w in ((64, 64), (64, 96), (96, 96)):
        print(f'\n-- latent {h}x{w}: conv3x3 tile rows that are pixels (CPU, planner rule)')
        for lvl in range(len(cfg['channel_mult'])):
            H, W = h >> lvl, w >> lvl
            box, tiles, use = row_use(W, H, B)
            print(f'   map {H:3d}x{W:<3d} box {box[0]}x{box[1]}x{box[2]:<3d} tiles {tiles:5d}  row use {use:.3f}')
        g = torch.Generator(device='cuda').manual_seed(h * 1000 + w)
        x = torch.randn(B, 4, h, w, device='cuda', generator=g)
        t = torch.full((B,), 501., device='cuda')
        ctx = torch.randn(B, 77, 768, device='cuda', generator=g)
        report(f'U-Net B{B} latent {h}x{w}', eng, lambda: unet(x, t, ctx), args.reps)
    del unet
    torch.cuda.empty_cache()
    vcfg = specs.kl_f8_config()
    vae = VAE(eng, vcfg).load_state_dict(specs.synth_state_dict(specs.kl_vae_params(vcfg), 4321))
    z = torch.randn(1, 4, 64, 96, device='cuda', generator=torch.Generator(device='cuda').manual_seed(5))
    print('\n-- VAE decode 64x96 -> 512x768: conv3x3 tile rows that are pixels (CPU, planner rule)')
    for lvl in range(len(vcfg['ch_mult'])):
        H, W = 64 << lvl, 96 << lvl
        box, tiles, use = row_use(W, H, 1)
        print(f'   map {H:3d}x{W:<3d} box {box[0]}x{box[1]}x{box[2]:<3d} tiles {tiles:5d}  row use {use:.3f}')
    try:
        report('VAE decode B1 512x768', eng, lambda: vae.decode(z), args.reps)
    except AssertionError as ex:                     # an engine without rectangular first-stage support
        print(f'\n== VAE decode B1 512x768: not supported by this engine ({ex})')


if __name__ == '__main__':
    main()
