#!/usr/bin/env python
"""Unpaired pixel translation (cat -> dog shape): the two-phase path against the lock-step loop on one and on two engines.

    python tools/bench_unpaired.py [--reps 3] [--steps 100] [--batches 1,8] [--full 850]

Two synthetic improved-DDPM 256^2 U-Nets (different weights), custom_steps 1000, ddim eta 0.1, es_steps --steps: the per-step work
of the reference's 850-step cat -> dog configuration.  Three arms, each one whole translation (image -> image, host draws included):
  two_phase   target(source.encode(image)): z and the noise of every step on the device;
  lock_one    source.cycle(image, target) with both nets on one engine: the two U-Net calls of a step run in order;
  lock_two    the same with the nets on two engines (what UnsupervisedTranslation builds): the calls overlap on two streams.
The arms are warmed up, then alternated --reps times, each timed by the host clock between device synchronisations.  Printed per arm:
ms per translation step (median, min-max spread), peak device memory (torch allocations plus both engines' workspaces), and whether
the output equals the two-phase output bit for bit.  Also printed: the z + noise bytes the two-phase path needs at es_steps = --full
(computed from shapes), and the wall time of one --full-step lock-step translation at batch 1 on two engines.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from cycle_diffusion_b200 import specs  # noqa: E402
from cycle_diffusion_b200.engine import Engine, UNet  # noqa: E402
from cycle_diffusion_b200.wrappers import DDPMDDIMWrapper  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--reps', type=int, default=3)
ap.add_argument('--steps', type=int, default=100)
ap.add_argument('--batches', default='1,8')
ap.add_argument('--full', type=int, default=850)
args = ap.parse_args()

R = 256


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        lim = r.stdout.strip() or 'unknown'
    except (OSError, subprocess.SubprocessError):
        lim = 'unknown'
    return f'{name}, power limit / max SM clock: {lim}'


def wrapper(net, es_steps):
    return DDPMDDIMWrapper('afhq256', 'ddim', custom_steps=1000, es_steps=es_steps, eta=0.1, unet=net, image_size=R)


def run(arm, src, tgt, img):
    torch.manual_seed(0)
    return tgt(src.encode(img)) if arm == 'two_phase' else src.cycle(img, tgt)


def main():
    assert torch.cuda.is_available(), 'needs a CUDA device'
    print(f'# {card()}', flush=True)
    cfg = specs.iddpm_config(R)
    params = specs.iddpm_unet_params(cfg)
    sd_s, sd_t = specs.synth_state_dict(params, 1234), specs.synth_state_dict(params, 4321)
    e1, e2 = Engine(0), Engine(0)
    n_src = UNet(e1, cfg, 'iddpm').load_state_dict(sd_s)
    n_tgt1 = UNet(e1, cfg, 'iddpm').load_state_dict(sd_t)
    n_tgt2 = UNet(e2, cfg, 'iddpm').load_state_dict(sd_t)
    arms = {'two_phase': n_tgt2, 'lock_one': n_tgt1, 'lock_two': n_tgt2}
    for B in [int(b) for b in args.batches.split(',')]:
        img = torch.rand(B, 3, R, R, generator=torch.Generator().manual_seed(1))
        src = wrapper(n_src, args.steps)
        tgts = {a: wrapper(n, args.steps) for a, n in arms.items()}
        outs = {}
        for a in arms:                                           # warm-up (module loads, arena sizing, GEMM plans)
            outs[a] = run(a, src, tgts[a], img).cpu()
        times = {a: [] for a in arms}
        peak = {}
        for _ in range(args.reps):
            for a in arms:
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                out = run(a, src, tgts[a], img)
                torch.cuda.synchronize()
                times[a].append((time.perf_counter() - t0) * 1e3 / args.steps)
                peak[a] = max(peak.get(a, 0), torch.cuda.max_memory_allocated() - base + e1.workspace_bytes + e2.workspace_bytes)
                del out
        for a in arms:
            ts = times[a]
            print(json.dumps(dict(batch=B, arm=a, es_steps=args.steps, ms_per_step_median=round(statistics.median(ts), 3),
                                  ms_per_step_min=round(min(ts), 3), ms_per_step_max=round(max(ts), 3),
                                  peak_device_gb=round(peak[a] / 1e9, 3),
                                  equals_two_phase=bool(torch.equal(outs[a], outs['two_phase'])))), flush=True)
        zn = 2 * args.full * B * 3 * R * R * 4
        print(json.dumps(dict(batch=B, two_phase_z_plus_noise_gb_at_es_steps=args.full, computed_gb=round(zn / 1e9, 3))), flush=True)
        del img, src, tgts, outs
    img = torch.rand(1, 3, R, R, generator=torch.Generator().manual_seed(1))
    src, tgt = wrapper(n_src, args.full), wrapper(n_tgt2, args.full)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = run('lock_two', src, tgt, img)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    # torch allocations only: the engines' workspaces still have the size the largest batch above gave them
    print(json.dumps(dict(batch=1, arm='lock_two', es_steps=args.full, wall_s=round(wall, 2), ms_per_step=round(wall * 1e3 / args.full, 3),
                          peak_torch_gb=round((torch.cuda.max_memory_allocated() - base) / 1e9, 3),
                          finite=bool(torch.isfinite(out).all()))), flush=True)


if __name__ == '__main__':
    main()
