#!/usr/bin/env python
"""Cost of the edit-friendly inversion against CycleDiffusion's: the same pipeline call under inversion='cycle' and 'dpmsolver++'.

    python tools/bench_edit_friendly.py [--runs 3] [--B 4]

Workload (config 2): SD v1-4 topology with synthetic weights (specs.sd_unet_config(768), KL-f8 VAE), 512^2, batch B,
CycleDiffusionPipeline at strength 0.8, CFG 7.5, VAE encode and decode included, a fixed random [B, 77, 768] context.  Three arms:
'cycle' at 50 steps (40 lock-step steps), 'dpmsolver++' at the same 40 loop steps, and 'dpmsolver++' at 25 steps (20 loop steps).
The arms alternate run by run after one warm-up call each; median and min-max of --runs runs as ms per loop step (host time of the
whole call over the loop's steps) and images/s, with the launch count per call.  The last JSON line names the card, its power limit
and maximum SM clock.  Whether 20 solver steps edit as well as 40 DDIM steps cannot be judged with synthetic weights.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from cycle_diffusion_b200.engine import Engine  # noqa: E402
from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline  # noqa: E402
from cycle_diffusion_b200.wrappers import SDStochasticTextWrapper  # noqa: E402

# arm -> (inversion, num_inference_steps); strength 0.8 throughout
ARMS = {'cycle-40': ('cycle', 50), 'dpmsolver++-40': ('dpmsolver++', 50), 'dpmsolver++-20': ('dpmsolver++', 25)}
L = 77


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--B', type=int, default=4)
    a = ap.parse_args()
    eng = Engine(0)
    ctx = torch.randn(max(a.B, 2), L, 768, generator=torch.Generator().manual_seed(0))
    cond = lambda texts: ctx[:len(texts)].to(eng.device)
    w = SDStochasticTextWrapper('synthetic', custom_steps=50, eta=0.1, white_box_steps=51, skip_steps=[0],
                                encoder_unconditional_guidance_scales=[1.0], decoder_unconditional_guidance_scales=[7.5], n_trials=1,
                                engine=eng, state_dict='synthetic', cond_stage=cond)
    R = w.resolution
    pipe = CycleDiffusionPipeline(w.generator)
    image = torch.rand(a.B, 3, R, R, generator=torch.Generator().manual_seed(1)).to(eng.device)
    launches = {}

    def run(arm):
        inversion, steps = ARMS[arm]
        torch.cuda.synchronize()
        n0 = eng.launches
        t0 = time.perf_counter()
        pipe(['t'] * a.B, ['s'] * a.B, image, strength=0.8, num_inference_steps=steps, guidance_scale=7.5, source_guidance_scale=1.0,
             generator=torch.Generator().manual_seed(2), inversion=inversion)
        torch.cuda.synchronize()
        launches[arm] = eng.launches - n0
        return time.perf_counter() - t0

    for arm in ARMS:
        run(arm)
    times = {arm: [] for arm in ARMS}
    for _ in range(a.runs):
        for arm in ARMS:
            times[arm].append(run(arm))
    for arm, (inversion, steps) in ARMS.items():
        n_loop = int(steps * 0.8)
        ts = sorted(times[arm])
        ms = [1e3 * t / n_loop for t in ts]
        print(json.dumps(dict(arm=arm, inversion=inversion, B=a.B, resolution=R, loop_steps=n_loop, cfg=7.5,
                              ms_per_step_median=round(statistics.median(ms), 2), ms_per_step_min=round(ms[0], 2),
                              ms_per_step_max=round(ms[-1], 2), images_per_s=round(a.B / statistics.median(ts), 4),
                              images_per_s_min=round(a.B / ts[-1], 4), images_per_s_max=round(a.B / ts[0], 4),
                              launches_per_call=launches[arm])))
    print(json.dumps(dict(card=card(), runs=a.runs)))


if __name__ == '__main__':
    main()
