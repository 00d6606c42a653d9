#!/usr/bin/env python
"""Cost of mask-guided local editing on the lock-step loop: the same pipeline call with and without a mask.

    python tools/bench_masked.py [--runs 3] [--B 4] [--steps 50]

Workload (config 2): SD v1-4 topology with synthetic weights (specs.sd_unet_config(768), KL-f8 VAE), 512^2, batch B,
CycleDiffusionPipeline with strength 1 -- VAE encode, a 50-step DPM-Encoder under the source prompt at scale 1 and a 50-step
CFG 7.5 decode under the target prompt in lock-step, VAE decode.  The conditioning is a fixed random [B, 77, 768] context.  Two arms:
no mask, and a centred box covering half the image (the middle half of the columns, full height).  The masked arm adds one mask
pooling launch per call and, per step, one read of the [B, 1, 64, 64] latent mask (16 KiB per image) inside the step kernel.
The arms are alternated run by run after one warm-up call each; median and min-max of --runs runs, as ms per step (the whole
call's host time between device synchronisations over --steps, VAE included) and images/s.  Prints one JSON line per arm
and a final JSON line with the card's name, power limit and maximum SM clock.
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

ARMS = ['no-mask', 'half-box-mask']


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--B', type=int, default=4)
    ap.add_argument('--steps', type=int, default=50)
    a = ap.parse_args()
    eng = Engine(0)
    ctx = torch.randn(a.B, 77, 768, generator=torch.Generator().manual_seed(0))
    cond = lambda texts: ctx[:len(texts)].to(eng.device)
    w = SDStochasticTextWrapper('synthetic', custom_steps=a.steps, eta=0.1, white_box_steps=a.steps + 1, skip_steps=[0],
                                encoder_unconditional_guidance_scales=[1.0], decoder_unconditional_guidance_scales=[7.5], n_trials=1,
                                engine=eng, state_dict='synthetic', cond_stage=cond)
    R = w.resolution
    pipe = CycleDiffusionPipeline(w.generator)
    image = torch.rand(a.B, 3, R, R, generator=torch.Generator().manual_seed(1)).to(eng.device)
    box = torch.zeros(1, 1, R, R, device=eng.device)
    box[..., :, R // 4: 3 * R // 4] = 1.0
    masks = {'no-mask': None, 'half-box-mask': box}

    def run(arm):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pipe(['t'] * a.B, ['s'] * a.B, image, strength=1.0, num_inference_steps=a.steps, guidance_scale=7.5, source_guidance_scale=1.0,
             eta=0.1, generator=torch.Generator().manual_seed(2), mask_image=masks[arm])
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for arm in ARMS:
        run(arm)
    times = {arm: [] for arm in ARMS}
    for _ in range(a.runs):
        for arm in ARMS:
            times[arm].append(run(arm))
    info = card()
    for arm in ARMS:
        ts = sorted(times[arm])
        ms = [1e3 * t / a.steps for t in ts]
        print(json.dumps(dict(arm=arm, B=a.B, resolution=R, steps=f'{a.steps}+{a.steps} lock-step', cfg=7.5,
                              ms_per_step_median=round(statistics.median(ms), 2), ms_per_step_min=round(ms[0], 2),
                              ms_per_step_max=round(ms[-1], 2), images_per_s=round(a.B / statistics.median(ts), 4),
                              images_per_s_min=round(a.B / ts[-1], 4), images_per_s_max=round(a.B / ts[0], 4))))
    print(json.dumps(dict(card=info, runs=a.runs)))


if __name__ == '__main__':
    main()
