#!/usr/bin/env python
"""Cost of generating the edit mask from the prompts (DiffEdit) in front of the masked lock-step cycle.

    python tools/bench_edit_mask.py [--runs 3] [--B 4] [--steps 50]

Workload (config 2): SD v1-4 topology with synthetic weights (specs.sd_unet_config(768), KL-f8 VAE), 512^2, batch B,
CycleDiffusionPipeline at strength 0.8 and 50 steps (40 lock-step steps of 3B U-Net rows), CFG 7.5, VAE encode and decode.  Each
prompt maps to a fixed random [77, 768] context of its own, so source and target conditionings differ.  Three arms: no mask, a
given box mask (the middle half of the columns, full height), and mask_image='auto' (generate_mask with its defaults: 10 maps,
strength 0.5, so 2 x 10 x B U-Net sample-forwards at t = 481 in calls of min(48, max(12, 3B)) rows, plus one more VAE encode).
generate_mask is also timed alone.  Arms are alternated run by run after one warm-up call each; median and min-max of --runs runs
of the whole call's host time between device synchronisations.  Prints one JSON line per arm and a final JSON line with the
card's name, power limit and maximum SM clock, read in the same process.
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

ARMS = ['no-mask', 'box-mask', 'auto-mask', 'generate_mask-alone']


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
    ctxs = {}

    def cond(texts):
        for t in texts:
            if t not in ctxs:
                ctxs[t] = torch.randn(77, 768, generator=torch.Generator().manual_seed(len(ctxs)))
        return torch.stack([ctxs[t] for t in texts]).to(eng.device)

    w = SDStochasticTextWrapper('synthetic', custom_steps=a.steps, eta=0.1, white_box_steps=a.steps + 1, skip_steps=[0],
                                encoder_unconditional_guidance_scales=[1.0], decoder_unconditional_guidance_scales=[7.5], n_trials=1,
                                engine=eng, state_dict='synthetic', cond_stage=cond)
    R = w.resolution
    pipe = CycleDiffusionPipeline(w.generator)
    image = torch.rand(a.B, 3, R, R, generator=torch.Generator().manual_seed(1)).to(eng.device)
    box = torch.zeros(1, 1, R, R, device=eng.device)
    box[..., :, R // 4: 3 * R // 4] = 1.0
    src, tgt = ['a cat'] * a.B, ['a dog'] * a.B
    coverage = []

    def run(arm):
        gen = torch.Generator().manual_seed(2)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if arm == 'generate_mask-alone':
            m = pipe.generate_mask(image, src, tgt, num_inference_steps=a.steps, generator=gen)
        else:
            mask = {'no-mask': None, 'box-mask': box, 'auto-mask': 'auto'}[arm]
            pipe(tgt, src, image, strength=0.8, num_inference_steps=a.steps, guidance_scale=7.5, source_guidance_scale=1.0, eta=0.1,
                 generator=gen, mask_image=mask)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if arm == 'generate_mask-alone':
            coverage.append(float(m.mean()))
        return dt

    for arm in ARMS:
        run(arm)
    times = {arm: [] for arm in ARMS}
    for _ in range(a.runs):
        for arm in ARMS:
            times[arm].append(run(arm))
    info = card()
    base = statistics.median(times['no-mask'])
    for arm in ARMS:
        ts = sorted(times[arm])
        med = statistics.median(ts)
        print(json.dumps(dict(arm=arm, B=a.B, resolution=R, steps=a.steps, strength=0.8, cfg=7.5, s_median=round(med, 3),
                              s_min=round(ts[0], 3), s_max=round(ts[-1], 3), images_per_s=round(a.B / med, 4),
                              vs_no_mask=round(med / base, 3))))
    print(json.dumps(dict(card=info, runs=a.runs, auto_mask_coverage=round(coverage[-1], 4))))


if __name__ == '__main__':
    main()
