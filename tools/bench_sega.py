#!/usr/bin/env python
"""Cost of semantic guidance on the lock-step loop: the same pipeline call with no, one and two editing prompts.

    python tools/bench_sega.py [--runs 3] [--B 4] [--steps 50]

Workload (config 2): SD v1-4 topology with synthetic weights (specs.sd_unet_config(768), KL-f8 VAE), 512^2, batch B,
CycleDiffusionPipeline at strength 0.8 -- VAE encode, a DPM-Encoder under the source prompt at scale 1 and a CFG 7.5 decode under
the target prompt in lock-step (40 of the 50 steps), VAE decode.  The conditioning is a fixed random [B, 77, 768] context.  Three
arms: no concepts (12 U-Net rows per step at B = 4), one editing prompt (16 rows) and two (20 rows), SEGA's defaults otherwise.  The
arms are alternated run by run after one warm-up call each; median and min-max of --runs runs, as ms per step (the whole call's host
time between device synchronisations over the loop's steps, VAE included) and images/s.  Then the engine's event profiler times a
4-step loop in each concept arm and reports the threshold stage's kernel time per step (tag 'other': the loop's only launches
there) and the launch count per step.  Prints one JSON line per arm, one for the profile, and a final one with the card's name,
power limit and maximum SM clock.
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
from cycle_diffusion_b200.schedule import DDIMSchedule  # noqa: E402
from cycle_diffusion_b200.semantic import SemanticGuidance  # noqa: E402
from cycle_diffusion_b200.wrappers import SDStochasticTextWrapper  # noqa: E402

ARMS = {'no-concepts': None, 'one-concept': ['e1'], 'two-concepts': ['e1', 'e2']}
L = 77


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
    ctx = torch.randn(max(a.B, 2), L, 768, generator=torch.Generator().manual_seed(0))
    cond = lambda texts: ctx[:len(texts)].to(eng.device)
    w = SDStochasticTextWrapper('synthetic', custom_steps=a.steps, eta=0.1, white_box_steps=a.steps + 1, skip_steps=[0],
                                encoder_unconditional_guidance_scales=[1.0], decoder_unconditional_guidance_scales=[7.5], n_trials=1,
                                engine=eng, state_dict='synthetic', cond_stage=cond)
    R = w.resolution
    pipe = CycleDiffusionPipeline(w.generator)
    image = torch.rand(a.B, 3, R, R, generator=torch.Generator().manual_seed(1)).to(eng.device)
    n_loop = int(a.steps * 0.8)

    def run(arm):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pipe(['t'] * a.B, ['s'] * a.B, image, strength=0.8, num_inference_steps=a.steps, guidance_scale=7.5, source_guidance_scale=1.0,
             eta=0.1, generator=torch.Generator().manual_seed(2), editing_prompt=ARMS[arm])
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for arm in ARMS:
        run(arm)
    times = {arm: [] for arm in ARMS}
    for _ in range(a.runs):
        for arm in ARMS:
            times[arm].append(run(arm))
    for arm, concepts in ARMS.items():
        ts = sorted(times[arm])
        ms = [1e3 * t / n_loop for t in ts]
        print(json.dumps(dict(arm=arm, B=a.B, rows=a.B * (3 + len(concepts or [])), resolution=R, steps=f'{n_loop}+{n_loop} lock-step',
                              cfg=7.5, ms_per_step_median=round(statistics.median(ms), 2), ms_per_step_min=round(ms[0], 2),
                              ms_per_step_max=round(ms[-1], 2), images_per_s=round(a.B / statistics.median(ts), 4),
                              images_per_s_min=round(a.B / ts[-1], 4), images_per_s_max=round(a.B / ts[0], 4))))
    # a 4-step loop per concept arm under the event profiler: the threshold stage's time and the launches per step
    g = w.generator
    n_prof = 4
    sched = DDIMSchedule(a.steps, 0.1, a.steps - n_prof, g.alphas_cumprod)
    h = R // 8
    gen = torch.Generator().manual_seed(3)
    x0 = torch.randn(a.B, 4, h, h, generator=gen).to(eng.device)
    noise = torch.randn(n_prof + 1, a.B, 4, h, h, generator=gen)
    uc = torch.zeros(a.B, L, 768, device=eng.device)
    c = ctx[:a.B].to(eng.device)
    prof = {}
    for arm, m in (('no-concepts', 0), ('one-concept', 1), ('two-concepts', 2)):
        sg = SemanticGuidance.for_concepts(m) if m else None
        c_edit = ctx[:m].to(eng.device) if m else None
        for enable in (False, True):                  # a warm-up call, then the profiled one
            eng.profile(enable)
            n0 = eng.launches
            g.unet.cycle_lockstep(x0, c, c.flip(0), uc, 1.0, 7.5, sched, noise, semantic=sg, c_edit=c_edit)
        torch.cuda.synchronize()
        launches = eng.launches - n0
        rec = eng.profile_read()
        eng.profile(False)
        th = rec.get('other', dict(ms=0.0, launches=0, bytes=0.0))
        prof[arm] = dict(threshold_ms_per_step=round(th['ms'] / n_prof, 4), threshold_launches_per_step=th['launches'] / n_prof,
                         threshold_MB_per_step=round(th['bytes'] / n_prof / 1e6, 3), launches_per_step=launches / n_prof)
    print(json.dumps(dict(profile=f'{n_prof}-step loop, threshold stage (event profiler) and launches', **prof)))
    print(json.dumps(dict(card=card(), runs=a.runs)))


if __name__ == '__main__':
    main()
