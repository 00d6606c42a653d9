#!/usr/bin/env python
"""Cost of Prompt-to-Prompt's LocalBlend on the lock-step loop: the same replace edit with and without LocalBlend.

    python tools/bench_local_blend.py [--runs 3] [--B 4] [--steps 50]

Workload (config 2): SD v1-4 topology with synthetic weights (specs.sd_unet_config(768), KL-f8 VAE), 512^2, batch B,
CycleDiffusionPipeline at strength 0.8 (40 lock-step steps of 50, 3B U-Net rows), CFG 7.5, VAE encode and decode included, a fixed
random [B, 77, 768] context.  Two arms: edit_type 'replace' (cross 0.8, self 0.4), and the same plus LocalBlend (start_blend 0.2,
thresholds (0.3, 0.3), one blend word per prompt).  The arms alternate run by run after one warm-up call each; median and min-max
of --runs runs as ms per step (host time of the whole call over the loop's steps).  Then the engine's event profiler times a 4-step
loop per arm: the probe's kernel time per step (tag 'softmax': with fused attention the probe is the loop's only launch there), the
mask stage's (tag 'other') and the launch count per step.  The last JSON line names the card, its power limit and maximum SM clock.
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

from cycle_diffusion_b200.attn_control import AttentionControl, LocalBlend  # noqa: E402
from cycle_diffusion_b200.engine import Engine  # noqa: E402
from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline  # noqa: E402
from cycle_diffusion_b200.schedule import DDIMSchedule  # noqa: E402
from cycle_diffusion_b200.wrappers import SDStochasticTextWrapper  # noqa: E402

L = 77
ARMS = ('replace', 'replace+blend')


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
    alpha = torch.zeros(L)
    alpha[2] = 1.0
    blend = LocalBlend(alpha, alpha, start_blend=0.2)
    base = {'edit_type': 'replace', 'cross_replace_steps': 0.8, 'self_replace_steps': 0.4}

    def run(arm):
        kw = dict(base, local_blend=blend) if arm == 'replace+blend' else base
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pipe(['t'] * a.B, ['s'] * a.B, image, strength=0.8, num_inference_steps=a.steps, guidance_scale=7.5, source_guidance_scale=1.0,
             eta=0.1, generator=torch.Generator().manual_seed(2), cross_attention_kwargs=kw)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for arm in ARMS:
        run(arm)
    times = {arm: [] for arm in ARMS}
    for _ in range(a.runs):
        for arm in ARMS:
            times[arm].append(run(arm))
    for arm in ARMS:
        ts = sorted(times[arm])
        ms = [1e3 * t / n_loop for t in ts]
        print(json.dumps(dict(arm=arm, B=a.B, rows=3 * a.B, resolution=R, steps=f'{n_loop} lock-step', cfg=7.5,
                              ms_per_step_median=round(statistics.median(ms), 2), ms_per_step_min=round(ms[0], 2),
                              ms_per_step_max=round(ms[-1], 2), images_per_s=round(a.B / statistics.median(ts), 4))))
    g = w.generator
    n_prof = 4
    sched = DDIMSchedule(a.steps, 0.1, a.steps - n_prof, g.alphas_cumprod)
    h = R // 8
    gen = torch.Generator().manual_seed(3)
    x0 = torch.randn(a.B, 4, h, h, generator=gen).to(eng.device)
    noise = torch.randn(n_prof + 1, a.B, 4, h, h, generator=gen)
    uc = torch.zeros(a.B, L, 768, device=eng.device)
    c = ctx[:a.B].to(eng.device)
    ctl = AttentionControl(0.8, 0.4)
    prof = {}
    for arm in ARMS:
        lb = blend if arm == 'replace+blend' else None
        for enable in (False, True):                  # a warm-up call, then the profiled one
            eng.profile(enable)
            n0 = eng.launches
            g.unet.cycle_lockstep(x0, c, c.flip(0), uc, 1.0, 7.5, sched, noise, attn_control=ctl, local_blend=lb)
        torch.cuda.synchronize()
        launches = eng.launches - n0
        rec = eng.profile_read()
        eng.profile(False)
        zero = dict(ms=0.0, launches=0, bytes=0.0)
        pr, st = rec.get('softmax', zero), rec.get('other', zero)
        prof[arm] = dict(probe_ms_per_step=round(pr['ms'] / n_prof, 4), probe_launches_per_step=pr['launches'] / n_prof,
                         mask_stage_ms_per_step=round(st['ms'] / n_prof, 4), launches_per_step=launches / n_prof)
    print(json.dumps(dict(profile=f'{n_prof}-step loop, probe and mask stage (event profiler) and launches', **prof)))
    print(json.dumps(dict(card=card(), runs=a.runs)))


if __name__ == '__main__':
    main()
