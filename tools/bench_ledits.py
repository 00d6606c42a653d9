#!/usr/bin/env python
"""Cost of LEDITS++'s implicit masks on the semantic-guidance loop: the same pipeline call with SEGA's per-channel rule, the
cross-attention mask, and the mask intersected with the magnitude mask.

    python tools/bench_ledits.py [--runs 3] [--B 4] [--steps 50]

Workload (config 2): SD v1-4 topology with synthetic weights (specs.sd_unet_config(768), KL-f8 VAE), 512^2, batch B,
CycleDiffusionPipeline at strength 0.8 (40 lock-step steps of 50), CFG 7.5, VAE encode and decode included, a fixed random
[B, 77, 768] context.  Four arms: SEGA with one concept, plus use_cross_attn_mask, plus use_intersect_mask, and intersect with two
concepts; each concept counts 2 tokens.  The arms alternate run by run after one warm-up call each; median and min-max of --runs
runs as ms per step (host time of the whole call over the loop's steps) and images/s.  Then the engine's event profiler times a
4-step loop per arm: the probe's kernel time per step (tag 'softmax': with fused attention the probe is the loop's only launch
there), the threshold stage's (tag 'other') and the launch count per step.  The last JSON line names the card, its power limit
and maximum SM clock.
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

# arm -> (concepts, use_cross_attn_mask, use_intersect_mask)
ARMS = {'sega-1': (1, False, False), 'attn-mask-1': (1, True, False), 'intersect-1': (1, False, True), 'intersect-2': (2, False, True)}
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
        m, cross, inter = ARMS[arm]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pipe(['t'] * a.B, ['s'] * a.B, image, strength=0.8, num_inference_steps=a.steps, guidance_scale=7.5, source_guidance_scale=1.0,
             eta=0.1, generator=torch.Generator().manual_seed(2), editing_prompt=['e1', 'e2'][:m], use_cross_attn_mask=cross,
             use_intersect_mask=inter, edit_token_counts=2)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for arm in ARMS:
        run(arm)
    times = {arm: [] for arm in ARMS}
    for _ in range(a.runs):
        for arm in ARMS:
            times[arm].append(run(arm))
    for arm, (m, cross, inter) in ARMS.items():
        ts = sorted(times[arm])
        ms = [1e3 * t / n_loop for t in ts]
        print(json.dumps(dict(arm=arm, B=a.B, rows=a.B * (3 + m), resolution=R, steps=f'{n_loop}+{n_loop} lock-step', cfg=7.5,
                              ms_per_step_median=round(statistics.median(ms), 2), ms_per_step_min=round(ms[0], 2),
                              ms_per_step_max=round(ms[-1], 2), images_per_s=round(a.B / statistics.median(ts), 4),
                              images_per_s_min=round(a.B / ts[-1], 4), images_per_s_max=round(a.B / ts[0], 4))))
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
    for arm, (m, cross, inter) in ARMS.items():
        sg = SemanticGuidance.for_concepts(m, use_cross_attn_mask=cross, use_intersect_mask=inter,
                                           edit_token_counts=2 if cross or inter else None)
        c_edit = ctx[:m].to(eng.device)
        for enable in (False, True):                  # a warm-up call, then the profiled one
            eng.profile(enable)
            n0 = eng.launches
            g.unet.cycle_lockstep(x0, c, c.flip(0), uc, 1.0, 7.5, sched, noise, semantic=sg, c_edit=c_edit)
        torch.cuda.synchronize()
        launches = eng.launches - n0
        rec = eng.profile_read()
        eng.profile(False)
        zero = dict(ms=0.0, launches=0, bytes=0.0)
        pr, th = rec.get('softmax', zero), rec.get('other', zero)
        prof[arm] = dict(probe_ms_per_step=round(pr['ms'] / n_prof, 4), probe_launches_per_step=pr['launches'] / n_prof,
                         threshold_ms_per_step=round(th['ms'] / n_prof, 4), launches_per_step=launches / n_prof)
    print(json.dumps(dict(profile=f'{n_prof}-step loop, probe and threshold stage (event profiler) and launches', **prof)))
    print(json.dumps(dict(card=card(), runs=a.runs)))


if __name__ == '__main__':
    main()
