#!/usr/bin/env python
"""Cost of Plug-and-Play injection on the lock-step loop: the same pipeline call without and with PnP.

    python tools/bench_pnp.py [--runs 3] [--B 4] [--steps 50]

Workload (config 2): SD v1-4 topology with synthetic weights (specs.sd_unet_config(768), KL-f8 VAE), 512^2, batch B,
CycleDiffusionPipeline at strength 0.8 -- VAE encode, a DPM-Encoder under the source prompt at scale 1 and a CFG 7.5 decode under
the target prompt in lock-step (40 of the 50 steps, 12 U-Net rows per step at B = 4), VAE decode.  The conditioning is a fixed
random [B, 77, 768] context.  Two arms: no control, and cross_attention_kwargs={'edit_type': 'pnp'} (PnP's defaults: output block
4's ResBlock features for 80 % of the steps, the self-attention queries and keys of layers 8-15 for 50 %).  The arms are
alternated run by run after one warm-up call each; median and min-max of --runs runs, as ms per step (the whole call's host time
between device synchronisations over the loop's steps, VAE included) and images/s.  Then the engine's event profiler times one
12-row U-Net call (a 1-step loop at B = 4; in the PnP arm every output block's ResBlock and every self-attention layer controlled)
in each arm and reports the GroupNorm kernels' time (tag groupnorm), the fused attention kernels' time (tag batched_tc) and the
call's launch count over all tags.  Prints one JSON line per arm, one for the profile, and a final one with the card's name, power
limit and maximum SM clock.
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

from cycle_diffusion_b200.attn_control import PnPControl  # noqa: E402
from cycle_diffusion_b200.engine import Engine  # noqa: E402
from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline  # noqa: E402
from cycle_diffusion_b200.schedule import DDIMSchedule  # noqa: E402
from cycle_diffusion_b200.wrappers import SDStochasticTextWrapper  # noqa: E402

ARMS = ['no-control', 'pnp']
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
    ctx = torch.randn(a.B, L, 768, generator=torch.Generator().manual_seed(0))
    cond = lambda texts: ctx[:len(texts)].to(eng.device)
    w = SDStochasticTextWrapper('synthetic', custom_steps=a.steps, eta=0.1, white_box_steps=a.steps + 1, skip_steps=[0],
                                encoder_unconditional_guidance_scales=[1.0], decoder_unconditional_guidance_scales=[7.5], n_trials=1,
                                engine=eng, state_dict='synthetic', cond_stage=cond)
    R = w.resolution
    pipe = CycleDiffusionPipeline(w.generator)
    image = torch.rand(a.B, 3, R, R, generator=torch.Generator().manual_seed(1)).to(eng.device)
    kwargs = {'no-control': None, 'pnp': {'edit_type': 'pnp'}}
    n_loop = int(a.steps * 0.8)

    def run(arm):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pipe(['t'] * a.B, ['s'] * a.B, image, strength=0.8, num_inference_steps=a.steps, guidance_scale=7.5, source_guidance_scale=1.0,
             eta=0.1, generator=torch.Generator().manual_seed(2), cross_attention_kwargs=kwargs[arm])
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
        print(json.dumps(dict(arm=arm, B=a.B, resolution=R, steps=f'{n_loop}+{n_loop} lock-step', cfg=7.5,
                              ms_per_step_median=round(statistics.median(ms), 2), ms_per_step_min=round(ms[0], 2),
                              ms_per_step_max=round(ms[-1], 2), images_per_s=round(a.B / statistics.median(ts), 4),
                              images_per_s_min=round(a.B / ts[-1], 4), images_per_s_max=round(a.B / ts[0], 4))))
    # one 12-row U-Net call: a 1-step loop, every output block's ResBlock and every self-attention layer controlled on its only step
    g = w.generator
    sched = DDIMSchedule(a.steps, 0.1, a.steps - 1, g.alphas_cumprod)
    h = R // 8
    gen = torch.Generator().manual_seed(3)
    x0 = torch.randn(a.B, 4, h, h, generator=gen).to(eng.device)
    noise = torch.randn(2, a.B, 4, h, h, generator=gen)
    uc = torch.zeros(a.B, L, 768, device=eng.device)
    c = ctx.to(eng.device)
    n_out = len(g.unet.cfg['channel_mult']) * (g.unet.cfg['num_res_blocks'] + 1)
    prof = {}
    for arm, ctl in (('no-control', None), ('pnp', PnPControl(1.0, 1.0, tuple(range(n_out)), 0))):
        for enable in (False, True):                  # a warm-up call, then the profiled one
            eng.profile(enable)
            g.unet.cycle_lockstep(x0, c, c.flip(0), uc, 1.0, 7.5, sched, noise, attn_control=ctl)
        rec = eng.profile_read()
        eng.profile(False)
        prof[arm] = {k: dict(ms=round(v['ms'], 3), launches=v['launches']) for k, v in rec.items() if k in ('groupnorm', 'batched_tc')}
        prof[arm]['all_launches'] = sum(v['launches'] for v in rec.values())
    print(json.dumps(dict(profile='one 12-row U-Net call (1-step loop), GroupNorm and fused attention kernels', **prof)))
    print(json.dumps(dict(card=card(), runs=a.runs)))


if __name__ == '__main__':
    main()
