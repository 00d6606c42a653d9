#!/usr/bin/env python
"""Speed of the SD 2.x paths: SD 2-base at 512^2 (eps-prediction) and SD 2-v at 768^2 (v-prediction), each in the "full" and
"autocast" precisions.

    python tools/bench_sd2.py [--runs 3] [--B 4] [--steps 50]

Workload per configuration: synthetic SD 2 U-Net (specs.sd2_unet_config) and KL-f8 VAE, batch B, CycleDiffusionPipeline with
strength 1 -- VAE encode, a 50-step DPM-Encoder under the source prompt at scale 1 and a 50-step CFG 7.5 decode under the target
prompt in lock-step (one U-Net call per step on [source | target uncond | target cond] = 3B rows), VAE decode.  The conditioning
is a fixed random [B, 77, 1024] context (the text tower runs once per call and is not what is measured).  The four arms are
alternated run by run; median and min-max of --runs runs each.  Then, per arm: ms per U-Net call at B and 2B rows, the per-family
in-engine profile (CUDA events) of one 2B call, and the attention path each transformer level takes.  Prints one JSON line per arm
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

from cycle_diffusion_b200 import specs  # noqa: E402
from cycle_diffusion_b200.engine import Engine  # noqa: E402
from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline  # noqa: E402
from cycle_diffusion_b200.wrappers import SD2StochasticTextWrapper  # noqa: E402

ARMS = [('sd2-base-512', 'eps', 'full'), ('sd2-base-512', 'eps', 'autocast'), ('sd2-v-768', 'v', 'full'), ('sd2-v-768', 'v', 'autocast')]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def attention_paths(cfg, latent, mode):
    """The self-attention path of each transformer level, by the dispatch rule of csrc/nets.cu spatial_transformer: the fused
    fp16-split (mode 1) / one-term (mode 5) kernel when HW % 128 == 0 and d_head is one it covers, else the unfused path."""
    out = {}
    for lvl, m in enumerate(cfg['channel_mult']):
        ds = 2 ** lvl
        if ds not in cfg['attention_resolutions']:
            continue
        hw = (latent // ds) ** 2
        d = cfg['num_head_channels']
        fused = hw % 128 == 0 and d in (16, 32, 40, 64, 80)
        out[f'{latent // ds}x{latent // ds} C={m * cfg["model_channels"]} heads={m * cfg["model_channels"] // d}'] = \
            ('fused ' + ('one-term' if mode == 5 else 'fp16-split')) if fused else 'unfused'
    mid = latent // 2 ** (len(cfg['channel_mult']) - 1)
    out[f'mid {mid}x{mid}'] = 'fused' if (mid * mid) % 128 == 0 else 'unfused'
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--B', type=int, default=4)
    ap.add_argument('--steps', type=int, default=50)
    a = ap.parse_args()
    eng = Engine(0)
    ctx = torch.randn(a.B, 77, 1024, generator=torch.Generator().manual_seed(0))
    cond = lambda texts: ctx[:len(texts)].to(eng.device)
    wrappers, images = {}, {}
    for name, pred, _ in ARMS:
        if name in wrappers:
            continue
        w = SD2StochasticTextWrapper('synthetic', custom_steps=a.steps, eta=0.1, white_box_steps=a.steps + 1, skip_steps=[0],
                                     encoder_unconditional_guidance_scales=[1.0], decoder_unconditional_guidance_scales=[7.5],
                                     n_trials=1, engine=eng, state_dict='synthetic', cond_stage=cond, parameterization=pred)
        wrappers[name] = w
        images[name] = torch.rand(a.B, 3, w.resolution, w.resolution, generator=torch.Generator().manual_seed(1))

    def run(name, precision):
        w = wrappers[name]
        pipe = CycleDiffusionPipeline(w.generator, precision=precision)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pipe(['t'] * a.B, ['s'] * a.B, images[name], strength=1.0, num_inference_steps=a.steps, guidance_scale=7.5,
             source_guidance_scale=1.0, eta=0.1, generator=torch.Generator().manual_seed(2))
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for name, _, prec in ARMS:                                # warm-up: arena growth, first-call planning
        run(name, prec)
    times = {arm: [] for arm in ARMS}
    for _ in range(a.runs):
        for arm in ARMS:
            times[arm].append(run(arm[0], arm[2]))
    info = card()
    for arm in ARMS:
        name, pred, prec = arm
        w = wrappers[name]
        unet, lat = w.generator.unet, w.resolution // 8
        mode = 5 if prec == 'autocast' else 1
        per_call = {}
        with eng.precision(prec):
            for rows in (a.B, 2 * a.B):
                x = torch.randn(rows, 4, lat, lat, device=eng.device)
                t = torch.full((rows,), 501.0, device=eng.device)
                c = torch.randn(rows, 77, 1024, device=eng.device)
                unet(x, t, c)
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                ev[0].record()
                for _ in range(5):
                    unet(x, t, c)
                ev[1].record()
                torch.cuda.synchronize()
                per_call[f'B{rows}'] = round(ev[0].elapsed_time(ev[1]) / 5, 2)
            eng.profile(True)
            unet(x, t, c)
            fam = {k: round(v['ms'], 3) for k, v in eng.profile_read().items()}
            eng.profile(False)
        ts = sorted(times[arm])
        print(json.dumps(dict(config=name, prediction=pred, precision=prec, B=a.B, steps=f'{a.steps}+{a.steps} lock-step', cfg=7.5,
                              images_per_s=round(a.B / statistics.median(ts), 3), s_median=round(statistics.median(ts), 3),
                              s_min=round(ts[0], 3), s_max=round(ts[-1], 3), unet_ms=per_call, families_ms_2B=fam,
                              attention=attention_paths(specs.sd2_unet_config(), lat, mode))))
    print(json.dumps(dict(card=info, runs=a.runs)))


if __name__ == '__main__':
    main()
