#!/usr/bin/env python
"""The published text-translation ensemble search: two-phase encode() + forward() against the lock-step cycle_ensemble().

    python tools/bench_ensemble.py --part timing [--runs N] [--trials T]
    python tools/bench_ensemble.py --part count [--trials T] [--rows 12,24,36,48,96] [--sweep-steps S]

Workload: SD v1-4 topology with synthetic weights, 512 x 512, batch 1, Directional-CLIP ViT-B/32 with synthetic weights, the
ensemble of all 16 published text configurations (custom_steps 99, white_box_steps 100, eta 0.1, encoder scales [1], decoder
scales [1, 1.5, 2, 3, 4, 5], skips [15, 20, 25, 30, 40, 50]) at --trials trials (the published 15 scale linearly).  The two arms
alternate run by run after a short warm-up of every shape; median and min-max seconds per image of --runs runs each, peak torch
allocation per arm, and agreement of the chosen candidate and image between the arms.  --part count (a separate process, so the
profiler's events stay out of the timings): one profiled run per arm counts the U-Net sample-forwards from the conv3x3 FLOPs
(over those of a one-row U-Net call) and reads the engine workspace after each arm; then the row-budget sweep times the lock-step
loop alone, per U-Net sample-forward, at each --rows budget (chains of 12 rows: source at scale 1 + six decoder chains) over
--sweep-steps steps.  Prints one JSON object with the card's name, power limit and maximum SM clock, read in the same run.
"""
import argparse
import hashlib
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
from cycle_diffusion_b200._cabi import CdxError  # noqa: E402
from cycle_diffusion_b200.clip_rank import DirectionalCLIP  # noqa: E402
from cycle_diffusion_b200.engine import Engine  # noqa: E402
from cycle_diffusion_b200.schedule import DDIMSchedule  # noqa: E402
from cycle_diffusion_b200.wrappers import SDStochasticTextWrapper  # noqa: E402

PUBLISHED = dict(custom_steps=99, white_box_steps=100, eta=0.1, encoder_unconditional_guidance_scales=[1],
                 decoder_unconditional_guidance_scales=[1, 1.5, 2, 3, 4, 5], skip_steps=[15, 20, 25, 30, 40, 50])


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def stub_tokenizer(texts):
    """Deterministic ids per prompt with the end-of-text token (the largest id) after them, as clip.tokenize lays them out."""
    out = torch.zeros(len(texts), 77, dtype=torch.long)
    for i, t in enumerate(texts):
        g = torch.Generator().manual_seed(int.from_bytes(hashlib.sha256(t.encode()).digest()[:4], 'little'))
        out[i, 0] = 49406
        out[i, 1:9] = torch.randint(1, 49000, (8,), generator=g)
        out[i, 9] = 49407
    return out


def conv_flops(eng):
    return sum(v['flops'] for k, v in eng.profile_read().items() if k.startswith('conv3x3'))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--trials', type=int, default=1)
    ap.add_argument('--rows', default='12,24,36,48,96')
    ap.add_argument('--sweep-steps', type=int, default=10)
    ap.add_argument('--part', choices=('timing', 'count'), default='timing')
    args = ap.parse_args()
    eng = Engine(0)
    vc, tc = specs.clip_b32_vision_config(), specs.clip_b32_text_config()
    csd = dict(specs.synth_state_dict(specs.clip_vision_params(vc), 31))
    csd.update(specs.synth_state_dict(specs.clip_text_params(tc) + [('text_projection.weight', (tc['proj_dim'], tc['width']), 'w')], 32))
    dclip = DirectionalCLIP(eng, csd, stub_tokenizer, vision_cfg=vc, text_cfg=tc)
    w = SDStochasticTextWrapper('sd-v1-4.ckpt', state_dict='synthetic', engine=eng, ranker=dclip, n_trials=args.trials, **PUBLISHED)
    image = torch.rand(1, 3, 512, 512, generator=torch.Generator().manual_seed(0))
    src, tgt = ['a photo of a cat'], ['a photo of a dog']
    assert w.lockstep_ensemble()

    def two_phase():
        z = w.encode(image, src)
        img_ens = [eng.shift_scale(i, 1.0, 0.5) for i in w.generate(z, tgt)]
        return dclip.rank(img_ens, image, src, tgt)[:2]

    def lockstep():
        return w.cycle_ensemble(image, src, tgt)[:2]

    arms = {'two_phase': two_phase, 'lockstep': lockstep}
    summary = {'card': card(),
               'workload': f'SD v1-4 topology (synthetic weights), 512x512, batch 1, DirectionalCLIP ViT-B/32 (synthetic), published '
                           f'ensemble at n_trials={args.trials}: {w.n_candidates()} candidates, ensemble_rows={w.ensemble_rows}'}
    if args.part == 'timing':
        skips = w.skip_steps
        w.skip_steps = [PUBLISHED['custom_steps'] - 4]          # warm-up: every shape of the timed runs, 4 steps per loop
        for fn in arms.values():
            fn()
        w.skip_steps = skips
        res, mem, out = {k: [] for k in arms}, {}, {}
        for _ in range(args.runs):
            for name, fn in arms.items():
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                torch.manual_seed(11)
                t0 = time.perf_counter()
                img, idx = fn()
                torch.cuda.synchronize()
                res[name].append(time.perf_counter() - t0)
                mem[name] = max(mem.get(name, 0), torch.cuda.max_memory_allocated())
                out[name] = (img.cpu(), idx.cpu())
        (img_t, idx_t), (img_l, idx_l) = out['two_phase'], out['lockstep']
        summary.update({
            's_per_image': {k: {'median': round(statistics.median(v), 2), 'min': round(min(v), 2), 'max': round(max(v), 2)} for k, v in res.items()},
            'peak_torch_alloc_MiB': {k: round(v / 2 ** 20, 1) for k, v in mem.items()},
            'workspace_MiB_after_both_arms': round(eng.workspace_bytes / 2 ** 20, 1),
            'same_index': bool(torch.equal(idx_t, idx_l)), 'index': {'two_phase': idx_t.tolist(), 'lockstep': idx_l.tolist()},
            'max_abs_delta_image': float((img_t - img_l).abs().max()),
        })
        print(json.dumps(summary, indent=1))
        return

    # --part count: one profiled run per arm (U-Net sample-forwards = conv3x3 FLOPs over those of a one-row U-Net call), the
    # workspace each arm needs on a fresh engine, then the row-budget sweep
    x1 = torch.randn(1, 4, 64, 64, device=eng.device)
    c1 = w.generator.get_learned_conditioning(src).to(eng.device)
    eng.profile(True)
    w.generator.unet(x1, torch.tensor([500.0]), c1)
    unit = conv_flops(eng)
    fwd, ws = {}, {}
    for name in ('lockstep', 'two_phase'):                  # the workspace only grows: the lock-step arm's is its own
        fn = arms[name]
        eng.profile(True)
        torch.manual_seed(11)
        fn()
        fwd[name] = round(conv_flops(eng) / unit, 2)
        ws[name] = round(eng.workspace_bytes / 2 ** 20, 1)
    eng.profile(False)
    plan = w.ensemble_plan(1)[0]
    summary.update({'unet_sample_forwards': fwd,
                    'planned_sample_forwards': {'two_phase': plan.two_phase_sample_forwards(), 'lockstep': plan.sample_forwards()},
                    'workspace_MiB_after': ws})
    # the lock-step loop alone: n_src source chains of 12 rows (scale-1 source + six decoder chains) per call
    sched = DDIMSchedule(PUBLISHED['custom_steps'], PUBLISHED['eta'], PUBLISHED['custom_steps'] - args.sweep_steps)
    dec = [float(s) for s in PUBLISHED['decoder_unconditional_guidance_scales']]
    sweep = {}
    for rows in [int(r) for r in args.rows.split(',')]:
        n_src = max(1, rows // 12)
        x0 = torch.randn(n_src, 4, 64, 64, device=eng.device)
        ctx = c1.expand(n_src, -1, -1).contiguous()
        noise = torch.randn(sched.refine_steps + 1, n_src, 4, 64, 64, device=eng.device)
        run = lambda: w.generator.unet.cycle_fan(x0, ctx, ctx, ctx, [1.0] * n_src, [dec] * n_src, sched, noise)
        try:
            run()
        except CdxError as err:                             # a budget the engine cannot run: recorded, not timed
            sweep[rows] = dict(rows_per_call=12 * n_src, error=str(err))
            continue
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        sweep[rows] = dict(rows_per_call=12 * n_src, ms_per_sample_forward=round(dt * 1e3 / (12 * n_src * sched.refine_steps), 3))
    summary['row_budget_sweep'] = sweep
    print(json.dumps(summary, indent=1))


if __name__ == '__main__':
    main()
