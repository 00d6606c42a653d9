#!/usr/bin/env python
"""Speed and pixel agreement of the three tensor-core precisions on the headline workload (bench.py --config 2).

    python tools/bench_precision.py [--runs N] [--B B] [--steps S]

Workload: SD v1-4 topology with synthetic weights, 512 x 512 images, batch 4, 50-step DPM-Encoder + 50-step CFG decode in
lock-step (one U-Net call per step on [source | target uncond | target cond]), VAE encode and decode included -- bench.py's
resident cycle.  Arms: mma mode 1 (fp32-faithful fp16 split, the default), 4 (single-term fp16 weight GEMMs / convs, three-term
attention) and 5 ("autocast": as 4 with single-term fused attention), alternated run by run so that drift of the shared host hits
every arm alike; median and min-max of --runs runs each.  Then, per mode, the per-family in-engine profile (CUDA events) of one
CFG batch-8 U-Net call, and max |delta pixel| of modes 4 and 5 against mode 1 on the same seeds.  Prints one JSON object with
the card's name, power limit and maximum SM clock, read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from bench import CONFIGS, ETA, encode_noise, synthetic_inputs, time_call  # noqa: E402
from cycle_diffusion_b200 import specs  # noqa: E402
from cycle_diffusion_b200.engine import VAE, Engine, UNet  # noqa: E402
from cycle_diffusion_b200.schedule import DDIMSchedule  # noqa: E402

MODES = (1, 4, 5)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--B', type=int, default=CONFIGS[2]['B'])
    ap.add_argument('--steps', type=int, default=CONFIGS[2]['steps'])
    args = ap.parse_args()
    cfg = CONFIGS[2]
    B, S, LAT = args.B, args.steps, cfg['lat']
    eng = Engine(0)
    ucfg, vcfg = specs.sd_unet_config(cfg['ctx']), specs.kl_f8_config()
    unet = UNet(eng, ucfg, 'openai').load_state_dict(specs.synth_state_dict(specs.openai_unet_params(ucfg), 1234))
    vae = VAE(eng, vcfg).load_state_dict(specs.synth_state_dict(specs.kl_vae_params(vcfg), 1235))
    image, c_src, c_tgt, uc = synthetic_inputs(cfg, B, seed=0)
    gen = torch.Generator().manual_seed(7)
    sched = DDIMSchedule(S, ETA, 0)
    post = torch.randn(B, 4, LAT, LAT, generator=gen)
    noise = encode_noise(sched, sched.refine_steps, (B, 4, LAT, LAT), gen)
    d = eng.device
    image, c_src, c_tgt, uc, post, noise = (t.to(d) for t in (image, c_src, c_tgt, uc, post, noise))

    def cycle():
        x0 = eng.vae_posterior(vae.encode_moments(eng.shift_scale(image, -0.5, 2.0)), post, 0.18215)
        s = unet.cycle_lockstep(x0, c_src, c_tgt, uc, cfg['enc_scale'], cfg['dec_scale'], sched, noise)
        return eng.shift_scale(vae.decode(eng.affine(s, 1. / 0.18215, 0.0)), 1.0, 0.5)

    ms = {m: [] for m in MODES}
    imgs = {}
    for m in MODES:                                   # warm every mode's shapes (arena sizing, tensor maps, first launches)
        eng.set_mma_mode(m)
        imgs[m] = cycle().cpu()
    for _ in range(args.runs):
        for m in MODES:
            eng.set_mma_mode(m)
            ms[m].append(time_call(cycle, reps=1, warm=0))

    t1 = torch.full((2 * B,), 501., device=d)
    x2 = torch.randn(2 * B, 4, LAT, LAT, device=d, generator=torch.Generator(device=d).manual_seed(3))
    ctx2 = torch.cat([uc, c_tgt])
    families, unet_ms = {}, {}
    for m in MODES:
        eng.set_mma_mode(m)
        unet_ms[m] = round(time_call(lambda: unet(x2, t1, ctx2), reps=5, warm=2), 2)
        eng.profile(True)
        unet(x2, t1, ctx2)
        fam = eng.profile_read()
        eng.profile(False)
        for v in fam.values():
            if v['flops'] and v['ms'] > 0:
                v['tflops'] = round(v['flops'] / (v['ms'] * 1e-3) / 1e12, 1)
            v['ms'] = round(v['ms'], 2)
            v.pop('bytes', None)
            v.pop('flops', None)
        families[m] = fam
    eng.set_mma_mode(1)

    out = {
        'card': card(),
        'workload': f'SD v1-4 topology (synthetic weights), {cfg["res"]}x{cfg["res"]}, batch {B}, {S}-step encode + {S}-step CFG decode '
                    f'in lock-step, VAE encode / decode included',
        'images_per_s': {m: {'median': round(B / (statistics.median(v) / 1e3), 4), 'min': round(B / (max(v) / 1e3), 4),
                             'max': round(B / (min(v) / 1e3), 4)} for m, v in ms.items()},
        'ms_per_cycle': {m: [round(x, 1) for x in v] for m, v in ms.items()},
        'unet_ms_cfg_batch%d' % (2 * B): unet_ms,
        'families_cfg_batch%d' % (2 * B): families,
        'max_abs_delta_pixel_vs_mode1': {m: float((imgs[m] - imgs[1]).abs().max()) for m in MODES if m != 1},
    }
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
