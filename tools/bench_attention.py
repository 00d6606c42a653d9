#!/usr/bin/env python
"""Attention at the shapes the fused kernel gained (any token count, 160-channel heads): two checkouts compared in one run.

    python tools/bench_attention.py --root DIR_A --root DIR_B [--runs 3] [--reps 20]

For each checkout (--root, imported in a fresh process per run; the runs alternate A, B, A, B, ...):
  * every moved layer shape through Engine.op_attention (mma mode 1: operand preparation + attention, as the U-Net runs it),
    ms per call and TFLOP/s (4 B heads N Nk d per call);
  * one U-Net call: SD v1 512x512 at 8 rows, SD 2-v 768x768 at 8 rows, SD v1 576x576 at 12 rows (synthetic weights);
  * the first checkout only: the engine workspace of one SD v1 960x960 call at 12 rows, on a fresh engine.
Printed: median and min-max over the runs, and max |delta| between the two checkouts' outputs on identical inputs.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (label, B, N, Nk, heads, d)
LAYERS = [
    ('SD v1 512 16x16 self', 8, 256, 256, 8, 160),
    ('SD v1 512 16x16 cross', 8, 256, 77, 8, 160),
    ('SD v1 512 mid self', 8, 64, 64, 8, 160),
    ('SD v1 512 mid cross', 8, 64, 77, 8, 160),
    ('LDM 256 mid self', 8, 16, 16, 8, 160),
    ('LDM 256 mid cross', 8, 16, 77, 8, 160),
    ('SD 2-v 768 24x24 self', 8, 576, 576, 20, 64),
    ('SD 2-v 768 24x24 cross', 8, 576, 77, 20, 64),
    ('SD 2-v 768 mid self', 8, 144, 144, 20, 64),
    ('SD v1 576 72x72 self', 12, 5184, 5184, 8, 40),
    ('SD v1 576 9x9 self', 12, 81, 81, 8, 160),
]
# (label, config, context width, rows, latent)
UNETS = [
    ('U-Net SD v1 512 x8', 'sd1', 768, 8, 64),
    ('U-Net SD 2-v 768 x8', 'sd2', 1024, 8, 96),
    ('U-Net SD v1 576 x12', 'sd1', 768, 12, 72),
]


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        lim = r.stdout.strip() or 'unknown'
    except (OSError, subprocess.SubprocessError):
        lim = 'unknown'
    return f'{name}, power limit / max SM clock: {lim}'


def timed(fn, reps):
    import torch
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def weights(specs, cfg, kind, cache):
    """The synthetic state dict of a config, generated once per run and shared by the worker processes through `cache`."""
    import torch
    path = os.path.join(cache, f'{kind}.pt')
    if os.path.exists(path):
        return torch.load(path)
    sd = specs.synth_state_dict(specs.openai_unet_params(cfg), 1234)
    torch.save(sd, path)
    return sd


def worker(root, out, reps, what, cache):
    sys.path.insert(0, os.path.abspath(root))
    import torch
    from cycle_diffusion_b200 import specs
    from cycle_diffusion_b200.engine import Engine, UNet
    res, tensors = {'card': card()}, {}
    if what == 'workspace':
        cfg = specs.sd_unet_config(768)
        eng = Engine(0)
        net = UNet(eng, cfg, 'openai').load_state_dict(weights(specs, cfg, 'sd1', cache))
        g = torch.Generator(device='cuda').manual_seed(3)
        x = torch.randn(12, 4, 120, 120, device='cuda', generator=g)
        ctx = torch.randn(12, 77, 768, device='cuda', generator=g)
        try:
            net(x, torch.full((12,), 501., device='cuda'), ctx)
            torch.cuda.synchronize()
            res['workspace'] = eng.workspace_bytes
        except Exception as ex:  # noqa: BLE001 -- reported, not raised: the older engine may not fit
            res['workspace'] = f'failed: {str(ex).splitlines()[0][:120]}'
        json.dump(res, open(out + '.json', 'w'))
        return
    eng = Engine(0)
    for label, B, N, Nk, heads, d in LAYERS:
        g = torch.Generator(device='cuda').manual_seed(N * 131 + Nk + d)
        q = torch.randn(B, N, heads * d, device='cuda', generator=g)
        k, v = (torch.randn(B, Nk, heads * d, device='cuda', generator=g) for _ in range(2))
        y = eng.op_attention(q, k, v, heads, d ** -0.5)
        tensors[label] = y.cpu()
        res[label] = timed(lambda: eng.op_attention(q, k, v, heads, d ** -0.5), reps)
    for label, kind, cdim, R, lat in UNETS:
        cfg = specs.sd_unet_config(768) if kind == 'sd1' else specs.sd2_unet_config()
        net = UNet(eng, cfg, 'openai').load_state_dict(weights(specs, cfg, kind, cache))
        g = torch.Generator(device='cuda').manual_seed(R * 100 + lat)
        x = torch.randn(R, 4, lat, lat, device='cuda', generator=g)
        ctx = torch.randn(R, 77, cdim, device='cuda', generator=g)
        t = torch.linspace(981., 1., R, device='cuda')
        tensors[label] = net(x, t, ctx).cpu()
        res[label] = timed(lambda: net(x, t, ctx), max(2, reps // 5))
        del net
        torch.cuda.empty_cache()
    torch.save(tensors, out + '.pt')
    json.dump(res, open(out + '.json', 'w'))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--root', action='append', default=[])
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--worker', default=None)
    ap.add_argument('--what', default='time')
    ap.add_argument('--cache', default=None)
    args = ap.parse_args()
    if args.worker:
        worker(args.root[0], args.worker, args.reps, args.what, args.cache)
        return
    roots = [os.path.abspath(r) for r in (args.root or [HERE])]
    tmp = tempfile.mkdtemp(prefix='bench_attention_')
    runs = {r: [] for r in roots}
    for i in range(args.runs):
        for j, r in enumerate(roots):
            out = os.path.join(tmp, f'{j}_{i}')
            subprocess.run([sys.executable, os.path.abspath(__file__), '--root', r, '--worker', out, '--reps', str(args.reps), '--cache', tmp],
                           check=True)
            runs[r].append(json.load(open(out + '.json')))
    ws = {}
    for j, r in enumerate(roots[:1]):        # the first arm only: an engine that materialises the scores needs ~80 GB there
        out = os.path.join(tmp, f'{j}_ws')
        subprocess.run([sys.executable, os.path.abspath(__file__), '--root', r, '--worker', out, '--what', 'workspace', '--cache', tmp], check=True)
        ws[r] = json.load(open(out + '.json'))['workspace']
    import shutil
    import torch
    outs = [torch.load(os.path.join(tmp, f'{j}_0.pt')) for j in range(len(roots))]
    print(f'card: {runs[roots[0]][0]["card"]}')
    for j, r in enumerate(roots):
        print(f'arm {j}: {r}')
    print(f'{args.runs} runs per arm, alternating; median (min-max) ms per call\n')
    hdr = ''.join(f'{"arm " + str(j):>34s}' for j in range(len(roots)))
    print(f'{"shape":28s}{hdr}   max|delta| arm0-arm1')
    flops = {l: 4.0 * B * heads * N * Nk * d for l, B, N, Nk, heads, d in LAYERS}
    for label in [l[0] for l in LAYERS] + [u[0] for u in UNETS]:
        cells = ''
        for r in roots:
            v = [x[label] for x in runs[r]]
            med = statistics.median(v)
            tf = f' {flops[label] / (med * 1e-3) / 1e12:5.1f} TF/s' if label in flops else ' ' * 11
            cells += f'{med:9.3f} ({min(v):.3f}-{max(v):.3f}){tf}'
        dl = f'{float((outs[0][label].double() - outs[1][label].double()).abs().max()):.2e}' if len(outs) > 1 else ''
        print(f'{label:28s}{cells}   {dl}')
    for j, r in enumerate(roots[:1]):
        w = ws[r]
        print(f'workspace SD v1 960x960 x12, arm {j}: ' + (f'{w / 1e9:.2f} GB' if isinstance(w, int) else w))
    shutil.rmtree(tmp, ignore_errors=True)


if __name__ == '__main__':
    main()
