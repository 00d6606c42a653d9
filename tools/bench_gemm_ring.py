#!/usr/bin/env python
"""The tensor-core GEMM (tc_gemm_kernel) at the 12-row lock-step shapes of the headline workload: two checkouts compared in one run.

    python tools/bench_gemm_ring.py --root DIR_A --root DIR_B [--runs 3] [--reps 10]

For each checkout (--root, imported in a fresh process per run; the runs alternate A, B, A, B, ...), in mma mode 1 (fp16 split):
  * every Linear / 1x1 shape and every conv3x3 shape of the SD v1-4 U-Net (the tools/bench_ops.py lists) at batch 12 -- the
    encode chain plus the two CFG rows of each of the four decode chains in lock-step: kernel time from the in-engine CUDA-event
    profiler (dense_tc / conv3x3_tc family), ms per call and TFLOP/s (2 M N K);
  * the same shapes through Engine.op_gemm with the epilogue terms the U-Net fuses ('gemm' rows): bias and range slot, plus GroupNorm
    statistics on the convs ('-stats': without them), '+res' a residual on the 320 / 640 / 1280-wide outputs, 'geglu' on the FF1
    shapes -- the with / without difference is the epilogue's share of the kernel time;
  * one 12-row SD v1-4 U-Net call at 512x512 (synthetic weights): ms per call unprofiled, and the per-family profile in modes 1 and 5.
Printed: the card, its power limit and max SM clock; median and min-max over the runs; max |delta| between the two checkouts'
outputs on identical inputs (first run of each arm).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS = 12
# (Cin, Cout, H) and (tokens per image, K, N): the SD v1-4 U-Net's layers (tools/bench_ops.py)
CONVS = [(320, 320, 64), (640, 640, 32), (1280, 1280, 16), (1280, 1280, 8), (2560, 1280, 8), (2560, 1280, 16), (1920, 1280, 16),
         (1920, 640, 32), (1280, 640, 32), (960, 640, 32), (960, 320, 64), (640, 320, 64), (320, 640, 32), (640, 1280, 16)]
LINEARS = [(4096, 320, 320), (4096, 320, 960), (4096, 320, 2560), (4096, 1280, 320), (1024, 640, 640), (1024, 640, 5120), (1024, 2560, 640),
           (256, 1280, 1280), (256, 1280, 10240), (256, 5120, 1280), (64, 1280, 1280)]
FAMILIES = ['conv3x3_tc', 'dense_tc', 'batched_tc', 'groupnorm', 'layernorm', 'softmax', 'other']


def conv_label(cin, cout, h):
    return f'conv3x3 {cin}->{cout} @{h}^2'


def lin_label(m, k, n):
    return f'linear M{m * ROWS} K{k} N{n}'


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


def weights(specs, cfg, cache):
    import torch
    path = os.path.join(cache, 'sd1.pt')
    if os.path.exists(path):
        return torch.load(path)
    sd = specs.synth_state_dict(specs.openai_unet_params(cfg), 1234)
    torch.save(sd, path)
    return sd


def epilogue_arms(eng, x, w, b, M, N, conv, rows_per_img, g):
    """Engine.op_gemm calls carrying the epilogue terms the U-Net fuses: label suffix -> (call, output).  Every arm has the bias and
    the range slot; convs add the GroupNorm statistics (every U-Net conv3x3 tracks them), '+res' a residual at ldr = N, and the FF1
    shapes (N = 8 * K) the GEGLU epilogue."""
    import torch
    K = w[0].numel() if conv else w.shape[1]
    f = dict(M=M, N=N, K=K, A=x, C1=x.shape[-1], lda=x.shape[-1], w=w, bias=b, ldc=N, rows_per_batch=rows_per_img)
    if conv:
        h = x.shape[1]
        f.update(mode=1, Hin=h, Win=h, Hout=h, Wout=h)
    else:
        f.update(mode=0, ldb=K)
    res = torch.randn(M, N, device='cuda', generator=g)
    amax = torch.zeros(1, device='cuda')
    stats = torch.zeros(M // rows_per_img, N, 2, dtype=torch.float64, device='cuda')
    arms = {}

    def arm(name, out, **extra):
        def call():
            amax.zero_()
            if 'c_stats' in extra:
                stats.zero_()
            eng.op_gemm(**f, C=out, c_amax=amax, **extra)
        arms[name] = (call, out)

    side = dict(c_stats=stats) if conv else {}
    arm('', torch.empty(M, N, device='cuda'), **side)
    if N in (320, 640, 1280):
        arm(' +res', torch.empty(M, N, device='cuda'), residual=res, ldr=N, **side)
    if conv:
        arm(' -stats', torch.empty(M, N, device='cuda'))
    if not conv and N == 8 * K:
        f2 = dict(f, ldc=N // 2)
        out = torch.empty(M, N // 2, device='cuda')

        def geglu():
            amax.zero_()
            eng.op_gemm(**f2, C=out, c_amax=amax, geglu=1)
        arms[' geglu'] = (geglu, out)
    return arms


def op_time(eng, fn, family, reps):
    """Kernel time of one call (ms) from the engine's CUDA-event profiler; the first call warms up the shape."""
    fn()
    eng.profile(True)
    for _ in range(reps):
        fn()
    fam = eng.profile_read()
    eng.profile(False)
    return fam[family]['ms'] / reps


def worker(root, out, reps, cache, save):
    sys.path.insert(0, os.path.abspath(root))
    import torch
    from cycle_diffusion_b200 import specs
    from cycle_diffusion_b200.engine import Engine, UNet
    res, tensors = {'card': card()}, {}
    eng = Engine(0)
    eng.set_mma_mode(1)
    for cin, cout, h in CONVS:
        g = torch.Generator(device='cuda').manual_seed(cin * 7 + cout + h)
        x = torch.randn(ROWS, h, h, cin, device='cuda', generator=g)
        w = torch.randn(cout, cin, 3, 3, device='cuda', generator=g) / (9 * cin) ** 0.5
        b = torch.randn(cout, device='cuda', generator=g)
        label = conv_label(cin, cout, h)
        if save:
            tensors[label] = eng.op_conv3x3(x, w, b).cpu()
        res[label] = op_time(eng, lambda: eng.op_conv3x3(x, w, b), 'conv3x3_tc', reps)
        for suffix, (fn, y) in epilogue_arms(eng, x, w, b, ROWS * h * h, cout, True, h * h, g).items():
            res[label + ' gemm' + suffix] = op_time(eng, fn, 'conv3x3_tc', reps)
            if save:
                fn()
                tensors[label + ' gemm' + suffix] = y.cpu()
        del x, w, b
    for m, k, n in LINEARS:
        g = torch.Generator(device='cuda').manual_seed(m * 7 + k + n)
        x = torch.randn(m * ROWS, k, device='cuda', generator=g)
        w = torch.randn(n, k, device='cuda', generator=g) / k ** 0.5
        b = torch.randn(n, device='cuda', generator=g)
        label = lin_label(m, k, n)
        if save:
            tensors[label] = eng.op_linear(x, w, b).cpu()
        res[label] = op_time(eng, lambda: eng.op_linear(x, w, b), 'dense_tc', reps)
        for suffix, (fn, y) in epilogue_arms(eng, x, w, b, m * ROWS, n, False, m, g).items():
            res[label + ' gemm' + suffix] = op_time(eng, fn, 'dense_tc', reps)
            if save:
                fn()
                tensors[label + ' gemm' + suffix] = y.cpu()
        del x, w, b
    torch.cuda.empty_cache()
    cfg = specs.sd_unet_config(768)
    net = UNet(eng, cfg, 'openai').load_state_dict(weights(specs, cfg, cache))
    g = torch.Generator(device='cuda').manual_seed(12)
    x = torch.randn(ROWS, 4, 64, 64, device='cuda', generator=g)
    ctx = torch.randn(ROWS, 77, 768, device='cuda', generator=g)
    t = torch.linspace(981., 1., ROWS, device='cuda')
    for mode in (1, 5):
        eng.set_mma_mode(mode)
        y = net(x, t, ctx)
        if save:
            tensors[f'U-Net x{ROWS} mode {mode}'] = y.cpu()
        net(x, t, ctx)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(max(3, reps // 2)):
            net(x, t, ctx)
        b.record()
        torch.cuda.synchronize()
        res[f'U-Net x{ROWS} mode {mode}'] = a.elapsed_time(b) / max(3, reps // 2)
        eng.profile(True)
        for _ in range(3):
            net(x, t, ctx)
        fam = eng.profile_read()
        eng.profile(False)
        for f in FAMILIES:
            if f in fam:
                res[f'  mode {mode} {f}'] = fam[f]['ms'] / 3
                res[f'  mode {mode} {f} flops'] = fam[f]['flops'] / 3
    if save:
        torch.save(tensors, out + '.pt')
    json.dump(res, open(out + '.json', 'w'))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--root', action='append', default=[])
    ap.add_argument('--runs', type=int, default=3)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--worker', default=None)
    ap.add_argument('--cache', default=None)
    ap.add_argument('--save', type=int, default=0)
    args = ap.parse_args()
    if args.worker:
        worker(args.root[0], args.worker, args.reps, args.cache, args.save)
        return
    roots = [os.path.abspath(r) for r in (args.root or [HERE])]
    tmp = tempfile.mkdtemp(prefix='bench_gemm_ring_')
    runs = {r: [] for r in roots}
    for i in range(args.runs):
        for j, r in enumerate(roots):
            out = os.path.join(tmp, f'{j}_{i}')
            subprocess.run([sys.executable, os.path.abspath(__file__), '--root', r, '--worker', out, '--reps', str(args.reps),
                            '--cache', tmp, '--save', str(int(i == 0))], check=True)
            runs[r].append(json.load(open(out + '.json')))
    import shutil
    import torch
    outs = [torch.load(os.path.join(tmp, f'{j}_0.pt')) for j in range(len(roots))]
    print(f'card: {runs[roots[0]][0]["card"]}')
    for j, r in enumerate(roots):
        print(f'arm {j}: {r}')
    print(f'{args.runs} runs per arm, alternating; median (min-max) ms per call, kernel time (profiler) for the single ops\n')
    flops = {conv_label(ci, co, h): 2.0 * ROWS * h * h * co * 9 * ci for ci, co, h in CONVS}
    flops.update({lin_label(m, k, n): 2.0 * ROWS * m * k * n for m, k, n in LINEARS})
    labels = [k for k in runs[roots[0]][0] if k != 'card' and not k.endswith('flops')]
    hdr = ''.join(f'{"arm " + str(j):>36s}' for j in range(len(roots)))
    print(f'{"shape":48s}{hdr}   {"arm1/arm0":>9s}  max|delta|')
    for label in labels:
        cells, meds = '', []
        for r in roots:
            v = [x.get(label, float('nan')) for x in runs[r]]
            med = statistics.median(v)
            meds.append(med)
            fl = flops.get(label.split(' gemm')[0]) or runs[r][0].get(label + ' flops', 0.0)
            tf = f' {fl / (med * 1e-3) / 1e12:5.1f} TF/s' if fl else ' ' * 11
            cells += f'{med:9.3f} ({min(v):.3f}-{max(v):.3f}){tf}'
        ratio = f'{meds[1] / meds[0]:9.3f}' if len(meds) > 1 else ''
        dl = ''
        if len(outs) > 1 and label in outs[0]:
            dl = f'{float((outs[0][label].double() - outs[1][label].double()).abs().max()):.2e}'
        print(f'{label:48s}{cells}   {ratio}  {dl}')
    shutil.rmtree(tmp, ignore_errors=True)


if __name__ == '__main__':
    main()
