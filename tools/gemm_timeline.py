#!/usr/bin/env python
"""Where a tensor-core GEMM work item's time goes: per-CTA %globaltimer stamps from tc_gemm_kernel, median per phase.

    python tools/gemm_timeline.py [--out DIR] [--reps 5]

Builds libcdx with -DCDX_GEMM_TIMELINE into DIR (default: a temporary directory; never the package's own libcdx.so) beside a copy
of the package's Python files, and imports that copy.  Then runs the 12-row lock-step shapes below through Engine.op_gemm with the
epilogue terms the U-Net fuses (bias and range slot; residual on the Linear layers; GroupNorm sums on the conv), in mma mode 1,
with the persistent GEMM off and on (Engine.set_persist), and prints per arm the median over CTAs and repetitions of each phase:
  launch    entry -> after griddepcontrol.wait
  fill      -> the first stage has landed
  main      -> the last stage has retired (persistent: first item's first stage to last item's last stage)
  res       -> bar_res passed (the epilogue's buffer is free, the residual has landed)
  epi       -> the TMA store issued
  drain     -> bulk_wait0 returned
plus the items per CTA, the CTA's life (entry -> drain) per item, and the kernel's span (first entry -> last drain).
"""
import argparse
import ctypes as C
import glob
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(HERE, 'cycle_diffusion_b200')
ROWS = 12
SLOTS = 8           # TL_SLOTS in kernels_tc.cu
PHASES = ['launch', 'fill', 'main', 'res', 'epi', 'drain']
# (label, kind, shape): Linear (tokens per image, K, N) with a residual; conv3x3 (Cin, Cout, H) with GroupNorm sums
SHAPES = [('Linear 49152x320x320 +res', 'lin', (4096, 320, 320)), ('Linear 12288x640x640 +res', 'lin', (1024, 640, 640)),
          ('Linear 49152x1280x320 +res', 'lin', (4096, 1280, 320)), ('conv3x3 320->320 @64^2', 'conv', (320, 320, 64))]


def build(out):
    sys.path.insert(0, PKG)
    import _build
    sys.path.pop(0)
    pkg = os.path.join(out, 'pkg', 'cycle_diffusion_b200')
    objdir = os.path.join(out, 'obj')
    os.makedirs(pkg, exist_ok=True)
    os.makedirs(objdir, exist_ok=True)
    for f in glob.glob(os.path.join(PKG, '*.py')):
        shutil.copy(f, pkg)
    flags = list(_build.NVCC_FLAGS)
    if '-Xptxas' in flags:
        i = flags.index('-Xptxas')
        del flags[i:i + 2]                          # (the -v report)
    flags = [f for f in flags if f != '--use_fast_math=false'] + ['-DCDX_GEMM_TIMELINE']
    procs, objs = [], []
    for src in _build.SOURCES:
        obj = os.path.join(objdir, src.replace('.cu', '.o'))
        objs.append(obj)
        procs.append(subprocess.Popen([_build._nvcc()] + flags + ['-c', os.path.join(_build.CSRC, src), '-o', obj]))
    if any(p.wait() != 0 for p in procs):
        raise RuntimeError('nvcc failed')
    lib = os.path.join(pkg, 'libcdx.so')
    subprocess.run([_build._nvcc(), '-shared', '-o', lib] + objs + _build.ARCH + ['-lcudart_static', '-lpthread', '-ldl', '-lrt'], check=True)
    return os.path.join(out, 'pkg'), lib


def card():
    import torch
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        lim = r.stdout.strip() or 'unknown'
    except (OSError, subprocess.SubprocessError):
        lim = 'unknown'
    return f'{torch.cuda.get_device_name(0)}, power limit / max SM clock: {lim}'


def call_for(eng, kind, shape, g):
    import torch
    if kind == 'lin':
        tokens, K, N = shape
        M = tokens * ROWS
        f = dict(mode=0, M=M, N=N, K=K, A=torch.randn(M, K, device='cuda', generator=g), lda=K, C1=K, ldb=K,
                 w=torch.randn(N, K, device='cuda', generator=g) / K ** 0.5, residual=torch.randn(M, N, device='cuda', generator=g), ldr=N)
        side = {}
    else:
        cin, N, h = shape
        M, K = ROWS * h * h, 9 * cin
        f = dict(mode=1, M=M, N=N, K=K, A=torch.randn(ROWS, h, h, cin, device='cuda', generator=g), lda=cin, C1=cin, Hin=h, Win=h,
                 Hout=h, Wout=h, w=torch.randn(N, cin, 3, 3, device='cuda', generator=g) / K ** 0.5, rows_per_batch=h * h)
        side = dict(c_stats=torch.zeros(ROWS, N, 2, dtype=torch.float64, device='cuda'))
    f.update(bias=torch.randn(N, device='cuda', generator=g), ldc=N, C=torch.empty(M, N, device='cuda'),
             c_amax=torch.zeros(1, device='cuda'), **side)
    return lambda: eng.op_gemm(**f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='build directory of the timeline variant (default: a temporary one)')
    ap.add_argument('--reps', type=int, default=5)
    args = ap.parse_args()
    out = args.out or tempfile.mkdtemp(prefix='gemm_timeline_')
    root, libpath = build(out)
    sys.path.insert(0, root)
    import torch
    from cycle_diffusion_b200.engine import Engine
    lib = C.CDLL(libpath)
    lib.cdx_gemm_timeline_buffer.argtypes = [C.c_void_p]
    eng = Engine(0)
    eng.set_mma_mode(1)
    buf = torch.zeros(4096 * SLOTS, dtype=torch.int64, device='cuda')
    assert lib.cdx_gemm_timeline_buffer(C.c_void_p(buf.data_ptr())) == 0
    print(card())
    print(f'{"shape":28s} {"arm":8s} {"CTAs":>5s} {"items/CTA":>9s} ' + ' '.join(f'{p:>7s}' for p in PHASES) +
          f' {"life/item":>9s} {"span":>8s}   (us, medians)')
    for label, kind, shape in SHAPES:
        g = torch.Generator(device='cuda').manual_seed(sum(shape))
        fn = call_for(eng, kind, shape, g)
        for arm, persist in (('items', False), ('persist', True)):
            eng.set_persist(persist)
            fn()
            ph, life, spans, ctas, items = {p: [] for p in PHASES}, [], [], 0, 0
            for _ in range(args.reps):
                buf.zero_()
                plan = fn()
                torch.cuda.synchronize()
                st = buf.view(-1, SLOTS).cpu()
                st = st[st[:, 0] > 0]
                ctas = st.shape[0]
                total = -(-shape[0] * ROWS // 128) * -(-shape[2] // plan['width']) if kind == 'lin' else None
                if total is None:
                    h = shape[2]
                    total = -(-ROWS * h * h // 128) * -(-shape[1] // plan['width'])
                items = total / ctas
                for i, p in enumerate(PHASES):
                    ph[p] += ((st[:, i + 1] - st[:, i]).double() / 1e3).tolist()
                life += ((st[:, 6] - st[:, 0]).double() / 1e3 / items).tolist()
                spans.append((st[:, 6].max() - st[:, 0].min()).item() / 1e3)
            print(f'{label:28s} {arm:8s} {ctas:5d} {items:9.2f} ' + ' '.join(f'{statistics.median(ph[p]):7.2f}' for p in PHASES) +
                  f' {statistics.median(life):9.2f} {statistics.median(spans):8.1f}')
    eng.set_persist(True)
    lib.cdx_gemm_timeline_buffer(None)


if __name__ == '__main__':
    main()
