"""In-tree build of libcdx.so (nvcc, sm_90a only).  Used by __graft_entry__.build() and by the tests.

The shared library lands next to this file (cycle_diffusion_b200/libcdx.so), so the package imports from the source
tree; it is git-ignored.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libcdx.so')
STAMP = os.path.join(HERE, '.libcdx.stamp')

ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']      # H100 (Hopper): wgmma / TMA / setmaxnreg need the 'a' target
SOURCES = ['engine.cu', 'kernels_gemm.cu', 'kernels_tc.cu', 'kernels_attn.cu', 'kernels_norm.cu', 'kernels_elem.cu', 'nets.cu', 'cabi.cu']
NVCC_FLAGS = ARCH + ['-lineinfo', '-O3', '-std=c++17', '--use_fast_math=false',
              '-Xcompiler', '-fPIC', '-Xcompiler', '-O2', '--expt-relaxed-constexpr', '-Xptxas', '-v']


def _nvcc():
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return 'nvcc'


def _digest():
    h = hashlib.sha256()
    files = sorted(os.listdir(CSRC)) + [os.path.join('..', '..', 'include', 'cdx.h')]
    for f in files:
        with open(os.path.join(CSRC, f), 'rb') as fh:
            h.update(f.encode())
            h.update(fh.read())
    h.update(' '.join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every CUDA source for sm_90a into libcdx.so (object files under build/). Returns the path."""
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read().strip() == dig:
        return LIB
    flags = [f for f in NVCC_FLAGS if f != '--use_fast_math=false']
    objdir = os.path.join(HERE, 'build')
    os.makedirs(objdir, exist_ok=True)
    procs = []
    objs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace('.cu', '.o'))
        objs.append(obj)
        cmd = [_nvcc()] + flags + ['-c', os.path.join(CSRC, src), '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f'==== {src}\n{out}')
        if p.returncode != 0:
            failed = True
    with open(os.path.join(objdir, 'build.log'), 'w') as f:
        f.write('\n'.join(log))
    if failed:
        errs = [l for l in '\n'.join(log).splitlines() if 'error' in l.lower()]
        sys.stderr.write('\n'.join(errs[:40]) + '\n')
        raise RuntimeError('nvcc failed; see cycle_diffusion_b200/build/build.log')
    link = [_nvcc(), '-shared', '-o', LIB] + objs + ARCH + ['-lcudart_static', '-lpthread', '-ldl', '-lrt']
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError('link failed')
    with open(STAMP, 'w') as f:
        f.write(dig)
    if verbose:
        print('\n'.join(log))
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
