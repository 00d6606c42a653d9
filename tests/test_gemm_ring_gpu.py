"""The tensor-core GEMM's shared-memory ring at the K lengths and tile widths where its stage bookkeeping can go wrong.

The ring holds 32-K stages (7 deep at BN 128, 9 at BN 64 in the fp16-split kinds; 4 / 7 for the TF32 kinds); the consumers accumulate
in chunks of 256 K (one chunk when a work item's K is at most 512) and split-K items cover whole 64-K blocks.  Every shape below is
checked against a float64 reference with the bounds of test_tc_gpu.py, in mma modes 1 (fp16 split), 3 (3xTF32), 4 and 5 (single-term
fp16: reduced precision), and run twice with bitwise-equal results.
"""
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

MODES = [1, 3, 4, 5]
FAITHFUL = {1: 2e-5, 3: 2e-5, 4: 5e-3, 5: 5e-3}       # relative bound per op (modes 4 / 5: hi*hi only)


@pytest.fixture(scope='module', params=MODES, ids=[f'mode{m}' for m in MODES])
def eng(request):
    from cycle_diffusion_b200.engine import Engine
    e = Engine(0)
    e.set_mma_mode(request.param)
    return e


def rel(a, ref):
    return float((a.double() - ref).abs().max() / max(1e-30, float(ref.abs().max())))


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def profiled(eng, fn):
    eng.profile(True)
    y = fn()
    fam = eng.profile_read()
    eng.profile(False)
    return y, fam


# (M, K, N): K = 32 (one stage), 96, 224 (exactly one ring at BN 128), 256, 288 (ring wrap, 256-K chunk edge), 544 (two chunks),
# 11520 (hundreds of ring wraps); N = 64 / 96 / 320 / 2560 (BN 64 and 128 tiles); small M with K 11520 / 5120: split-K work items
LINEARS = [(256, 32, 128), (512, 96, 64), (1024, 224, 128), (512, 256, 96), (768, 288, 320), (1024, 544, 320), (512, 11520, 128),
           (4096, 320, 2560), (384, 11520, 64), (256, 5120, 1280)]


@pytest.mark.parametrize('M,K,N', LINEARS)
def test_ring_linear(eng, M, K, N):
    g = torch.Generator().manual_seed(M * 7 + K * 3 + N)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / math.sqrt(K)
    b = torch.randn(N, generator=g)
    xc, wc, bc = x.cuda(), w.cuda(), b.cuda()
    y, fam = profiled(eng, lambda: eng.op_linear(xc, wc, bc).cpu())
    assert 'dense_tc' in fam, f'tensor-core path was not taken: {sorted(fam)}'
    r = rel(y, F.linear(x.double(), w.double(), b.double()))
    print(f'ring linear mode {eng.mma_mode} M{M} K{K} N{N}: rel {r:.2e}')
    assert r < FAITHFUL[eng.mma_mode]
    assert torch.equal(eng.op_linear(xc, wc, bc).cpu(), y), 'two runs of the same GEMM differ'


# (B, Cin, Cout, H, W, stride): stride 1 and 2, 8x8 to 64x64 maps, K = 9 Cin from 288 to 11520; a ragged 24x40 map
CONVS = [(2, 32, 64, 16, 16, 1), (4, 320, 320, 32, 32, 1), (12, 1280, 1280, 8, 8, 1), (2, 640, 640, 32, 32, 2), (3, 96, 160, 16, 16, 2),
         (2, 64, 96, 24, 40, 1), (12, 2560, 1280, 8, 8, 1)]


@pytest.mark.parametrize('B,Cin,Cout,H,W,stride', CONVS)
def test_ring_conv3x3(eng, B, Cin, Cout, H, W, stride):
    g = torch.Generator().manual_seed(Cin * 1000 + Cout + H + W + stride)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(9 * Cin)
    b = torch.randn(Cout, generator=g)
    xc, wc, bc = nhwc(x).cuda(), w.cuda(), b.cuda()
    y, fam = profiled(eng, lambda: eng.op_conv3x3(xc, wc, bc, stride, 1, 1).cpu())
    assert 'conv3x3_tc' in fam, f'tensor-core path was not taken: {sorted(fam)}'
    r = rel(nchw(y), F.conv2d(x.double(), w.double(), b.double(), stride=stride, padding=1))
    print(f'ring conv3x3 mode {eng.mma_mode} B{B} {Cin}->{Cout} {H}x{W} s{stride}: rel {r:.2e}')
    assert r < FAITHFUL[eng.mma_mode]
    assert torch.equal(eng.op_conv3x3(xc, wc, bc, stride, 1, 1).cpu(), y), 'two runs of the same conv differ'


# A U-Net whose 160-channel level makes the output ResBlocks' 1x1 skip convs two-source GEMMs ([h | skip] concatenated inside the
# kernel) whose first source is 5 ring stages wide; its GEGLU feed-forwards are 1280 wide.
ODD = dict(in_channels=4, out_channels=4, model_channels=160, attention_resolutions=(1, 2), num_res_blocks=1, channel_mult=(1, 2),
           num_heads=4, context_dim=768)

_UNET_SCRIPT = r'''
import sys, torch
from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.engine import Engine, UNet
from oracle import unet_openai
from tests.test_gemm_ring_gpu import ODD
mode = int(sys.argv[1])
sd = specs.synth_state_dict(specs.openai_unet_params(ODD), 21)
g = torch.Generator().manual_seed(4)
x, ctx = torch.randn(2, 4, 16, 16, generator=g), torch.randn(2, 77, 768, generator=g)
t = torch.tensor([901., 17.])
eng = Engine(0)
eng.set_mma_mode(mode)
net = UNet(eng, ODD, 'openai').load_state_dict(sd)
eng.profile(True)
y = net(x.cuda(), t.cuda(), ctx.cuda()).cpu()
fam = eng.profile_read()
eng.profile(False)
y2 = net(x.cuda(), t.cuda(), ctx.cuda()).cpu()
with torch.no_grad():
    ref = unet_openai.unet_forward(sd, ODD, x, t, ctx).double()
rel = float((y.double() - ref).abs().max() / ref.abs().max())
print('RESULT', rel, int(torch.equal(y, y2)), int('dense_tc' in fam and 'conv3x3_tc' in fam))
'''


def run_unet(mode):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, '-c', _UNET_SCRIPT, str(mode)], capture_output=True, text=True, cwd=root, timeout=600)
    assert r.returncode == 0, r.stderr[-1500:]
    f = [l for l in r.stdout.splitlines() if l.startswith('RESULT')][-1].split()
    return float(f[1]), f[2] == '1', f[3] == '1'


@pytest.mark.parametrize('mode', [1, 3])
def test_ring_unet_two_source_dense(mode):
    """Whole U-Net against the fp32 reference (test_tc_gpu.py's network bound), twice with bitwise-equal outputs."""
    r, same, tc = run_unet(mode)
    print(f'ring U-Net mode {mode}: rel {r:.2e}')
    assert tc and same and r < 2e-4

