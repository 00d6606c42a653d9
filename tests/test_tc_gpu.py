"""Tensor-core (wgmma) back end: per-op and network-level parity against fp32 references, for both fp32-faithful product schemes --
mma_mode 1 (default): weight GEMMs / convs as 3 x wgmma .f16 over an fp16 hi/lo split of power-of-two-scaled operands;
mma_mode 3: everything as 3 x wgmma .tf32.

Both keep ~2^-21 relative error per product (hi*hi + lo*hi + hi*lo with fp32 accumulation in registers, chunked every 256 K elements),
so the same fp32 round-off budgets as the FFMA path apply (2e-5 relative per op, 2e-4 through a whole U-Net)."""
import math

import pytest
import torch
import torch.nn.functional as F

from cycle_diffusion_b200 import specs
from tests.common import NARROW, VAE_SMALL, WIDE, golden, maxdiff

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', params=[1, 3], ids=['h16', 'tf32'])
def eng(request):
    from cycle_diffusion_b200.engine import Engine
    e = Engine(0)
    e.set_mma_mode(request.param)
    return e


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / max(1e-30, float(b.double().abs().max())))


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


@pytest.mark.parametrize('M,K,N', [(128, 32, 128), (128, 64, 128), (256, 320, 128), (4096, 320, 2560), (1000, 96, 100), (300, 1280, 36),
                                   (20000, 640, 640), (308, 768, 640), (640, 2592, 320), (512, 11520, 1280)])
def test_linear_tc(eng, M, K, N):
    g = torch.Generator().manual_seed(M + K + N)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / math.sqrt(K)
    b = torch.randn(N, generator=g)
    l0 = eng.profile(True)
    y = eng.op_linear(x.cuda(), w.cuda(), b.cuda()).cpu()
    fam = eng.profile_read()
    eng.profile(False)
    assert 'dense_tc' in fam, f'tensor-core path was not taken: {fam}'
    r = rel(y, F.linear(x, w, b))
    print(f'linear_tc {M}x{K}x{N}: rel {r:.2e}')
    assert r < 2e-5


@pytest.mark.parametrize('B,Cin,Cout,H', [(1, 32, 128, 16), (2, 64, 64, 16), (1, 320, 320, 32), (4, 128, 256, 64), (3, 96, 160, 8), (8, 64, 32, 4),
                                           (2, 1280, 1280, 8),
                                           # Cin % 64 == 0, W >= 16: split-K items that start / end inside a channel
                                           # block, ragged batch, ragged N tile, many channel blocks
                                           (1, 1280, 640, 16), (8, 640, 640, 32), (3, 192, 96, 32), (1, 1920, 320, 64), (5, 64, 48, 16),
                                           # 8 x 8 level: two images per 128-row tile; ragged batch / N
                                           (8, 1280, 1280, 8), (4, 128, 64, 8), (12, 192, 80, 8), (7, 64, 48, 8)])
def test_conv3x3_tc(eng, B, Cin, Cout, H):
    g = torch.Generator().manual_seed(Cin * 1000 + Cout + H)
    x = torch.randn(B, Cin, H, H, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(9 * Cin)
    b = torch.randn(Cout, generator=g)
    eng.profile(True)
    y = nchw(eng.op_conv3x3(nhwc(x).cuda(), w.cuda(), b.cuda(), 1, 1, 1).cpu())
    fam = eng.profile_read()
    eng.profile(False)
    assert 'conv3x3_tc' in fam, f'tensor-core path was not taken: {fam}'
    r = rel(y, F.conv2d(x, w, b, padding=1))
    print(f'conv_tc B{B} {Cin}->{Cout} @{H}: rel {r:.2e}')
    assert r < 2e-5


@pytest.mark.parametrize('name,cfg', [('unet_sd_narrow', NARROW), ('unet_sd_wide', WIDE)])
def test_unet_tc_vs_reference_fixture(eng, name, cfg):
    from cycle_diffusion_b200.engine import UNet
    g = golden(name)
    sd = specs.synth_state_dict(specs.openai_unet_params(cfg), int(g['seed']))
    net = UNet(eng, cfg, 'openai').load_state_dict(sd)
    eng.profile(True)
    y = net(g['x'], g['t'], g['ctx']).cpu()
    fam = eng.profile_read()
    eng.profile(False)
    r = float((y.double() - g['y'].double()).abs().max() / max(1.0, float(g['y'].abs().max())))
    print(f'{name} (tensor cores): rel max err {r:.3e}; families {{k: v["launches"] for k, v in fam.items()}}')
    assert 'conv3x3_tc' in fam or 'dense_tc' in fam
    assert r < 2e-4


def test_cycle_tc_vs_reference_fixture(eng):
    from cycle_diffusion_b200.engine import UNet
    from cycle_diffusion_b200.schedule import DDIMSchedule
    g = golden('ddim_cycle_narrow')
    S, skip, wb, enc_scale, dec_scale, seed = [float(v) for v in g['cfg_a']]
    S, skip, wb, seed = int(S), int(skip), int(wb), int(seed)
    sd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    unet = UNet(eng, NARROW, 'openai').load_state_dict(sd)
    sched = DDIMSchedule(S, 0.1, skip)
    n_rec = min(sched.refine_steps, wb - skip - 1)
    torch.manual_seed(seed)
    noise = torch.zeros((n_rec + 1,) + tuple(g['x0'].shape))
    noise[0] = torch.randn(g['x0'].shape)
    for i in range(n_rec):
        if sched.refine_steps - 1 - i != 0:
            noise[1 + i] = torch.randn(g['x0'].shape)
    z = unet.latent_encode(g['x0'], g['c_src'], g['uc'], enc_scale, sched, n_rec, noise)
    zref = g['z_a'].view(z.shape)
    rz = maxdiff(z.cpu(), zref) / float(zref.abs().max())
    tgt = unet.latent_decode(zref, g['c_tgt'], g['uc'], dec_scale, sched).cpu()
    own = unet.latent_decode(z, g['c_src'], g['uc'], enc_scale, sched).cpu()
    print(f'cycle (tensor cores): rel|dz| {rz:.2e} |d tgt| {maxdiff(tgt, g["tgt_a"]):.2e} own-cycle {maxdiff(own, g["x0"]):.2e}')
    assert rz < 2e-4 and maxdiff(tgt, g['tgt_a']) < 1e-3 and maxdiff(own, g['x0']) < 1e-3


@pytest.mark.parametrize('mode', [1, 2, 3])
@pytest.mark.parametrize('B,N,heads,d', [(1, 4096, 8, 40), (2, 1024, 8, 80), (2, 256, 2, 16), (1, 128, 4, 64), (1, 256, 3, 32), (3, 384, 2, 40)])
def test_attention_tc(B, N, heads, d, mode):
    """mode 1: fused flash kernel on fp16-split operands (wgmma .f16, S/P never leave the SM); mode 2: unfused tensor-core
    QK^T / softmax / PV^T; mode 3: the fused kernel on TF32 planes (round-1 scheme, kept for --mma 3)."""
    from cycle_diffusion_b200.engine import Engine
    e = Engine(0)
    e.set_mma_mode(mode)
    g = torch.Generator().manual_seed(N + d)
    C = heads * d
    q, k, v = (torch.randn(B, N, C, generator=g) for _ in range(3))
    q = q * 1.5
    scale = d ** -0.5
    sp = lambda t: t.reshape(B, -1, heads, d).permute(0, 2, 1, 3)
    attn = (torch.einsum('bhid,bhjd->bhij', sp(q), sp(k)) * scale).softmax(-1)
    ref = torch.einsum('bhij,bhjd->bhid', attn, sp(v)).permute(0, 2, 1, 3).reshape(B, N, C)
    e.profile(True)
    y = e.op_attention(q.cuda(), k.cuda(), v.cuda(), heads, scale).cpu()
    fam = e.profile_read()
    e.profile(False)
    err = float((y - ref).abs().max())
    print(f'attention mode {mode} B{B} N{N} h{heads} d{d}: max abs err {err:.2e}  ({ {k_: round(v_["ms"], 3) for k_, v_ in fam.items()} })')
    assert 'batched_tc' in fam
    assert err < 2e-5


def test_attention_tc_vae_shape():
    """The KL-f8 mid-block attention at 512x512 (AEM:178-202): one head, d = 512, 4096 tokens.  It is outside the fused kernel's
    head dims, so it must take the unfused tensor-core route (two batched contractions around the row softmax), not the FFMA tiles."""
    from cycle_diffusion_b200.engine import Engine
    e = Engine(0)
    e.set_mma_mode(1)
    B, N, heads, d = 1, 4096, 1, 512
    g = torch.Generator().manual_seed(512)
    q, k, v = (torch.randn(B, N, d, generator=g) for _ in range(3))
    scale = d ** -0.5
    ref = torch.einsum('bij,bjd->bid', (torch.einsum('bid,bjd->bij', q, k) * scale).softmax(-1), v)
    e.profile(True)
    y = e.op_attention(q.cuda(), k.cuda(), v.cuda(), heads, scale).cpu()
    fam = e.profile_read()
    e.profile(False)
    err = float((y - ref).abs().max())
    print(f'attention d=512 N=4096: max abs err {err:.2e}  families {sorted(fam)}')
    assert 'batched_tc' in fam and 'batched_ffma' not in fam, sorted(fam)
    assert err < 2e-5


@pytest.mark.gpu
@pytest.mark.parametrize('sq,sk,sv', [(1e3, 1e-3, 1.0), (1e-4, 1e4, 3e4), (1.0, 1.0, 1e-10), (2e-3, 5e2, 1e6)])
def test_attention_h16_is_scale_invariant(sq, sk, sv):
    """The fp16-split attention rescales q, k and v by exact powers of two from their measured ranges: operands far outside
    fp16's own range must give the same relative accuracy as O(1) data (same scores, output proportional to sv)."""
    from cycle_diffusion_b200.engine import Engine
    e = Engine(0)
    e.set_mma_mode(1)
    B, N, heads, d = 2, 256, 4, 40
    g = torch.Generator().manual_seed(77)
    C = heads * d
    q, k, v = (torch.randn(B, N, C, generator=g) for _ in range(3))
    q, k, v = q * 1.5 * sq, k * sk, v * sv
    scale = d ** -0.5
    sp = lambda t: t.double().reshape(B, -1, heads, d).permute(0, 2, 1, 3)
    attn = (torch.einsum('bhid,bhjd->bhij', sp(q), sp(k)) * scale).softmax(-1)
    ref = torch.einsum('bhij,bhjd->bhid', attn, sp(v)).permute(0, 2, 1, 3).reshape(B, N, C)
    y = e.op_attention(q.cuda(), k.cuda(), v.cuda(), heads, scale).cpu().double()
    r = float((y - ref).abs().max() / ref.abs().max())
    print(f'attention scales q{sq:g} k{sk:g} v{sv:g}: rel err {r:.2e}')
    assert r < 2e-5


@pytest.mark.gpu
@pytest.mark.parametrize('B,N,Nk,heads,d', [(2, 256, 77, 2, 40), (1, 128, 77, 2, 80), (2, 128, 130, 1, 64), (3, 128, 64, 2, 32), (2, 256, 5, 1, 16)])
def test_cross_attention_flash(B, N, Nk, heads, d):
    """Cross-attention (Nk != N, ragged last key block masked in the kernel; CrossAttention.forward attention.py:170-193)."""
    from cycle_diffusion_b200.engine import Engine
    e = Engine(0)
    e.set_mma_mode(1)
    g = torch.Generator().manual_seed(N + Nk + d)
    C = heads * d
    q = torch.randn(B, N, C, generator=g) * 1.5
    k, v = (torch.randn(B, Nk, C, generator=g) for _ in range(2))
    scale = d ** -0.5
    sp = lambda t: t.reshape(B, -1, heads, d).permute(0, 2, 1, 3)
    attn = (torch.einsum('bhid,bhjd->bhij', sp(q), sp(k)) * scale).softmax(-1)
    ref = torch.einsum('bhij,bhjd->bhid', attn, sp(v)).permute(0, 2, 1, 3).reshape(B, N, C)
    e.profile(True)
    y = e.op_attention(q.cuda(), k.cuda(), v.cuda(), heads, scale).cpu()
    fam = e.profile_read()
    e.profile(False)
    err = float((y - ref).abs().max())
    print(f'cross attention B{B} N{N} Nk{Nk} h{heads} d{d}: max abs err {err:.2e}')
    assert 'batched_tc' in fam, fam.keys()
    assert err < 2e-5


@pytest.mark.parametrize('scale_x,scale_w', [(1e-6, 1.0), (3e4, 1e-3), (1.0, 250.0), (1e-12, 1e3)])
def test_h16_split_is_scale_invariant(scale_x, scale_w):
    """The fp16-split path rescales both operands by exact powers of two derived from their tracked max: activations and
    weights far outside fp16's own range (1e-12 ... 3e4) must give the same relative accuracy as O(1) data, including a
    tensor with one huge outlier next to small values."""
    from cycle_diffusion_b200.engine import Engine
    e = Engine(0)
    e.set_mma_mode(1)
    g = torch.Generator().manual_seed(5)
    M, K, N = 512, 640, 256
    x = torch.randn(M, K, generator=g) * scale_x
    x[3, 7] = 1000.0 * scale_x                      # outlier: 1000 x the typical magnitude
    w = torch.randn(N, K, generator=g) / math.sqrt(K) * scale_w
    b = torch.randn(N, generator=g) * scale_x * scale_w
    y = e.op_linear(x.cuda(), w.cuda(), b.cuda()).cpu()
    ref = F.linear(x.double(), w.double(), b.double())
    r = float((y.double() - ref).abs().max() / ref.abs().max())
    # rows without the outlier must be as accurate as the rest (absolute error of the lo plane is relative to the tensor max)
    r_typ = float((y[8:].double() - ref[8:]).abs().max() / ref[8:].abs().max())
    print(f'h16 scale test x{scale_x:g} w{scale_w:g}: rel {r:.2e}  typical rows {r_typ:.2e}')
    assert r < 2e-5 and r_typ < 2e-5


def test_fast_path_is_reduced_precision_and_marked():
    """mma_mode 4 (hi*hi only) is the separately reported fast path: ~1e-3 relative, NOT a parity mode."""
    from cycle_diffusion_b200.engine import Engine
    e = Engine(0)
    g = torch.Generator().manual_seed(6)
    x, w = torch.randn(1024, 640, generator=g), torch.randn(320, 640, generator=g) / math.sqrt(640)
    ref = F.linear(x, w)
    e.set_mma_mode(4)
    r_fast = rel(e.op_linear(x.cuda(), w.cuda(), None).cpu(), ref)
    e.set_mma_mode(1)
    r_full = rel(e.op_linear(x.cuda(), w.cuda(), None).cpu(), ref)
    print(f'fast path rel {r_fast:.2e} vs faithful {r_full:.2e}')
    assert r_full < 2e-5 and 1e-5 < r_fast < 5e-3

