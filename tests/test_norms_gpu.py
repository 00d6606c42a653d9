"""GroupNorm, LayerNorm and row softmax in every form the network executors call them, against float64 references of the
same operation written out here (plain torch on float64 copies; tests/test_norms_cpu.py checks them against
torch.nn.functional where torch has the operation).

Forms covered: two-source GroupNorm over the never-materialised U-Net skip concat, including groups that straddle the two
sources; the improved-DDPM scale-shift norm gn(x)*(1+scale)+shift with scale / shift rows of stride 2C; SiLU; GroupNorm statistics
made by the producing GEMM's epilogue (or, where it cannot, by the standalone pass) and trusted by the norm; the tracked range
slot every norm and producer writes for the fp16-split GEMM that consumes its output; the (a, o) table the GroupNorm kernel
applies, as it stores it; LayerNorm at the text-tower widths and across the kernel's register-blocking boundaries; causal
softmax.

The fp32-affine bound.  With u = 2^-24, the kernels hold per channel a = fp32(rstd) * gamma (* (1 + scale)) and
o = (beta - fp32(mean) * a') (* (1 + scale) + shift), a' = rstd * gamma, from float64 statistics, and store y = fma(x, a, o).
Each of a, mean, a' * mean, the subtraction, the products with (1 + scale) and the sum with shift is one rounding, so
    |a - a64| <= 4u |a64| (checked at 8u),   |o - o64| <= 8u o_terms,   o_terms = |1 + scale| (|beta| + |mean a'64|) + |shift|
(o_terms, not |o64|: o is formed by sums that may cancel, and each rounding is relative to the magnitudes summed), and
    |y - y64| <= 8u (|x| |a64| + o_terms) + 8u |y64|.
SiLU multiplies the pre-activation error by |silu'(t64)|: the first term is scaled by it.  The kernel's SiLU is
__fdividef(t, 1 + __expf(-t)).  __expf is within 2 + 1.173|t| ulp (<= 2u relative each) and carries into the divisor with
weight e^-t / (1 + e^-t) = sigmoid(-t); the sum and __fdividef (2 ulp) add a few u more, so the second term becomes
u (8 + (4 + 2.346 |t64|) sigmoid(-t64)) |y64|.  For t < -126 ln 2 the divisor reaches 2^126, __fdividef returns 0, and
|silu(t)| = |t| e^t <= |t| 2^-126: an absolute term 2^-126 (1 + |t64|) covers that underflow.  It is tight by construction:
elements just past the threshold print ratios up to |t| / (1 + |t|) ~ 0.989.

LayerNorm computes its row mean and sum of squared deviations in fp32 (GroupNorm's statistics are fp64): each is a sum of depth
d = ceil(C / 128) + 7 (pairs, the per-lane loop, five shuffles), so |mean - mean64| <= d u mean|x| and rstd is off by at most
d u / 2 relative; the LayerNorm bound adds d u |a64| (mean|x| + |x - mean64| / 2) to the one above.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
GROUPS = 32


def f32(v):
    """the value an fp32 argument carries (the kernels take eps as a float)"""
    return float(torch.tensor(v, dtype=torch.float32))


# ---------------------------------------------------------------------------------------------------- float64 references
def groupnorm_ref(x1, x2, gamma, beta, eps, scale=None, shift=None, silu=False):
    """GroupNorm(32) of cat(x1, x2) over [B, HW, C] (channels last), then * (1 + scale) + shift ([B, C]), then SiLU; float64.
    Returns y, the pre-activation t, the per-(image, channel) table a, o (t = x a + o) and o_terms (module docstring)."""
    x = (torch.cat([x1, x2], dim=-1) if x2 is not None else x1).double()
    B, HW, C = x.shape
    cpg = C // GROUPS
    xg = x.reshape(B, HW, GROUPS, cpg)
    mean = xg.mean(dim=(1, 3))
    var = ((xg - mean[:, None, :, None]) ** 2).mean(dim=(1, 3))
    rstd = 1.0 / torch.sqrt(var + f32(eps))
    mean_c, rstd_c = mean.repeat_interleave(cpg, dim=1), rstd.repeat_interleave(cpg, dim=1)
    a1 = rstd_c * gamma.double()
    o1 = beta.double() - mean_c * a1
    o_terms = beta.double().abs() + (mean_c * a1).abs()
    if scale is not None:
        s1 = 1.0 + scale.double()
        a, o = a1 * s1, o1 * s1 + shift.double()
        o_terms = s1.abs() * o_terms + shift.double().abs()
    else:
        a, o = a1.expand(B, C), o1
    t = x * a[:, None, :] + o[:, None, :]
    y = t * torch.sigmoid(t) if silu else t
    return y, t, a, o, o_terms.expand(B, C)


def layernorm_ref(x, gamma, beta, eps=1e-5):
    """LayerNorm over the last dim of [M, C]; float64.  Returns y, a [M, C], o [M, C], o_terms [M, C]."""
    x = x.double()
    mean = x.mean(dim=-1, keepdim=True)
    var = ((x - mean) ** 2).mean(dim=-1, keepdim=True)
    a = gamma.double() / torch.sqrt(var + f32(eps))
    o = beta.double() - mean * a
    return x * a + o, a, o, beta.double().abs() + (mean * a).abs()


def softmax_ref(x, causal_nq=0):
    """Row softmax of [rows, L]; causal_nq > 0: row r sees columns j <= r % causal_nq and the others are 0.  float64."""
    x = x.double()
    rows, L = x.shape
    valid = valid_mask(rows, L, causal_nq, x.device)
    return torch.softmax(x.masked_fill(~valid, -math.inf), dim=-1), valid


def valid_mask(rows, L, causal_nq, device):
    j = torch.arange(L, device=device)[None, :]
    if causal_nq <= 0:
        return torch.ones(rows, L, dtype=torch.bool, device=device)
    r = torch.arange(rows, device=device)[:, None]
    return j <= r % causal_nq


def dsilu(t):
    s = torch.sigmoid(t)
    return s * (1.0 + t * (1.0 - s))


def affine_bound(x, a, o_terms, t, y, silu):
    """the fp32-affine bound of the module docstring, elementwise over [B, HW, C] (a, o_terms: [B, C])"""
    err_t = 8 * U * (x.double().abs() * a.abs()[:, None, :] + o_terms[:, None, :])
    if not silu:
        return err_t + 8 * U * y.abs()
    return err_t * dsilu(t).abs() + U * (8.0 + (4.0 + 2.346 * t.abs()) * torch.sigmoid(-t)) * y.abs() + 2.0 ** -126 * (1.0 + t.abs())


def worst(err, bound):
    return float((err / bound).max())


# ---------------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope='module')
def eng():
    from cycle_diffusion_b200.engine import Engine
    e = Engine(0)
    yield e
    e.set_mma_mode(1)


def gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def randn(g, *shape):
    return torch.randn(*shape, generator=g, device='cuda')


def rand(g, *shape):
    return torch.rand(*shape, generator=g, device='cuda')


# ---------------------------------------------------------------------------------------------------- GroupNorm
# data classes: N(0,1); offset (|mean| / std = 50); one group constant (var 0, rstd = 1/sqrt(eps)); gamma driving the
# pre-activation to about +-100
GN_CASES = [
    # C1, C2, B, HW, eps, silu, scale-shift, data
    (32, 0, 3, 65536, 1e-5, False, False, 'normal'),
    (32, 0, 1, 1, 1e-5, True, False, 'normal'),
    (96, 0, 8, 7, 1e-6, True, False, 'offset'),
    (96, 0, 1, 4096, 1e-5, False, True, 'const'),
    (160, 0, 3, 81, 1e-5, True, True, 'normal'),
    (160, 0, 1, 960, 1e-6, False, False, 'big_gamma'),
    (320, 0, 8, 960, 1e-5, True, False, 'const'),
    (320, 0, 1, 65536, 1e-6, True, False, 'offset'),
    (320, 0, 3, 64, 1e-5, False, True, 'offset'),
    (1280, 0, 3, 64, 1e-6, False, True, 'big_gamma'),
    (1280, 0, 1, 4096, 1e-5, True, False, 'normal'),
    (1280, 0, 8, 1, 1e-5, False, False, 'offset'),
    (2560, 0, 1, 1, 1e-5, False, False, 'normal'),
    (2560, 0, 8, 64, 1e-5, True, True, 'offset'),
    (2560, 0, 3, 81, 1e-6, True, False, 'big_gamma'),
    (1280, 1280, 8, 64, 1e-5, True, False, 'normal'),
    (1280, 1280, 1, 256, 1e-5, False, True, 'const'),
    (1280, 640, 8, 64, 1e-5, True, False, 'const'),
    (1280, 640, 3, 256, 1e-5, False, False, 'offset'),
    (1280, 640, 1, 1024, 1e-6, True, True, 'big_gamma'),
    (640, 640, 3, 256, 1e-5, True, False, 'offset'),
    (640, 640, 1, 1024, 1e-5, False, False, 'normal'),
    (640, 320, 8, 1024, 1e-5, True, False, 'normal'),
    (640, 320, 3, 960, 1e-6, False, True, 'const'),
    (640, 320, 1, 4096, 1e-5, True, False, 'big_gamma'),
    (320, 320, 3, 4096, 1e-5, True, False, 'offset'),
    (320, 320, 1, 65536, 1e-6, False, False, 'normal'),
    (160, 32, 8, 81, 1e-5, True, True, 'const'),
    (160, 32, 1, 7, 1e-6, False, False, 'offset'),
    (96, 64, 3, 960, 1e-5, True, False, 'big_gamma'),
    (96, 64, 8, 1, 1e-5, False, True, 'normal'),
    (128, 0, 1, 512 * 512, 1e-6, True, False, 'normal'),      # VAE decoder top: 512 x 512, 128 channels
]


def straddles(C1, C2):
    """does a GroupNorm(32) group of cat(C1, C2) hold channels of both sources?"""
    return C2 > 0 and C1 % ((C1 + C2) // GROUPS) != 0


def test_case_list_has_straddling_groups():
    pairs = sorted({(c[0], c[1]) for c in GN_CASES if c[1] > 0})
    assert pairs == sorted([(1280, 1280), (1280, 640), (640, 640), (640, 320), (320, 320), (160, 32), (96, 64)])
    assert sum(straddles(*p) for p in pairs) >= 3


def gn_data(C1, C2, B, HW, data, seed):
    g = gen(seed)
    C = C1 + C2
    x = randn(g, B, HW, C)
    gamma, beta = randn(g, C), randn(g, C)
    if data == 'offset':
        x = x + 50.0 * torch.where(rand(g, C) < 0.5, -1.0, 1.0)
    elif data == 'const':
        cpg = C // GROUPS
        grp = C1 // cpg if C2 else 5            # the group that straddles the sources when there is one
        x[0, :, grp * cpg:(grp + 1) * cpg] = 0.7
    elif data == 'big_gamma':
        gamma = 25.0 * (2.0 * rand(g, C) - 1.0)
    return x[..., :C1].contiguous(), (x[..., C1:].contiguous() if C2 else None), gamma, beta


@pytest.mark.parametrize('C1,C2,B,HW,eps,silu,ss,data', GN_CASES)
def test_groupnorm(eng, C1, C2, B, HW, eps, silu, ss, data):
    C = C1 + C2
    x1, x2, gamma, beta = gn_data(C1, C2, B, HW, data, seed=C1 * 7 + C2 * 3 + HW + B)
    scale = shift = None
    if ss:      # one [B, 2C] emb-projection output holding [scale | shift]: rows of stride 2C
        emb = 4.0 * rand(gen(C + B), B, 2 * C) - 2.0
        scale, shift = emb[:, :C], emb[:, C:]
    y, amax, ab = eng.op_groupnorm_ex(x1.view(B, HW, 1, C1), x2.view(B, HW, 1, C2) if x2 is not None else None, gamma, beta, eps, silu,
                                      scale, shift)
    torch.cuda.synchronize()
    y = y.view(B, HW, C)
    # the tracked range is a max over the stored values
    assert torch.equal(amax[0], y.abs().max()), (float(amax[0]), float(y.abs().max()))
    y64, t64, a64, o64, o_terms = groupnorm_ref(x1, x2, gamma, beta, eps, scale, shift, silu)
    x = torch.cat([x1, x2], dim=-1) if x2 is not None else x1
    a, o = ab[..., 0].double(), ab[..., 1].double()
    # the table the norm applies, as the kernel stored it
    ra = worst((a - a64).abs(), 8 * U * a64.abs() + 1e-300)
    ro = worst((o - o64).abs(), 8 * U * o_terms + 1e-300)
    ry = worst((y.double() - y64).abs(), affine_bound(x, a64, o_terms, t64, y64, silu))
    print(f'\n  gn C={C1}+{C2} B={B} HW={HW} eps={eps:g} silu={int(silu)} ss={int(ss)} {data}: '
          f'err/bound y {ry:.3f} a {ra:.3f} o {ro:.3f}')
    assert ra <= 1 and ro <= 1 and ry <= 1
    if not silu:
        # the kernel stores y = fma(x, a, o) from that same table: within 1 ulp of it
        v = x.double() * a[:, None, :] + o[:, None, :]
        ulp = (torch.nextafter(y.abs(), torch.tensor(math.inf, device=y.device)) - y.abs()).double()
        assert bool(((y.double() - v).abs() <= ulp).all())


# ---------------------------------------------------------------------------------------------------- LayerNorm
LN_CASES = [(32, 1), (32, 4097), (320, 7), (384, 77), (388, 154), (640, 4097), (768, 77), (768, 4097), (1024, 154), (1024, 7),
            (1280, 4097), (1280, 1), (2048, 7), (2048, 4097)]


@pytest.mark.parametrize('C,M', LN_CASES)
def test_layernorm(eng, C, M):
    g = gen(C * 31 + M)
    x = randn(g, M, C)
    x[::2] += 30.0                     # every other row has mean 30
    gamma, beta = randn(g, C), randn(g, C)
    y, amax = eng.op_layernorm_ex(x, gamma, beta)
    torch.cuda.synchronize()
    assert torch.equal(amax[0], y.abs().max()), (float(amax[0]), float(y.abs().max()))
    y64, a64, o64, o_terms = layernorm_ref(x, gamma, beta)
    x64 = x.double()
    d = math.ceil(C / 128) + 7
    bound = (8 * U * (x64.abs() * a64.abs() + o_terms) + 8 * U * y64.abs()
             + d * U * a64.abs() * (x64.abs().mean(dim=-1, keepdim=True) + (x64 - x64.mean(dim=-1, keepdim=True)).abs() / 2))
    r = worst((y.double() - y64).abs(), bound)
    print(f'\n  ln C={C} M={M}: err/bound {r:.3f}')
    assert r <= 1


# ---------------------------------------------------------------------------------------------------- softmax
@pytest.mark.parametrize('causal_nq', [0, 77])
@pytest.mark.parametrize('L', [1, 31, 77, 1000, 4096])
def test_softmax_rows(eng, L, causal_nq):
    rows = 2 * 77 if causal_nq else 300
    g = gen(L * 3 + causal_nq)
    x = randn(g, rows, L)
    x[: rows // 2] = 80.0 * (2.0 * rand(g, rows // 2, L) - 1.0)      # logits up to +-80 in half the rows
    p64, valid = softmax_ref(x, causal_nq)
    p = eng.op_softmax_rows(x.clone(), causal_nq)
    torch.cuda.synchronize()
    assert bool((p[~valid] == 0).all())                                # masked probabilities are exactly 0
    err = float((p.double() - p64).abs().max())
    sum_err = float((p.double().sum(dim=-1) - 1.0).abs().max())
    print(f'\n  softmax L={L} causal_nq={causal_nq}: max|p - p64| {err:.2e}  max|sum - 1| / (L u) {sum_err / (L * U):.3f}')
    assert err <= 1e-6
    assert sum_err <= L * U


# ---------------------------------------------------------------------------------------------------- producer -> norm
PRODUCER_CASES = [
    # name, conv, B, H, W, Cin, Cout, paths the tensor-core modes may take
    ('linear_hw64', False, 2, 64, 1, 320, 320, {'fused'}),
    ('linear_hw1024', False, 2, 1024, 1, 320, 320, {'fused'}),
    ('linear_hw4096', False, 1, 4096, 1, 320, 640, {'fused'}),
    ('linear_hw81', False, 2, 81, 1, 320, 320, {'tc_standalone'}),       # 81 rows per image: a warp's rows may span two images
    ('conv_8x8_b8', True, 8, 8, 8, 64, 64, {'fused'}),                  # two images per 128-row tile
    ('conv_16x16', True, 2, 16, 16, 64, 64, {'fused'}),
    ('conv_24x40', True, 1, 24, 40, 64, 64, {'tc_standalone', 'splitk'}),   # ragged tiles overhang the map
    ('linear_splitk', False, 2, 64, 1, 4096, 128, {'splitk'}),           # small M, large K: the planner splits K
    ('linear_m32', False, 1, 32, 1, 320, 64, {'ffma'}),                  # M < 64: the FFMA tiles
]
PRODUCER_PARAMS = [(m, c) for c in PRODUCER_CASES for m in (1, 3)] + [(0, PRODUCER_CASES[0])]


@pytest.mark.parametrize('mode,case', PRODUCER_PARAMS, ids=[f'mode{m}-{c[0]}' for m, c in PRODUCER_PARAMS])
def test_producer_stats_feed_groupnorm(eng, mode, case):
    name, conv, B, H, W, Cin, Cout, paths = case
    g = gen(Cin * 13 + Cout + H * W + B)
    HW = H * W
    x = randn(g, B, H, W, Cin) if conv else randn(g, B, HW, Cin)
    w = randn(g, Cout, Cin, 3, 3) / math.sqrt(9 * Cin) if conv else randn(g, Cout, Cin) / math.sqrt(Cin)
    bias, gamma, beta = randn(g, Cout), randn(g, Cout), randn(g, Cout)
    eng.set_mma_mode(mode)
    try:
        y, amax, stats, yn, path = eng.op_produce_norm(x, w, bias, gamma, beta, 1e-5, conv=conv)
        torch.cuda.synchronize()
    finally:
        eng.set_mma_mode(1)
    assert path in (paths if mode else {'ffma'}), path
    # the product itself (loosely: the epilogue's arithmetic is not under test here)
    x64, w64 = x.double().cpu(), w.double().cpu()
    if conv:
        ref = torch.nn.functional.conv2d(x64.permute(0, 3, 1, 2), w64, bias.double().cpu(), padding=1).permute(0, 2, 3, 1)
    else:
        ref = x64 @ w64.T + bias.double().cpu()
    ref = ref.reshape(B * HW, Cout)
    assert float((y.double().cpu() - ref).abs().max()) <= 1e-4 * float(ref.abs().max())
    # the range slot is a max over the stored values
    assert torch.equal(amax[0], y.abs().max()), (float(amax[0]), float(y.abs().max()))
    # statistics of the stored y, whichever pass made them
    y64 = y.double().view(B, HW, Cout)
    s64, q64, sabs = y64.sum(dim=1), (y64 * y64).sum(dim=1), y64.abs().sum(dim=1)
    rs = worst((stats[..., 0] - s64).abs(), 2.0 ** -20 * sabs)
    rq = worst((stats[..., 1] - q64).abs(), 2.0 ** -20 * q64)
    # the norm that trusts them
    yn64, t64, a64, o64, o_terms = groupnorm_ref(y.view(B, HW, Cout), None, gamma, beta, 1e-5)
    rn = worst((yn.double().view(B, HW, Cout) - yn64).abs(), affine_bound(y.view(B, HW, Cout), a64, o_terms, t64, yn64, False))
    print(f'\n  producer mode {mode} {name} ({path}): err/bound sum {rs:.3f} sumsq {rq:.3f} norm {rn:.3f}')
    assert rs <= 1 and rq <= 1 and rn <= 1
