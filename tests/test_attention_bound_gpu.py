"""Attention fed the way the networks feed it (cdx_op_attention_net: the SpatialTransformer's and the cross-attention's own operand
preparation, the text towers' and the VAE's generic route), against a float64 reference with the error bound derived in
tests/attention_oracle.py, element by element, on every route and mode at every level the networks run, with data chosen to break
one thing each.  The output sits inside a NaN-filled buffer: rows past B*N must stay NaN."""
import math

import pytest
import torch

from tests import attention_oracle as ao

pytestmark = pytest.mark.gpu

WORST = {}


@pytest.fixture(scope='module')
def engs():
    from cycle_diffusion_b200.engine import Engine
    out = {}
    for m in (0, 1, 2, 3, 5):
        out[m] = Engine(0)
        out[m].set_mma_mode(m)
    yield out
    print('\nworst |O - O64| / bound per route and mode: ' + '  '.join(f'{k}: {v:.3g}' for k, v in sorted(WORST.items())))


ROUTE = {1: 'fused_h16', 3: 'fused_tf32', 5: 'fused_one'}
GUARD = 64


def _guarded(M, C, dev, prev=None):
    buf = torch.full((M + GUARD, C), math.nan, device=dev)
    if prev is not None:
        buf[:M] = prev
    return buf


def _check(tag, out, buf, M, O64, O64r, b, extra=None):
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[M:]).all()), f'{tag}: rows past the output written'
    y = out.double()
    assert bool(torch.isfinite(y).all()), f'{tag}: non-finite output'
    err = (y - O64).abs()
    if extra is not None:
        b = b + extra
    ratio = err / b.clamp_min(1e-300)
    worst = float(ratio.max())
    WORST[tag] = max(WORST.get(tag, 0.0), worst)
    print(f'{tag}: worst |O - O64| / bound {worst:.3g}  max |O - O64| {float(err.max()):.3g}')
    assert worst <= 1.0, f'{tag}: {int((ratio > 1).sum())} elements outside the bound, worst {worst:.3g}'


def run_self(eng, mode, qkv, B, N, heads, d, slot=0.0, qk_rows=None, kv_rows=None, acc_rows=None, prev=None, expect=None):
    """one self-attention through the SpatialTransformer's preparation, checked against the bound"""
    C = heads * d
    dev = qkv.device
    M = B * N
    buf = _guarded(M, C, dev, prev)
    out = buf[:M]
    scale = d ** -0.5
    plan = eng.op_attention_net('self', out, B, N, heads, d, scale, qkv=qkv, slot=slot, qk_rows=qk_rows, kv_rows=kv_rows, acc_rows=acc_rows)
    if expect is not None:
        for k_, v_ in expect.items():
            assert plan[k_] == v_, (plan, expect)
    route = plan['route']
    fmt = {'fused_h16': 'h16', 'fused_tf32': 'tf32', 'fused_one': 'one'}.get(route, 'generic')
    x = qkv.view(B, N, 3 * C)
    q, k, v = x[..., :C], x[..., C:2 * C], x[..., 2 * C:]
    if qk_rows is not None:
        q, k = q[list(qk_rows)], k[list(qk_rows)]
    if kv_rows is not None:
        k, v = k[list(kv_rows)], v[list(kv_rows)]
    s = slot if slot > 0 else float(qkv.abs().max())
    O64, O64r, b = ao.bound(q, k, v, heads, scale, fmt, s, s)
    extra = None
    if acc_rows is not None:
        base = prev.view(B, N, C).double()
        sel = torch.zeros(B, dtype=torch.bool, device=dev)
        sel[list(acc_rows)] = True
        O64 = torch.where(sel[:, None, None], base + O64, base)
        b = torch.where(sel[:, None, None], b, torch.zeros_like(b))
        extra = 2 * ao.U * O64.abs()
    _check(f'self {route} m{mode}', out.view(B, N, C), buf, M, O64, O64r, b, extra)
    return plan


def run_cross(eng, mode, q, kvp, B, N, L, Lp, heads, d, slot=0.0, q_slot=0.0, expect=None):
    C = heads * d
    M = B * N
    buf = _guarded(M, C, q.device)
    out = buf[:M]
    scale = d ** -0.5
    plan = eng.op_attention_net('cross', out, B, N, heads, d, scale, q=q, kv=kvp, L=L, ctx_lp=Lp, slot=slot, q_slot=q_slot)
    if expect is not None:
        for k_, v_ in expect.items():
            assert plan[k_] == v_, (plan, expect)
    fmt = {'fused_h16': 'h16', 'fused_tf32': 'tf32', 'fused_one': 'one'}.get(plan['route'], 'generic')
    kv = kvp.view(B, Lp, 2 * C)[:, :L]
    qs = q_slot if q_slot > 0 else float(q.abs().max())
    ks = slot if slot > 0 else float(kvp.abs().max())
    O64, O64r, b = ao.bound(q.view(B, N, C), kv[..., :C], kv[..., C:], heads, scale, fmt, qs, ks)
    _check(f'cross {plan["route"]} m{mode}', out.view(B, N, C), buf, M, O64, O64r, b)
    return plan


def _qkv(B, N, C, seed, sq=1.0, sk=1.0, sv=1.0, dev='cuda'):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(B * N, 3 * C, device=dev, generator=g)
    x[:, :C] *= sq
    x[:, C:2 * C] *= sk
    x[:, 2 * C:] *= sv
    return x


def _ctx(B, N, L, Lp, C, seed, dev='cuda'):
    g = torch.Generator(device=dev).manual_seed(seed)
    q = torch.randn(B * N, C, device=dev, generator=g)
    kv = torch.zeros(B, Lp, 2 * C, device=dev)
    kv[:, :L] = torch.randn(B, L, 2 * C, device=dev, generator=g)
    return q, kv.view(B * Lp, 2 * C)


# ------------------------------------------------------------------------------------------------ every level the networks run
# (tokens, heads, d, batch): SD v1 at 512 and 576, SD 2 at 768, the rectangular 24x40 latent
LEVELS = [(4096, 8, 40, 1), (1024, 8, 80, 3), (256, 8, 160, 3), (64, 8, 160, 12),
          (5184, 8, 40, 1), (1296, 8, 80, 1), (324, 8, 160, 3), (81, 8, 160, 3),
          (9216, 5, 64, 1), (2304, 10, 64, 1), (576, 20, 64, 3), (144, 20, 64, 12),
          (960, 8, 40, 3), (240, 8, 80, 3), (60, 8, 160, 3), (15, 8, 160, 12)]


@pytest.mark.parametrize('mode', [1, 3, 5])
@pytest.mark.parametrize('N,heads,d,B', LEVELS)
def test_self_levels(engs, mode, N, heads, d, B):
    qkv = _qkv(B, N, heads * d, N + d + B + mode)
    expect = {'route': ROUTE[mode], 'Nks': N, 'Nvs': (N + 7) // 8 * 8 if mode != 3 else (N if N % 4 == 0 else (N + 3) // 4 * 4)}
    if mode == 3 and d > 80:                     # TF32 planes at d = 160 have no fused kernel
        expect = {'route': 'unfused_tc' if N % 32 == 0 and N >= 128 else 'generic'}
    elif mode != 3:
        expect.update(qrows=64 if d > 80 else 128, ksplit=int(d > 80), rag=int(N % (64 if d > 80 else 128) != 0))
    run_self(engs[mode], mode, qkv, B, N, heads, d, expect=expect)


@pytest.mark.parametrize('mode', [1, 3, 5])
@pytest.mark.parametrize('L', [77, 1, 8, 65])
def test_cross_context(engs, mode, L):
    Lp = (L + 7) // 8 * 8
    for N, heads, d, B in ((1024, 8, 40, 3), (81, 8, 160, 3) if mode != 3 else (81, 8, 80, 3), (15, 5, 64, 12)):
        q, kv = _ctx(B, N, L, Lp, heads * d, N + L + mode)
        run_cross(engs[mode], mode, q, kv, B, N, L, Lp, heads, d, expect={'route': ROUTE[mode], 'Nks': Lp, 'Nvs': Lp})


def test_text_towers_causal(engs):
    """CLIP-L (12 heads) and OpenCLIP-H (16 heads) self-attention: causal, L = 77, d = 64, generic route"""
    dev = 'cuda'
    for mode in (0, 1):
        for heads in (12, 16):
            B, L, d = 3, 77, 64
            C = heads * d
            g = torch.Generator(device=dev).manual_seed(heads + mode)
            q, k, v = (torch.randn(B * L, C, device=dev, generator=g) for _ in range(3))
            k[1::L] *= 40.0                      # key 1 dominates every row that may see it: a causal mask off by one moves row 0
            buf = _guarded(B * L, C, dev)
            out = buf[:B * L]
            plan = engs[mode].op_attention_net('generic', out, B, L, heads, d, d ** -0.5, q=q, k=k, v=v, L=L, causal=True)
            assert plan['route'] == 'generic'
            O64, O64r, b = ao.bound(q.view(B, L, C), k.view(B, L, C), v.view(B, L, C), heads, d ** -0.5, 'generic', causal=True)
            _check(f'causal generic m{mode}', out.view(B, L, C), buf, B * L, O64, O64r, b)


def test_unfused_and_vae(engs):
    """mode 2 (unfused tensor-core attention) at U-Net levels, mode 0 (FFMA) and the VAE AttnBlock (one head of 512)"""
    run_self(engs[2], 2, _qkv(3, 1024, 640, 5), 3, 1024, 8, 80, expect={'route': 'unfused_tc'})
    run_self(engs[2], 2, _qkv(1, 4096, 320, 6), 1, 4096, 8, 40, expect={'route': 'unfused_tc'})
    run_self(engs[0], 0, _qkv(3, 240, 640, 7), 3, 240, 8, 80, expect={'route': 'generic'})
    run_self(engs[0], 0, _qkv(1, 1024, 512, 8), 1, 1024, 1, 512, expect={'route': 'generic'})
    run_self(engs[1], 1, _qkv(1, 1024, 512, 9), 1, 1024, 1, 512, expect={'route': 'unfused_tc'})


# ------------------------------------------------------------------------------------------------ adversarial data
@pytest.mark.parametrize('mode', [1, 3, 5])
def test_dominant_key_first_and_last_block(engs, mode):
    for N, heads, d, B in ((200, 2, 64, 3), (130, 2, 160, 1) if mode != 3 else (130, 2, 80, 1)):
        C = heads * d
        qkv = _qkv(B, N, C, 11 + mode)
        for j in (0, N - 1):                     # the online max jumps in block 0 and in the last, ragged block
            y = qkv.clone().view(B, N, 3 * C)
            y[:, j, C:2 * C] = y[:, :, :C].mean(dim=1) * 8.0
            run_self(engs[mode], mode, y.view(B * N, 3 * C), B, N, heads, d)


@pytest.mark.parametrize('mode', [1, 3, 5])
@pytest.mark.parametrize('N', [15, 60, 81])
def test_mask_against_next_image(engs, mode, N):
    """K at the per-image stride N: the last 64-key box of image 0 reads image 1's first keys, which score 30 above the row's max"""
    heads, d, B = 2, (160 if mode != 3 else 80), 3
    C = heads * d
    qkv = _qkv(B, N, C, 21 + N + mode)
    x = qkv.view(B, N, 3 * C)
    u = x[0, :, :C].mean(dim=0)
    for h in range(heads):
        cs = slice(h * d, (h + 1) * d)
        x[0, :, cs] = u[cs] + 0.01 * x[0, :, cs]
        x[1, :8, C + h * d:C + (h + 1) * d] = u[cs] * (40.0 / float((u[cs] * u[cs]).sum() * d ** -0.5))
    run_self(engs[mode], mode, qkv, B, N, heads, d)


@pytest.mark.parametrize('mode', [1, 5])
@pytest.mark.parametrize('N', [15, 60, 65, 256])
def test_key_split_parity(engs, mode, N):
    """d = 160: the two warpgroups walk alternate key blocks.  All the weight in the odd blocks (or, for one block, in block 0 with
    the second warpgroup empty)"""
    heads, d, B = 2, 160, 3
    C = heads * d
    qkv = _qkv(B, N, C, 31 + N + mode)
    x = qkv.view(B, N, 3 * C)
    nb = -(-N // 64)
    for j in range(N):
        if nb > 1 and (j // 64) % 2 == 1:
            x[:, j, C:2 * C] = x[:, :, :C].mean(dim=1) * 4.0
    run_self(engs[mode], mode, qkv, B, N, heads, d, expect={'ksplit': 1, 'qrows': 64})


def test_uniform_scores_over_14400_keys(engs):
    """q = 0: every score 0, the output is mean(V) and l sums 225 blocks"""
    B, N, heads, d = 1, 14400, 8, 40
    qkv = _qkv(B, N, heads * d, 41, sq=0.0)
    run_self(engs[1], 1, qkv, B, N, heads, d)


@pytest.mark.parametrize('mode', [1, 5])
def test_peaked_scores_reach_fp16_subnormals(engs, mode):
    """scores so spread that most p fall below 2^-24: P's lo plane (and the one-term p 2^10) in the fp16 subnormals"""
    B, N, heads, d = 2, 1024, 2, 64
    qkv = _qkv(B, N, heads * d, 51 + mode, sq=6.0, sk=6.0)
    run_self(engs[mode], mode, qkv, B, N, heads, d)


@pytest.mark.parametrize('mode', [1, 3, 5])
def test_small_probabilities_stay_normal(engs, mode):
    """key 0 scores 16.3 above the 4095 others, whose p = 1.4 2^-24 carry all the output (v_0 = 0): p 2^10 keeps them in fp16's
    normal range (one-term), and P's lo plane in its subnormals (three-term).  Unscaled, each would round to 2^-24, all one way"""
    B, N, heads, d = 1, 4096, 1, 64
    C = heads * d
    qkv = torch.zeros(B * N, 3 * C, device='cuda')
    qkv[:, 0] = 1.0
    qkv[0, C] = -math.log(1.4 * 2.0 ** -24) / d ** -0.5
    g = torch.Generator(device='cuda').manual_seed(111)
    qkv[1:, 2 * C:] = 1.0 + 0.5 * torch.rand(N - 1, C, device='cuda', generator=g)
    run_self(engs[mode], mode, qkv, B, N, heads, d)


@pytest.mark.parametrize('mode', [1, 3, 5])
@pytest.mark.parametrize('sq,sv', [(2.0 ** -10, 1.0), (1.0, 2.0 ** -10)])
def test_shared_slot_disparity(engs, mode, sq, sv):
    """one range slot for q, k and v: |q|, |k| 2^10 below |v| lose the slot's exponent to v, and the reverse"""
    B, N, heads, d = 3, 200, 2, 64
    qkv = _qkv(B, N, heads * d, 61 + mode, sq=sq, sk=sq, sv=sv)
    run_self(engs[mode], mode, qkv, B, N, heads, d)


@pytest.mark.parametrize('mode', [1, 3, 5])
def test_value_offset_cancellation(engs, mode):
    B, N, heads, d = 3, 240, 2, 80
    qkv = _qkv(B, N, heads * d, 71 + mode)
    qkv[:, 2 * heads * d:] += 500.0
    run_self(engs[mode], mode, qkv, B, N, heads, d)


@pytest.mark.parametrize('mode', [1, 3, 5])
@pytest.mark.parametrize('amax', [2.0 ** -90, 2.0 ** 60])
def test_operand_scale_near_exponent_clamp(engs, mode, amax):
    B, N, heads, d = 1, 144, 2, 64
    qkv = _qkv(B, N, heads * d, 81 + mode)
    qkv *= amax / float(qkv.abs().max())
    if amax > 1:
        qkv[:, :2 * heads * d] *= 2.0 ** -63     # q, k back to a few units (finite scores) while the shared slot stays at 2^60
    run_self(engs[mode], mode, qkv, B, N, heads, d)


@pytest.mark.parametrize('mode', [1, 3, 5])
def test_all_zero(engs, mode):
    B, N, heads, d = 3, 81, 2, 64
    qkv = torch.zeros(B * N, 3 * heads * d, device='cuda')
    buf = _guarded(B * N, heads * d, qkv.device)
    engs[mode].op_attention_net('self', buf[:B * N], B, N, heads, d, d ** -0.5, qkv=qkv)
    torch.cuda.synchronize()
    assert bool((buf[:B * N] == 0).all()) and bool(torch.isnan(buf[B * N:]).all())


@pytest.mark.parametrize('mode', [1, 3, 5])
def test_conservative_slot(engs, mode):
    """a slot 2^8 above the operands' range (as V' and refine leave theirs): every element loses 8 bits to the split floor"""
    B, N, heads, d = 3, 200, 2, 40
    qkv = _qkv(B, N, heads * d, 91 + mode)
    run_self(engs[mode], mode, qkv, B, N, heads, d, slot=float(qkv.abs().max()) * 256.0)
    q, kv = _ctx(B, N, 77, 80, heads * d, 92 + mode)
    run_cross(engs[mode], mode, q, kv, B, N, 77, 80, heads, d, slot=float(kv.abs().max()) * 256.0)


# ------------------------------------------------------------------------------------------------ row tables, accumulating launch
@pytest.mark.parametrize('mode', [1, 3, 5])
def test_row_tables_and_accumulate(engs, mode):
    B, N, heads, d = 4, 81 if mode != 3 else 60, 2, (160 if mode != 3 else 80)
    C = heads * d
    qkv = _qkv(B, N, C, 101 + mode)
    run_self(engs[mode], mode, qkv, B, N, heads, d, qk_rows=[0, 1, 0, 1])
    run_self(engs[mode], mode, qkv, B, N, heads, d, kv_rows=[0, 1, 0, 1])
    prev = torch.randn(B * N, C, device='cuda')
    run_self(engs[mode], mode, qkv, B, N, heads, d, acc_rows=[2, 3], prev=prev)
