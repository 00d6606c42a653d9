"""The attention oracle (tests/attention_oracle.py) pinned on the CPU: its plane emulations equal the GEMM oracle's, and a float32
emulation of the fused kernel's online algorithm stays inside the derived bound while reaching a visible share of it."""
import math

import numpy as np
import pytest
import torch

from tests import attention_oracle as ao
from tests import gemm_epilogue_oracle as go


def test_h16_exponent_matches_the_device_rule():
    for a in (0.0, float('inf'), float('nan'), 2.0 ** -90, 1e-3, 1.0, 3.9, 4.0, 100.0, 2.0 ** 14, 32767.0, 2.0 ** 15, 2.0 ** 60, 2.0 ** 120):
        e = ao.h16_exp_dev(a)
        host = go.h16_exp(a)
        if a > 0 and math.isfinite(a) and 4.0 <= a < 2.0 ** 15:
            assert e == 0                        # no rescale: the split is already exact to 2^-25
        else:
            assert e == host, (a, e, host)
    assert ao.h16_exp_dev(2.0 ** -90) == 100 and ao.h16_exp_dev(2.0 ** 120) == -100


@pytest.mark.parametrize('e', [-100, -46, -3, 0, 7, 14, 100])
def test_plane_emulation_matches_the_gemm_oracle(e):
    g = torch.Generator().manual_seed(e + 200)
    x = torch.randn(4096, generator=g) * 2.0 ** (14 - e) * torch.rand(4096, generator=g) ** 6
    assert torch.equal(ao.rep_h16(x, e), go.split_h16(x, e))
    hi, lo = go.tf32_planes(x)
    assert torch.equal(ao.rep_tf32(x), hi.double() + lo.double())
    assert torch.equal(ao.rn_tf32(x), go.rn_tf32(x))
    one = ao.rep_h16(x, e, lo=False)
    assert torch.equal(one, (x * 2.0 ** e).half().double() / 2.0 ** e)


def _case(kind, N, L, C, seed):
    g = torch.Generator().manual_seed(seed)
    q, k, v = torch.randn(N, C, generator=g), torch.randn(L, C, generator=g), torch.randn(L, C, generator=g)
    if kind == 'peaked':                         # one key per query dominates; most p fall below 2^-24
        q = q * 4.0
        k[L - 1] = q[0] * 0.5
    elif kind == 'offset':                       # the output forms by cancellation against a large common offset
        v = v + 300.0
    elif kind == 'uniform':
        q = torch.zeros_like(q)
    elif kind == 'last_block':                   # the online max jumps in the last, ragged key block
        k[L - 1] = q.mean(dim=0) * 6.0
    return q, k, v


CASES = [('h16', 'gauss', 130, 200, 2 * 64), ('h16', 'peaked', 64, 300, 64), ('h16', 'offset', 64, 129, 2 * 40),
         ('one', 'gauss', 64, 200, 80), ('one', 'peaked', 64, 300, 64), ('tf32', 'gauss', 64, 150, 2 * 40),
         ('tf32', 'last_block', 64, 150, 80), ('h16', 'uniform', 16, 2000, 64), ('h16_ks', 'gauss', 64, 257, 160),
         ('h16_ks', 'last_block', 64, 60, 160), ('one_ks', 'offset', 64, 190, 160)]


@pytest.mark.parametrize('fmt,kind,N,L,C', CASES)
def test_online_emulation_inside_bound(fmt, kind, N, L, C):
    ksplit = fmt.endswith('_ks')
    fmt = fmt.replace('_ks', '')
    heads = C // 160 if ksplit else C // (40 if C % 40 == 0 and C // 40 <= 2 else 64)
    heads = max(heads, 1)
    d = C // heads
    q, k, v = _case(kind, N, L, C, N + L + C)
    scale = d ** -0.5
    slot_q = float(q.abs().max()) if q.abs().max() > 0 else 0.0
    slot_kv = float(max(k.abs().max(), v.abs().max()))
    qr = ao.represent(q, fmt, slot_q)
    kr, vr = ao.represent(k, fmt, slot_kv), ao.represent(v, fmt, slot_kv)
    O64r, b = ao.reference(qr[None], kr[None], vr[None], heads, scale, fmt)
    assert (d > 80) == ksplit
    emu = ao.emulate_online(qr.numpy(), kr.numpy(), vr.numpy(), heads, scale, fmt, ksplit=ksplit)
    err = np.abs(emu - O64r[0].numpy())
    ratio = float((err / b[0].numpy()).max())
    print(f'{fmt}{" ksplit" if ksplit else ""} {kind} N{N} L{L} d{d}: worst |err| / bound {ratio:.3f}')
    assert ratio <= 1.0


def test_bound_is_not_vacuous():
    """the emulation reaches a few percent of the bound somewhere: the bound is in the range of what the arithmetic does"""
    worst = 0.0
    for fmt, kind, N, L, C in [('one', 'gauss', 64, 200, 80), ('h16', 'offset', 64, 129, 80), ('tf32', 'gauss', 64, 150, 80)]:
        q, k, v = _case(kind, N, L, C, 7 + N + L)
        d = C // 2
        slot_kv = float(max(k.abs().max(), v.abs().max()))
        qr, kr, vr = ao.represent(q, fmt, float(q.abs().max())), ao.represent(k, fmt, slot_kv), ao.represent(v, fmt, slot_kv)
        O64r, b = ao.reference(qr[None], kr[None], vr[None], 2, d ** -0.5, fmt)
        emu = ao.emulate_online(qr.numpy(), kr.numpy(), vr.numpy(), 2, d ** -0.5, fmt)
        r = float((np.abs(emu - O64r[0].numpy()) / b[0].numpy()).max())
        print(f'{fmt} {kind}: worst ratio {r:.3f}')
        worst = max(worst, r)
    assert worst >= 0.03


@pytest.mark.parametrize('fmt', ['h16', 'one'])
def test_bound_catches_unscaled_p(fmt):
    """4095 keys at p = 1.4 2^-24 carry the output: with P split as fp16(p 2^10) the emulation stays inside the bound, without the
    scale the fp16 subnormals round every one of them down and the bound fails"""
    N, d = 4096, 64
    qkv = torch.zeros(N, 3 * d)
    qkv[:, 0] = 1.0
    qkv[0, d] = -math.log(1.4 * 2.0 ** -24) / d ** -0.5
    qkv[1:, 2 * d:] = 1.0 + 0.5 * torch.rand(N - 1, d, generator=torch.Generator().manual_seed(111))
    q, k, v = qkv[None, :, :d], qkv[None, :, d:2 * d], qkv[None, :, 2 * d:]
    slot = float(qkv.abs().max())
    O64, _, b = ao.bound(q, k, v, 1, d ** -0.5, fmt, slot, slot)
    qr, kr, vr = (ao.represent(t[0], fmt, slot).numpy() for t in (q, k, v))
    ratio = lambda pre: float((np.abs(ao.emulate_online(qr, kr, vr, 1, d ** -0.5, fmt, prescale=pre) - O64[0].numpy()) / b[0].numpy()).max())
    assert ratio(True) <= 1.0
    assert ratio(False) > 4.0


def test_representation_error_within_split_budget():
    """|O64r - O64| against the module docstring's per-element representation budget, three-term and one-term, with a shared slot
    far above q and k (the floor term)"""
    g = torch.Generator().manual_seed(3)
    q, k, v = torch.randn(32, 64, generator=g) * 2.0 ** -10, torch.randn(100, 64, generator=g) * 2.0 ** -10, torch.randn(100, 64, generator=g)
    slot = float(torch.cat([q, k, v]).abs().max())
    for fmt, rel in (('h16', 2.0 ** -22), ('one', 2.0 ** -11)):
        O64, O64r, _ = ao.bound(q[None], k[None], v[None], 1, 0.125, fmt, slot, slot)
        e = ao.h16_exp_dev(slot)
        dq = rel * q.abs().double() + 2.0 ** -25 * 2.0 ** -e
        dk = rel * k.abs().double() + 2.0 ** -25 * 2.0 ** -e
        dv = rel * v.abs().double() + 2.0 ** -25 * 2.0 ** -e
        s = 0.125 * (q.double() @ k.double().T)
        w = torch.softmax(s, dim=-1)
        ds = 0.125 * ((q.abs().double() + dq) @ dk.T + dq @ k.abs().double().T).max(dim=-1, keepdim=True).values
        O = w @ v.double()
        budget = torch.expm1(2 * ds) * (w @ v.abs().double() + O.abs()) + w @ dv
        assert bool(((O64r[0] - O64[0]).abs() <= budget).all()), fmt
