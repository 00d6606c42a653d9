"""CPU checks of the GEMM epilogue suite's references (tests/gemm_epilogue_oracle.py) and of the cdx_op_gemm binding."""
import math
import struct

import pytest
import torch
import torch.nn.functional as F

from tests import gemm_epilogue_oracle as O


def f32_bits(x):
    return struct.unpack('<I', struct.pack('<f', x))[0]


def from_bits(b):
    return torch.tensor([b & 0xFFFFFFFF], dtype=torch.int64).to(torch.int32).view(torch.float32)


def test_op_gemm_is_declared_exported_and_bound():
    from cycle_diffusion_b200 import _cabi
    from cycle_diffusion_b200.engine import Engine
    from tests.test_cabi import header_symbols
    assert 'cdx_op_gemm' in header_symbols() and 'cdx_op_gemm' in _cabi.SIGNATURES
    assert hasattr(_cabi.lib, 'cdx_op_gemm') and callable(Engine.op_gemm)
    d = _cabi.GemmDesc()
    for f in Engine.GEMM_POINTERS:
        assert hasattr(d, f)
    p = Engine.gemm_plan(8 | 2 << 4 | 64 << 8 | 5 << 16 | 1 | 4)
    assert p == dict(kind='h16', width=64, splits=5, amax_fused=True, stats_fused=False)
    assert Engine.gemm_plan(128 << 8 | 1 << 16)['kind'] == 'ffma'


# (input bit pattern, expected rn_tf32 bit pattern): (b + 0x1000) & 0xFFFFE000
RN_CASES = [
    (0x3F800000, 0x3F800000),                       # 1.0: already a TF32 value
    (0x3F800FFF, 0x3F800000),                       # just below half an ulp: down
    (0x3F801000, 0x3F802000),                       # a tie: away from zero (round-to-even would give 0x3F800000)
    (0x3F803000, 0x3F804000),                       # a tie on an odd TF32 mantissa: up as well
    (0x3FFFF000, 0x40000000),                       # carry through the mantissa into the exponent: 2.0
    (0xBF801000, 0xBF802000),                       # negative tie: away from zero in magnitude
    (0xBFFFF000, 0xC0000000),                       # negative carry into the exponent: -2.0
    (0x7F7FEFFF, 0x7F7FE000),                       # near the fp32 maximum, below the tie: stays finite
    (0x7F7FF000, 0x7F800000),                       # the fp32 maximum's tie carries into infinity
    (0x00000FFF, 0x00000000),                       # a subnormal below half a TF32 ulp: zero
    (0x80001000, 0x80002000),                       # negative subnormal tie
]


@pytest.mark.parametrize('src,want', RN_CASES, ids=[f'{s:08x}' for s, _ in RN_CASES])
def test_rn_tf32_bit_patterns(src, want):
    got = O.rn_tf32(from_bits(src)).view(torch.int32).item() & 0xFFFFFFFF
    assert got == want, f'{src:08x} -> {got:08x}, want {want:08x}'


def test_tf32_planes_reconstruct():
    x = torch.randn(4096, generator=torch.Generator().manual_seed(1)) * 1e3
    hi, lo = O.tf32_planes(x)
    assert torch.equal(hi, O.rn_tf32(x)) and torch.equal(lo, O.rn_tf32(x - hi))
    assert ((hi.view(torch.int32) & 0x1FFF) == 0).all() and ((lo.view(torch.int32) & 0x1FFF) == 0).all()
    err = (x.double() - hi.double() - lo.double()).abs()
    assert (err <= 2.0 ** -21 * x.double().abs()).all()


def test_geglu_reference_matches_torch():
    """the interleaved-layout reference equals F.gelu GEGLU on de-interleaved weights"""
    g = torch.Generator().manual_seed(2)
    M, K, N = 37, 48, 256
    x = torch.randn(M, K, generator=g, dtype=torch.float64)
    w = torch.randn(N, K, generator=g, dtype=torch.float64)
    o, v, gate = O.geglu_ref(x @ w.t())
    wv, wg = O.deinterleave_geglu(w)
    ref = (x @ wv.t()) * F.gelu(x @ wg.t())
    assert torch.allclose(o, ref, rtol=1e-12, atol=1e-12)
    assert torch.equal(v, x @ wv.t()) and torch.equal(gate, x @ wg.t())
    # block layout: rows 64 j .. 64 j + 31 are value rows, the next 32 their gates
    assert torch.equal(wv[:32], w[:32]) and torch.equal(wg[:32], w[32:64]) and torch.equal(wv[32:64], w[64:96])


def test_geglu_bound_covers_float32_evaluation():
    """an fp32 evaluation of v * (0.5 g (1 + erf(g c))) in torch stays inside the derived bound"""
    g = torch.Generator().manual_seed(3)
    v = (torch.randn(20000, generator=g) * 4).float()
    gate = (torch.randn(20000, generator=g) * 6).float()
    o32 = v * (0.5 * gate * (1.0 + torch.erf(gate * 0.70710678118654752440)))
    o64 = v.double() * 0.5 * gate.double() * (1.0 + torch.erf(gate.double() / math.sqrt(2.0)))
    ratio = float(((o32.double() - o64).abs() / (O.geglu_bound(v.double(), gate.double()) + 1e-300)).max())
    assert ratio <= 1.0


def test_h16_exp():
    assert O.h16_exp(1.0) == 14 and O.h16_exp(2.0 ** 14) == 0 and O.h16_exp(0.75) == 15 and O.h16_exp(0.0) == 0
    assert O.h16_exp(float('inf')) == 0 and O.h16_exp(1e-40) == 100 and O.h16_exp(1e38) == -100
    for a in (1e-3, 0.3, 7.0, 12345.0):
        assert 2.0 ** 14 <= a * 2.0 ** O.h16_exp(a) < 2.0 ** 15


@pytest.mark.parametrize('a_up,w_up', [(1.0, 1.0), (2.0 ** 8, 1.0), (1.0, 2.0 ** 10), (1.0, 2.0 ** 20), (2.0 ** 8, 2.0 ** 20)])
def test_split_floor_covers_simulated_split(a_up, w_up):
    """a float64 simulation of the fp16 split (hi * hi + hi * lo + lo * hi per product) never leaves floor + 2^-21 sum |A| |W|; with
    ranges far above the values the floor is what covers it"""
    g = torch.Generator().manual_seed(4)
    M, K, N = 64, 256, 48
    a = torch.randn(M, K, generator=g) * torch.logspace(-6, 0, K)[None, :]
    w = torch.randn(N, K, generator=g) / 16
    e_a = O.h16_exp(float(a.abs().max()) * a_up)
    b_exp = O.h16_exp(float(w.abs().max()) * w_up)
    xs, ws = a.float() * 2.0 ** e_a, w.float() * 2.0 ** b_exp
    ah, wh = xs.half().double(), ws.half().double()
    al, wl = (xs - xs.half().float()).half().double(), (ws - ws.half().float()).half().double()
    sim = (ah @ wh.t() + ah @ wl.t() + al @ wh.t()) * 2.0 ** (-e_a - b_exp)
    ref = a.double() @ w.double().t()
    floor = O.split_floor(a.double().abs().sum(1), w.double().abs().sum(1), e_a, b_exp)
    rel = 2.0 ** -21 * (a.double().abs() @ w.double().abs().t())
    assert ((sim - ref).abs() <= floor + rel).all()
    # each element: |x - (hi + lo) 2^-e| <= 2^-25 2^-e + 2^-22 |x|
    err = (O.split_h16(a, e_a) - a.double()).abs()
    assert (err <= 2.0 ** -25 * 2.0 ** -e_a + 2.0 ** -22 * a.double().abs()).all()
    if a_up > 1:     # the conservative slot really does push small elements into the floor
        assert float((err - 2.0 ** -22 * a.double().abs()).max()) > 0


def test_index_maps_agree_with_permute_and_transpose():
    B, R, N = 3, 10, 7
    y = torch.arange(B * R * N, dtype=torch.float32).reshape(B * R, N)
    out = torch.empty(B * N * R)
    for m in range(B * R):
        for n in range(N):
            out[O.nchw_index(m // R, n, m % R, N, R)] = y[m, n]
    assert torch.equal(out.reshape(B, N, R), y.reshape(B, R, N).permute(0, 2, 1))
    M, t0, ldt = 9, 3, 12
    ct = torch.full(((N - t0) * ldt,), -1.0)
    for m in range(M):
        for n in range(t0, N):
            ct[O.ct_index(m, n, t0, ldt)] = y[m, n]
    assert torch.equal(ct.reshape(N - t0, ldt)[:, :M], y[:M, t0:].t())
    assert (ct.reshape(N - t0, ldt)[:, M:] == -1).all()
