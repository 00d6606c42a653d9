"""Without a GPU: the normalisation test hooks are exported and bound, and the float64 references of tests/test_norms_gpu.py agree
with torch.nn.functional in float64 wherever torch has the same operation (one source, no scale-shift, no mask)."""
import math

import pytest
import torch
import torch.nn.functional as F

from cycle_diffusion_b200 import _cabi
from tests.test_norms_gpu import (GN_CASES, groupnorm_ref, layernorm_ref, softmax_ref, straddles, valid_mask)

HOOKS = ('cdx_op_groupnorm_ex', 'cdx_op_layernorm_ex', 'cdx_op_softmax_rows', 'cdx_op_produce_norm')


def test_norm_hooks_are_exported():
    for s in HOOKS:
        assert s in _cabi.SIGNATURES and hasattr(_cabi.lib, s)
    from cycle_diffusion_b200.engine import Engine
    for m in ('op_groupnorm_ex', 'op_layernorm_ex', 'op_softmax_rows', 'op_produce_norm'):
        assert callable(getattr(Engine, m))


def test_straddle_rule():
    # [1280 | 640]: 60 channels per group, channel 1280 falls inside group 21; [1280 | 1280]: 80 per group, on a boundary
    assert straddles(1280, 640) and straddles(640, 320) and not straddles(1280, 1280) and not straddles(320, 0)
    assert sum(straddles(c[0], c[1]) for c in GN_CASES if c[1]) >= 3


@pytest.mark.parametrize('B,HW,C,eps,silu', [(2, 7, 32, 1e-5, False), (1, 64, 96, 1e-6, True), (3, 1, 160, 1e-5, False),
                                             (2, 81, 320, 1e-6, True)])
def test_groupnorm_ref_matches_torch(B, HW, C, eps, silu):
    g = torch.Generator().manual_seed(C + HW)
    x = torch.randn(B, HW, C, generator=g, dtype=torch.float64) * 3 + 2
    gamma, beta = torch.randn(C, generator=g, dtype=torch.float64), torch.randn(C, generator=g, dtype=torch.float64)
    eps32 = float(torch.tensor(eps, dtype=torch.float32))
    ref = F.group_norm(x.permute(0, 2, 1), 32, gamma, beta, eps32).permute(0, 2, 1)
    if silu:
        ref = F.silu(ref)
    y, t, a, o, _ = groupnorm_ref(x, None, gamma, beta, eps, silu=silu)
    assert float((y - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max()))
    assert float((t - (x * a[:, None, :] + o[:, None, :])).abs().max()) == 0.0
    # the two-source form is the norm of the concat
    y2 = groupnorm_ref(x[..., :C // 2], x[..., C // 2:], gamma, beta, eps, silu=silu)[0]
    assert torch.equal(y2, y)


def test_groupnorm_ref_scale_shift():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 16, 64, generator=g, dtype=torch.float64)
    gamma, beta = torch.randn(64, generator=g, dtype=torch.float64), torch.randn(64, generator=g, dtype=torch.float64)
    emb = torch.rand(2, 128, generator=g, dtype=torch.float64) * 4 - 2
    scale, shift = emb[:, :64], emb[:, 64:]
    y = groupnorm_ref(x, None, gamma, beta, 1e-5, scale, shift)[0]
    plain = F.group_norm(x.permute(0, 2, 1), 32, gamma, beta, float(torch.tensor(1e-5, dtype=torch.float32))).permute(0, 2, 1)
    assert float((y - (plain * (1 + scale[:, None, :]) + shift[:, None, :])).abs().max()) <= 1e-12


@pytest.mark.parametrize('M,C', [(1, 32), (7, 388), (5, 2048)])
def test_layernorm_ref_matches_torch(M, C):
    g = torch.Generator().manual_seed(M * C)
    x = torch.randn(M, C, generator=g, dtype=torch.float64) + 30
    gamma, beta = torch.randn(C, generator=g, dtype=torch.float64), torch.randn(C, generator=g, dtype=torch.float64)
    y = layernorm_ref(x, gamma, beta)[0]
    ref = F.layer_norm(x, (C,), gamma, beta, float(torch.tensor(1e-5, dtype=torch.float32)))
    assert float((y - ref).abs().max()) <= 1e-11 * max(1.0, float(ref.abs().max()))


@pytest.mark.parametrize('L', [1, 31, 1000])
def test_softmax_ref_matches_torch(L):
    g = torch.Generator().manual_seed(L)
    x = (torch.rand(12, L, generator=g, dtype=torch.float64) * 2 - 1) * 80
    p, valid = softmax_ref(x)
    assert bool(valid.all()) and float((p - torch.softmax(x, dim=-1)).abs().max()) <= 1e-15


def test_causal_mask_rows():
    v = valid_mask(154, 100, 77, 'cpu')
    assert v[0].sum() == 1 and v[76].sum() == 77 and v[77].sum() == 1 and v[153].sum() == 77
    x = torch.randn(154, 100, dtype=torch.float64)
    p, _ = softmax_ref(x, 77)
    assert bool((p[~v] == 0).all()) and float((p.sum(-1) - 1).abs().max()) <= 1e-14
    assert math.isclose(float(p[5, :6].sum()), 1.0, rel_tol=1e-14)
