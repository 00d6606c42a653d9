"""CPU checks of semantic guidance: the oracle's quantile against torch.quantile, the oracle loop's no-op settings against the masked
oracle's plain cycle bit for bit, SemanticGuidance's and the pipeline's argument validation, and the new C symbols."""
import ctypes as C

import numpy as np
import pytest
import torch

from cycle_diffusion_b200 import _cabi, specs
from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
from cycle_diffusion_b200.semantic import SemanticGuidance
from tests.common import NARROW
from tests.sega_oracle import plane_thresholds, quantile, sega_cycle


def _ulps(a, b):
    """|a - b| in units in the last place of fp32, elementwise (a, b finite and of one sign)."""
    ia = a.contiguous().view(torch.int32).to(torch.int64)
    ib = b.contiguous().view(torch.int32).to(torch.int64)
    return (ia - ib).abs()


@pytest.mark.parametrize('lam', [0.0, 0.5, 0.9, 0.999])
@pytest.mark.parametrize('n', [2, 3, 7, 16, 100, 576, 960, 4096, 9216, 14400])
def test_quantile_matches_torch_quantile(lam, n):
    """The contract's Q within 1 ulp of torch.quantile (whose vectorised lerp may fuse), on random planes, planes with many ties,
    constant planes and planes of zeros; exactly the sorted value at an integer rank."""
    g = torch.Generator().manual_seed(n * 10 + int(lam * 1000))
    planes = torch.stack([torch.randn(n, generator=g).abs() * 3,
                          torch.randint(0, 5, (n,), generator=g).to(torch.float32) * 0.25,          # ties
                          torch.full((n,), 0.7),                                                 # constant
                          torch.zeros(n),
                          torch.rand(n, generator=g) ** 4])
    got = quantile(planes, lam)
    ref = torch.quantile(planes, lam, dim=-1)
    assert int(_ulps(got, ref).max()) <= 1, (got, ref)
    r = np.float32(lam) * np.float32(n - 1)
    if r == np.floor(r):
        assert torch.equal(got, torch.sort(planes, dim=-1).values[:, int(r)])
    assert torch.equal(quantile(planes[2:3], lam), planes[2:3, 0])                                  # constant plane: the value


def test_plane_thresholds_are_per_image_and_channel():
    a = torch.rand(2, 3, 4, 5, generator=torch.Generator().manual_seed(1))
    th = plane_thresholds(a, 0.9)
    assert th.shape == (2, 3, 1, 1)
    for b in range(2):
        for c in range(3):
            assert torch.equal(th[b, c, 0, 0], quantile(a[b, c].reshape(1, -1), 0.9)[0])


def _loop_inputs():
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    g = torch.Generator().manual_seed(7)
    x0 = torch.randn(2, 4, 8, 8, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(2, 77, 48, generator=g) for _ in range(3))
    c_edit = torch.randn(2, 2, 77, 48, generator=g)
    return usd, x0, c_src, c_tgt, uc, c_edit


@pytest.mark.parametrize('tgt_scale', [3.0, 1.0])
def test_oracle_no_op_settings_are_the_masked_cycle(tgt_scale):
    """Scale 0, a warmup at or past the loop's steps, and every cooldown 0 each give masked_cycle's loop bit for bit (3 steps);
    an active setting changes the edit."""
    from oracle import unet_openai
    from tests.masked_oracle import masked_cycle
    usd, x0, c_src, c_tgt, uc, c_edit = _loop_inputs()
    fn = lambda x, t, c: unet_openai.unet_forward(usd, NARROW, x, t, c)
    base = (fn, x0, c_src, c_tgt, uc, c_edit, 6, 0.1, 3, 2.0, tgt_scale)
    with torch.no_grad():
        torch.manual_seed(3)
        (y_ref,), z_ref = masked_cycle(fn, x0, c_src, c_tgt, uc, 6, 0.1, 3, 2.0, [tgt_scale], None)
        for args in (([0.0, -0.0], [0.9, 0.5], [3, 3], 0), ([4.0, -3.0], [0.9, 0.0], [3, 3], 3), ([4.0, -3.0], [0.9, 0.0], [0, 0], 0)):
            torch.manual_seed(3)
            y, z = sega_cycle(*base, *args, 0.3, 0.4)
            assert torch.equal(y, y_ref) and all(torch.equal(a, b) for a, b in zip(z, z_ref)), args
        torch.manual_seed(3)
        y, _ = sega_cycle(*base, [4.0, -3.0], [0.9, 0.0], [3, 1], 1, 0.3, 0.4)
    assert not torch.equal(y, y_ref)


def test_semantic_guidance_values_and_validation():
    g = SemanticGuidance()
    assert (g.m, g.edit_guidance_scale, g.edit_threshold, g.edit_cooldown_steps, g.edit_warmup_steps) == (1, (5.0,), (0.9,), (None,), 10)
    assert (g.edit_momentum_scale, g.edit_mom_beta) == (0.1, 0.4)
    g = SemanticGuidance.for_concepts(3, [1, 2, 3], [False, True, False], 0.8, [None, 2, 0], 2, 0.2, 0.6)
    assert g.signed_scales() == (1.0, -2.0, 3.0) and g.edit_threshold == (0.8,) * 3 and g.edit_cooldown_steps == (None, 2, 0)
    s = g.c_struct(7)
    assert s.m == 3 and list(s.scale)[:4] == [1.0, -2.0, 3.0, 0.0] and list(s.cooldown)[:3] == [7, 2, 0] and s.warmup == 2
    assert s.beta == np.float32(0.6) and s.beta1 == np.float32(1.0 - 0.6)                  # fp32(1 - beta), formed in double
    assert SemanticGuidance.for_concepts(2) == SemanticGuidance((5.0, 5.0), (False, False), (0.9, 0.9), (None, None))
    bad = [dict(m=0), dict(m=9), dict(m=2, edit_guidance_scale=[1.0]), dict(m=1, edit_threshold=1.0), dict(m=1, edit_threshold=-0.1),
           dict(m=2, reverse_editing_direction=[True]), dict(m=1, reverse_editing_direction=1), dict(m=1, edit_cooldown_steps=-1),
           dict(m=1, edit_cooldown_steps=1.5), dict(m=1, edit_warmup_steps=[1]), dict(m=1, edit_warmup_steps=-1),
           dict(m=1, edit_guidance_scale=float('nan')), dict(m=1, edit_mom_beta=1.5), dict(m=1, edit_momentum_scale=float('inf')),
           dict(m=2, edit_threshold=[0.5, 0.5, 0.5])]
    for kw in bad:
        with pytest.raises(ValueError):
            SemanticGuidance.for_concepts(**kw)
    with pytest.raises(AttributeError):                             # frozen
        g.edit_warmup_steps = 3


def test_pipeline_rejects_what_the_engine_cannot_do():
    """Rejected before any work: two_phase, an attention edit_type, list lengths other than m, and a per-concept warmup list."""
    pipe = CycleDiffusionPipeline.__new__(CycleDiffusionPipeline)
    call = lambda **k: pipe('a dog', 'a cat', None, **k)
    for kw in (dict(editing_prompt='glasses', two_phase=True),
               dict(editing_prompt='glasses', cross_attention_kwargs={'edit_type': 'mutual_self'}),
               dict(editing_prompt='glasses', cross_attention_kwargs={'edit_type': 'pnp'}),
               dict(editing_prompt=['glasses', 'hat'], edit_guidance_scale=[3.0]),
               dict(editing_prompt=['glasses', 'hat'], reverse_editing_direction=[True, False, True]),
               dict(editing_prompt=['glasses', 'hat'], edit_threshold=[0.9]),
               dict(editing_prompt=['glasses', 'hat'], edit_cooldown_steps=[3]),
               dict(editing_prompt=['glasses', 'hat'], edit_warmup_steps=[2, 3]),
               dict(editing_prompt=[]), dict(editing_prompt=['c'] * 9), dict(editing_prompt='glasses', edit_threshold=1.0)):
        with pytest.raises(ValueError):
            call(**kw)


def test_new_c_symbols_are_bound():
    assert hasattr(_cabi.lib, 'cdx_cycle_lockstep_semantic') and 'cdx_cycle_lockstep_semantic' in _cabi.SIGNATURES
    assert _cabi.CDX_SEMANTIC_MAX == 8
    assert C.sizeof(_cabi.SemanticGuidanceC) == 4 * (1 + 8 + 8 + 8 + 1 + 3)
    names = [f[0] for f in _cabi.LatentChainsDesc._fields_]
    assert names[names.index('hw') + 1:] == ['sg_m', 'sg_rows', 'sg_thr', 'sg_nu', 'sg_scale', 'sg_lambda', 'sg_active', 'sg_apply', 'sg_mu',
                                             'sg_beta', 'sg_beta1']
