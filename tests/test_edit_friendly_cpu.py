"""Edit-friendly inversion without a GPU: the SDE-DPM-Solver++ table against its float64 formulas, the draw scalars, the float64
algebra that pins the step (a first-order SDE-DPM-Solver++ step is the DDIM eta = 1 step), exact reconstruction of the oracle loop,
the descriptor layout, and the pipeline's rejections."""
import ctypes as C

import numpy as np
import pytest
import torch

from cycle_diffusion_b200 import _cabi
from cycle_diffusion_b200.schedule import DDIMSchedule, EditFriendlySchedule, ldm_alphas_cumprod
from tests.edit_friendly_oracle import ef_cycle

GEOMETRIES = [(4, 0), (6, 2), (10, 3), (20, 4), (50, 10), (50, 0), (100, 20), (1, 0), (2, 1)]


def dpm_reference(S, skip):
    """a, b, c, n and the order of every loop step, straight from the float64 formulas over the fp32 abar of the DDIM table"""
    d = DDIMSchedule(S, 1.0, skip)
    ac = ldm_alphas_cumprod().double().numpy()
    R = d.refine_steps
    levels = [ac[d.timesteps[R - 1 - i]] for i in range(R)] + [ac[0]]
    lam = lambda v: np.log(np.sqrt(v)) - np.log(np.sqrt(1 - v))
    rows = []
    for i in range(R):
        s, t = levels[i], levels[i + 1]
        h = lam(t) - lam(s)
        order = 1 if i == 0 or (i == R - 1 and R < 15) else 2
        b = np.sqrt(t) * -np.expm1(-2 * h)
        rows.append((np.sqrt(1 - t) / np.sqrt(1 - s) * np.exp(-h), b,
                     0.5 * b / ((lam(s) - lam(levels[i - 1])) / h) if order == 2 else 0.0, np.sqrt(1 - t) * np.sqrt(-np.expm1(-2 * h)), order))
    return rows


@pytest.mark.parametrize('S,skip', GEOMETRIES)
def test_dpm_table_matches_the_float64_formulas(S, skip):
    sched = EditFriendlySchedule(S, skip)
    ref = dpm_reference(S, skip)
    assert len(sched.dpm) == sched.refine_steps == len(ref)
    for i, (c, (a, b, cc, n, order)) in enumerate(zip(sched.dpm, ref)):
        assert (c.a, c.b, c.c, c.n) == tuple(float(np.float32(v)) for v in (a, b, cc, n)), i
        assert c.order == order and c.n > 0, i
    R = sched.refine_steps
    assert sched.dpm[0].order == 1
    assert sched.dpm[-1].order == (1 if R < 15 else 2 if R > 1 else 1)


@pytest.mark.parametrize('S,skip', GEOMETRIES)
def test_geometry_draw_scalars_and_ddim_table(S, skip):
    """The loop geometry and the step table are DDIMSchedule(S, 1, skip)'s; the draw scalars are sqrt_a_T's expression per step."""
    sched, ddim = EditFriendlySchedule(S, skip, solver='ddpm'), DDIMSchedule(S, 1.0, skip)
    assert sched.t_loop == ddim.t_loop and sched.refine_steps == ddim.refine_steps
    assert all(bytes(a) == bytes(b) for a, b in zip(sched.coef, ddim.coef))
    assert (sched.qa[0], sched.q1[0]) == (ddim.sqrt_a_T, ddim.sqrt_1ma_T)
    ac = ldm_alphas_cumprod()
    for k in range(sched.refine_steps):
        at = ac[ddim.timesteps[sched.refine_steps - 1 - k]]
        assert sched.qa[k] == at.sqrt().item() and sched.q1[k] == (1 - at).sqrt().item()
    with pytest.raises(ValueError):
        EditFriendlySchedule(S, skip, solver='dpmsolver')


@pytest.mark.parametrize('S,skip', [(10, 0), (50, 10), (250, 0)])
def test_first_order_step_is_the_ddim_eta1_step(S, skip):
    """In float64, the first-order SDE-DPM-Solver++ step (mean a*x + b*D, noise n) equals DDIM at eta = 1 (mean sqrt(a_prev)*D +
    sqrt(1 - a_prev - sigma^2)*eps, noise sigma) on the same x and D, at every step of the schedule: the same sampler."""
    d = DDIMSchedule(S, 1.0, skip)
    ac = ldm_alphas_cumprod().double().numpy()
    R = d.refine_steps
    levels = [ac[d.timesteps[R - 1 - i]] for i in range(R)] + [ac[0]]
    g = np.random.default_rng(0)
    x, D, z = g.standard_normal(64), g.standard_normal(64), g.standard_normal(64)
    lam = lambda v: np.log(np.sqrt(v)) - np.log(np.sqrt(1 - v))
    worst = 0.0
    for i in range(R):
        s, t = levels[i], levels[i + 1]
        h = lam(t) - lam(s)
        a, b, n = np.sqrt(1 - t) / np.sqrt(1 - s) * np.exp(-h), np.sqrt(t) * -np.expm1(-2 * h), np.sqrt(1 - t) * np.sqrt(-np.expm1(-2 * h))
        sigma = np.sqrt((1 - t) / (1 - s) * (1 - s / t))
        eps = (x - np.sqrt(s) * D) / np.sqrt(1 - s)
        ddim = np.sqrt(t) * D + np.sqrt(1 - t - sigma ** 2) * eps + sigma * z
        dpm = a * x + b * D + n * z
        worst = max(worst, float(np.abs(dpm - ddim).max()), abs(n - sigma))
    assert worst < 1e-12, worst


def toy_unet(x, t, c):
    """a smooth nonlinear stand-in for a U-Net: depends on x, the timestep and the context"""
    shape = (-1,) + (1,) * (x.dim() - 1)
    return torch.tanh(0.7 * x + c.mean(dim=(1, 2)).view(shape)) * (t.to(x.dtype) / 1000).view(shape) + 0.1 * x


def _inputs(R, seed=0, B=2):
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(B, 4, 6, 5, generator=g)
    c = torch.randn(B, 7, 8, generator=g)
    uc = torch.randn(B, 7, 8, generator=g)
    noise = torch.randn(R + 1, B, 4, 6, 5, generator=g)
    return x0, c, uc, noise


@pytest.mark.parametrize('solver', ['ddpm', 'dpmsolver++'])
@pytest.mark.parametrize('S,skip', [(6, 2), (20, 0), (50, 10)])
@pytest.mark.parametrize('scale', [1.0, 3.0])
def test_identical_chains_reconstruct_x0(solver, S, skip, scale):
    """The defining property of the noise space: with identical prompts and scales the target gets the source's draws back, so the
    loop returns x0 -- to rounding in float64 (1e-10) and within a few fp32 ulps of the latent's scale in fp32."""
    sched = EditFriendlySchedule(S, skip, solver=solver)
    x0, c, uc, noise = _inputs(sched.refine_steps)
    y64, z64 = ef_cycle(toy_unet, x0, c, c, uc, sched, scale, scale, noise, dtype=torch.float64)
    err64 = float((y64 - x0.double()).abs().max())
    y32, _ = ef_cycle(toy_unet, x0, c, c, uc, sched, scale, scale, noise)
    err32 = float((y32 - x0).abs().max())
    assert err64 < 1e-10, err64
    assert err32 < 64 * 2.0 ** -24 * float(x0.abs().max()) * sched.refine_steps, err32
    assert bool(torch.isfinite(z64).all())


def test_different_prompts_edit():
    """With different target prompts the loop does not reconstruct: the edit goes through"""
    sched = EditFriendlySchedule(20, 4)
    x0, c, uc, noise = _inputs(sched.refine_steps)
    y, _ = ef_cycle(toy_unet, x0, c, c + 1.0, uc, sched, 1.0, 3.0, noise)
    assert float((y - x0).abs().max()) > 1e-2


def test_descriptor_layout():
    """The edit-friendly fields trail the whole earlier descriptor, in cdx.h's order; the sampler entry point is bound."""
    D = _cabi.LatentChainsSamplerDesc
    assert issubclass(D, _cabi.LatentChainsMaskDesc)
    assert [f[0] for f in D._fields_] == ['solver', 'dc', 'd_src', 'd_tgt', 'qa', 'q1']
    assert D.solver.offset == C.sizeof(_cabi.LatentChainsMaskDesc)
    assert C.sizeof(_cabi.DpmCoef) == 20
    assert D.dc.offset == D.solver.offset + 4 and D.d_src.offset == -(-(D.dc.offset + 20) // 8) * 8
    assert 'cdx_cycle_lockstep_sampler' in _cabi.SIGNATURES
    sp, keep = EditFriendlySchedule(8, 2).sampler_struct()
    assert sp.kind == _cabi.CDX_SAMPLER_DPMSOLVER_DRAWS and sp.qa[0] == keep[0][0] and sp.dpm[1].order == 2


def _bare_pipeline():
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    return CycleDiffusionPipeline.__new__(CycleDiffusionPipeline)


@pytest.mark.parametrize('kw', [dict(inversion='ddim'), dict(inversion='ddpm', eta=0.1), dict(inversion='dpmsolver++', eta=0.0),
                                dict(inversion='dpmsolver++', two_phase=True), dict(inversion='ddpm', eta=1.0, two_phase=True)])
def test_pipeline_rejections(kw):
    """An unknown inversion, an eta other than 1 under the edit-friendly inversions, and two_phase with them raise ValueError before
    any work."""
    with pytest.raises(ValueError):
        _bare_pipeline()('a dog', 'a cat', image=None, **kw)


def test_pipeline_eta_default():
    import inspect
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    params = inspect.signature(CycleDiffusionPipeline.__call__).parameters
    assert params['eta'].default is None and params['inversion'].default == 'cycle'
