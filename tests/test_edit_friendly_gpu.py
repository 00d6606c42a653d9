"""The edit-friendly inversion on the lock-step loop (cdx_cycle_lockstep_sampler, cdx_op_latent_chains with solver 1 and 2): the init
and step launches bit for bit against tests/edit_friendly_oracle.py in every instantiation (eps and v, MASK 0 / 1, SEGA 0-3, orders 1
and 2, three launches on one pair of history buffers), the loop against the CPU oracle, reconstruction of x0 with identical chains,
masks, composition with every control, the rejections, and the pipeline's routing."""
import ctypes as C
import functools
import itertools

import pytest
import torch

from cycle_diffusion_b200 import _cabi, specs
from cycle_diffusion_b200.schedule import DDIMSchedule, EditFriendlySchedule, v_tables
from tests import edit_friendly_oracle as ef
from tests import step_oracle as so
from tests.common import NARROW, maxdiff
from tests.test_ledits_gpu import ledits_oracle_step, map_values, oracle_mask_thresholds
from tests.test_sega_gpu import _generator, eout_values, guarded, layout, oracle_thresholds, sega_oracle_step
from tests.test_step_kernels_gpu import GUARD, NAN, SA_V, S1_V, build, mask_of, same

pytestmark = pytest.mark.gpu

B, L = 2, 77
SCHEDS = [EditFriendlySchedule(10, 0), EditFriendlySchedule(10, 3), EditFriendlySchedule(50, 10)]


@pytest.fixture(scope='module')
def eng():
    from cycle_diffusion_b200.engine import Engine
    return Engine(0)


@pytest.fixture
def mode(eng):
    yield eng.set_mma_mode
    eng.set_mma_mode(1)


def step_scalars(sched, i, solver, pred, launch=0):
    """the per-step scalars the driver passes at step i (the draw of step i + 2, or x0 on the step before the last)"""
    R, t = sched.refine_steps, int(sched.t_loop[i])
    nxt = 3 if i + 2 < R else 2 if i + 1 < R else 0
    if launch == 1 and nxt == 3:
        nxt = 2                                         # the x0 branch too
    k = min(i + 2, R - 1)
    return dict(solver=solver, c=sched.coef[i], dc=sched.dpm[i], next=nxt, qa=sched.qa[k], q1=sched.q1[k], pred=pred,
                vsa=float(SA_V[t]), vs1=float(S1_V[t]))


# ================================================================================================ one launch
@pytest.mark.parametrize('K', [0, 1, 3])
def test_init_bit_exact(eng, K):
    """solver 1 / 2 init: x_T, the first independent draw (next 3) or x0 (next 2), z_out on and off, every chain-table shape"""
    for n, (nxt, z, kind, shuffle) in enumerate(itertools.product((0, 2, 3), (True, False), ('one', 'cfg', 'mixed'), (False, True))):
        sched = SCHEDS[n % len(SCHEDS)]
        Lb, meta, sc = build(0, n_src=3, K=K, src=1, C=4, h=3, w=5, kind=kind, shuffle=shuffle, next_=0, z=z,
                             sched=DDIMSchedule(10, 1.0), seed=n)
        sc.update(solver=1 + n % 2, next=nxt, sa=sched.sqrt_a_T, s1=sched.sqrt_1ma_T, qa=sched.qa[1], q1=sched.q1[1])
        host = {k: v.clone() for k, v in Lb.bufs.items()}
        ef.latent_init(**meta, **sc, **Lb.views(host))
        got = Lb.run(eng, 0, meta, sc)
        for name in host:
            assert same(got[name], host[name]), f'{name}: {kind} shuffle={shuffle} next={nxt}'


STEP_CASES = [(pred, solver, K, masked) for pred in (0, 1) for solver in (1, 2) for K in (1, 3) for masked in (False, True)]


@pytest.mark.parametrize('pred,solver,K,masked', STEP_CASES)
def test_step_bit_exact(eng, pred, solver, K, masked):
    """latent_chains_step<PRED, MASK, 0, 1 | 2>: three consecutive launches (orders 1, 2, 2 under solver 2) on one pair of history
    buffers, next 3 / 2 / 0, every chain-table shape, masks of every kind; every buffer guarded and compared after each launch"""
    for n, (kind, shuffle) in enumerate(itertools.product(('one', 'cfg', 'pick', 'mixed'), (False, True))):
        sched = SCHEDS[n % len(SCHEDS)]
        Lb, meta, _ = build(1, n_src=3, K=K, src=1, C=4, h=3, w=5, kind=kind, shuffle=shuffle, next_=1, pred=pred, sched=DDIMSchedule(10, 1.0),
                            mask='random' if masked else None, seed=300 + n)
        nsrc = 3 * 4 * 15
        Lb.add('d_src', nsrc)
        Lb.add('d_tgt', nsrc * K)
        host = {k: v.clone() for k, v in Lb.bufs.items()}
        dev = {k: v.cuda() for k, v in Lb.bufs.items()}
        for launch, i in enumerate((0, 1, sched.refine_steps - 1) if n % 2 else (0, sched.refine_steps // 2, sched.refine_steps - 2)):
            sc = dict(step_scalars(sched, i, solver, pred, launch), src=1, z_stride=3 * 4 * 15, hw=15 if masked else 0)
            ef.latent_step(**meta, **sc, **Lb.views(host))
            eng.op_latent_chains(1, **meta, **sc, **Lb.views(dev))
            torch.cuda.synchronize()
            for name in host:
                assert same(dev[name].cpu(), host[name]), f'{name} after launch {launch}: {kind} shuffle={shuffle}'


def _with_solver(step_fn, sc_extra):
    """run a SEGA / LEDITS++ oracle step (which calls step_oracle.latent_step) on the edit-friendly step instead"""
    plain = so.latent_step
    so.latent_step = functools.partial(ef.latent_step, **sc_extra)
    try:
        step_fn()
    finally:
        so.latent_step = plain


@pytest.mark.parametrize('pred,masked,sega,solver', [(p, mk, sg, s) for p in (0, 1) for mk in (False, True) for sg in (1, 2, 3) for s in (1, 2)])
def test_step_with_concepts_bit_exact(eng, pred, masked, sega, solver):
    """latent_chains_step<PRED, MASK, 1 | 2 | 3, 1 | 2>: SEGA's per-channel thresholds, LEDITS++'s attention mask and its
    intersection, m = 1 and 3, three launches on one momentum and one pair of history buffers"""
    n_src, K, C, gh, gw = 2, 2, 4, 2, 3
    h, w = 4 * gh, 4 * gw
    hw, chw = h * w, C * h * w
    sched = SCHEDS[0]
    for n, (m, kind) in enumerate(itertools.product((1, 3), ('cfg', 'mixed'))):
        g = torch.Generator().manual_seed(900 + n)
        chains, sg_rows, rows = layout(n_src, K, m, kind, n % 2 == 1, n)
        scales, lambdas = [[1.5], [3.0, 0.0, -1.25]][m > 1], [[0.9], [0.999, 0.3, 0.9]][m > 1]
        nsrc, nr = n_src * chw, n_src * K * m
        eout = eout_values(rows, chw, hw, g, chains, sg_rows, n_src, K, m)
        bufs = {'x0': guarded(nsrc, g=g), 'noise_next': guarded(nsrc, g=g), 'z_out': guarded(n_src * 3 * chw, NAN),
                'eout': guarded(rows * chw, eout), 'xt': guarded(nsrc, g=g), 'xn': guarded(nsrc, g=g), 'xn2': guarded(nsrc, NAN),
                'yt': guarded(nsrc * K, g=g), 'y_out': guarded(nsrc * K, NAN), 'xin': guarded(rows * chw, NAN),
                'sg_nu': guarded(n_src * K * chw, 0.0), 'd_src': guarded(nsrc, g=g), 'd_tgt': guarded(nsrc * K, g=g)}
        if sega > 1:
            amap = map_values(nr, gh, gw, g)
            bufs['sg_map'] = guarded(nr * gh * gw, amap.reshape(-1))
            bufs['sg_thr'] = guarded(2 * nr, oracle_mask_thresholds(eout, amap, chains, sg_rows, n_src, K, m, C, h, w, scales, lambdas, gh, gw))
        else:
            bufs['sg_thr'] = guarded(nr * C, oracle_thresholds(eout, chains, sg_rows, n_src, K, m, C, hw, scales, lambdas))
        if masked:
            bufs['mask'] = guarded(n_src * hw, mask_of('random', n_src, hw, n))
        meta = dict(chains=chains, chw=chw, n_src=n_src, K=K, rows=rows)
        dev = {k: v.cuda() for k, v in bufs.items()}
        host = {k: v.clone() for k, v in bufs.items()}
        views = lambda b: {k: b[k][GUARD: GUARD + (len(b[k]) - 2 * GUARD)] for k in b}
        for launch, i in enumerate((0, 1, 2)):
            st = step_scalars(sched, i, solver, pred, launch)
            sc = dict(src=1, c=st['c'], next=st['next'], pred=pred, vsa=st['vsa'], vs1=st['vs1'], z_stride=3 * chw, hw=hw)
            extra = dict(solver=solver, dc=st['dc'], qa=st['qa'], q1=st['q1'])
            sg = dict(sg_rows=sg_rows, sg_scale=scales, sg_lambda=lambdas, sg_active=[0b111, 0b101, 0b010][launch],
                      sg_apply=launch != 1, sg_mu=0.3, sg_beta=0.4, sg_beta1=float(torch.tensor(1 - 0.4, dtype=torch.float32)))
            hv = views(host)
            if sega > 1:
                _with_solver(lambda: ledits_oracle_step(hv, meta, sc, sg, gh, gw, w, sega == 3), extra)
            else:
                _with_solver(lambda: sega_oracle_step(hv, meta, sc, sg), extra)
            kw = dict(sg_mask=sega - 1, sg_gh=gh, sg_gw=gw, w=w) if sega > 1 else {}
            eng.op_latent_chains(1, **meta, **sc, **extra, **views(dev), **kw,
                                 **{k: (int(v) if k in ('sg_active', 'sg_apply') else v) for k, v in sg.items()})
            torch.cuda.synchronize()
            for name in bufs:
                assert same(dev[name].cpu(), host[name]), f'{name} after launch {launch}: m={m} {kind}'


# ================================================================================================ the loop
@pytest.fixture(scope='module')
def usd():
    return specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)


@pytest.fixture(scope='module')
def unet(eng, usd):
    from cycle_diffusion_b200.engine import UNet
    return UNet(eng, NARROW, 'openai').load_state_dict(usd)


@pytest.fixture
def with_prediction(unet):
    yield unet.set_prediction
    unet.set_prediction('eps')


def _inputs(R, h=16, w=16, seed=7, m=2):
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(B, 4, h, w, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(B, L, 48, generator=g) for _ in range(3))
    c_edit = torch.randn(B, m, L, 48, generator=g)
    noise = torch.randn(R + 1, B, 4, h, w, generator=g)
    noise[R] = 0.0                                     # the pipeline draws no noise for the last step
    return x0, c_src, c_tgt, uc, c_edit, noise


def _oracle(usd, x0, c_src, c_tgt, uc, sched, s, t, noise, **kw):
    from oracle import unet_openai
    fn = lambda x, ts, c: unet_openai.unet_forward(usd, NARROW, x, ts, c)
    with torch.no_grad():
        return ef.ef_cycle(fn, x0, c_src, c_tgt, uc, sched, s, t, noise, v_tabs=v_tables(), **kw)


LOOP_CASES = ([(solver, pred, s, t, (16, 16), 1) for solver in ('ddpm', 'dpmsolver++') for pred in ('eps', 'v') for s in (1.0, 2.0)
               for t in (1.0, 3.0)] + [(solver, 'eps', 2.0, 3.0, (16, 24), mma) for solver in ('ddpm', 'dpmsolver++') for mma in (1, 0)])


@pytest.mark.parametrize('solver,pred,src_scale,tgt_scale,hw,mma', LOOP_CASES)
def test_vs_oracle_loop(unet, usd, with_prediction, mode, solver, pred, src_scale, tgt_scale, hw, mma):
    """Engine against the CPU oracle loop within the bounds the SEGA / PnP / mutual loop tests use (rel|dz| < 2e-4, |dx| < 1e-3),
    the edit more than 10x the bound"""
    with_prediction(pred)
    mode(mma)
    sched = EditFriendlySchedule(6, 2, solver=solver)
    x0, c_src, c_tgt, uc, _, noise = _inputs(sched.refine_steps, *hw)
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise, return_z=True)
    y_ref, z_ref = _oracle(usd, x0, c_src, c_tgt, uc, sched, src_scale, tgt_scale, noise, prediction=pred)
    rz = maxdiff(z.cpu(), z_ref) / float(z_ref.abs().max())
    dx = maxdiff(out.cpu(), y_ref)
    edit = maxdiff(y_ref, x0)
    print(f'{solver} {pred} scales ({src_scale}, {tgt_scale}) {hw} mode {mma}: rel|dz| {rz:.2e} |dx| {dx:.2e} |x - x0| {edit:.2e}')
    assert rz < 2e-4 and dx < 1e-3 and edit > 10 * dx


@pytest.mark.parametrize('solver', ['ddpm', 'dpmsolver++'])
def test_identical_chains_reconstruct_x0(unet, usd, solver):
    """With identical prompts and scales the result is x0 up to rounding.  Bound: each step's round trip n*((x - mu)/n) + mu (or the
    DDIM step's) rounds a few times at the latent's scale, and a step's deviation is carried into the next U-Net call; the fp32
    oracle's own error on the same net and inputs measures both, floored at one ulp of max|x0| per step.  The device rounds at other
    places than the CPU, so it gets 4x that."""
    sched = EditFriendlySchedule(6, 2, solver=solver)
    x0, c_src, _, uc, _, noise = _inputs(sched.refine_steps)
    out = unet.cycle_lockstep(x0, c_src, c_src, uc, 3.0, 3.0, sched, noise).cpu()
    y_ref, _ = _oracle(usd, x0, c_src, c_src, uc, sched, 3.0, 3.0, noise)
    err_dev, err_ref = maxdiff(out, x0), maxdiff(y_ref, x0)
    ulp = 2.0 ** -23 * float(x0.abs().max())
    bound = 4 * max(err_ref, sched.refine_steps * ulp)
    print(f'{solver}: device |x - x0| {err_dev:.2e}, fp32 oracle {err_ref:.2e}, bound {bound:.2e}')
    assert err_dev <= bound


@pytest.mark.parametrize('solver', ['ddpm', 'dpmsolver++'])
def test_mask_keeps_x0_outside(unet, solver):
    """Where the mask is 0 the final latent is x0 bit for bit (the last step's next x is x0); inside it is edited"""
    sched = EditFriendlySchedule(6, 2, solver=solver)
    x0, c_src, c_tgt, uc, _, noise = _inputs(sched.refine_steps)
    m = torch.zeros(B, 1, 16, 16)
    m[..., 3:11, 5:13] = 1.0
    out = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=m).cpu()
    inside = m.expand_as(x0) == 1
    assert torch.equal(out[~inside], x0[~inside]) and float((out[inside] - x0[inside]).abs().max()) > 1e-2


def test_posterior_kind_is_cycle_lockstep(eng, unet):
    """cdx_cycle_lockstep_sampler with CDX_SAMPLER_DDIM_POSTERIOR is cdx_cycle_lockstep bit for bit"""
    from cycle_diffusion_b200.engine import _ptr
    sched = DDIMSchedule(6, 0.1, 2)
    x0, c_src, c_tgt, uc, _, noise = _inputs(sched.refine_steps)
    want = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise)
    xd, cs, ct, ud, nd = (t.cuda().contiguous() for t in (x0, c_src, c_tgt, uc, noise))
    out = torch.empty_like(xd)
    sp = _cabi.SamplerC(kind=_cabi.CDX_SAMPLER_DDIM_POSTERIOR)
    rc = _cabi.lib.cdx_cycle_lockstep_sampler(unet.h, _ptr(xd), _ptr(cs), _ptr(ct), _ptr(ud), L, 1.0, 3.0, sched.coef_array(), sched.t_array(),
                                              sched.refine_steps, _ptr(nd), sched.sqrt_a_T, sched.sqrt_1ma_T, _ptr(out), None, B, 4, 16, 16,
                                              eng.stream, C.byref(sp), None, None, None, None, None, None, None, None)
    assert rc == 0 and torch.equal(out, want)


def test_composes_with_every_control(unet):
    """Under 'dpmsolver++': SEGA with and without LEDITS++ masks, Prompt-to-Prompt replace, MasaCtrl and PnP each run; their no-op
    settings give the plain edit-friendly loop bit for bit (mode 0 for SEGA, whose extra rows share the fp16-split exponent in mode
    1), their active settings change it, and a zero mask region stays x0 under each"""
    from cycle_diffusion_b200.attn_control import AttentionControl, MutualSelfControl, PnPControl
    from cycle_diffusion_b200.semantic import SemanticGuidance
    sched = EditFriendlySchedule(6, 2)
    n = sched.refine_steps
    x0, c_src, c_tgt, uc, c_edit, noise = _inputs(sched.refine_steps)
    m = torch.zeros(B, 1, 16, 16)
    m[..., 4:12, 4:12] = 1.0
    outside = m.expand_as(x0) == 0
    run = lambda **kw: unet.cycle_lockstep(x0, c_src, c_tgt, uc, 2.0, 3.0, sched, noise, **kw).cpu()
    plain = run()
    noop = {'p2p': dict(attn_control=AttentionControl(0, 0)), 'mutual': dict(attn_control=MutualSelfControl(n, 0)),
            'pnp': dict(attn_control=PnPControl(0.0, 0.0))}
    active = {'p2p': dict(attn_control=AttentionControl(1.0, 0.5)), 'mutual': dict(attn_control=MutualSelfControl(0, 0)),
              'pnp': dict(attn_control=PnPControl()),
              'sega': dict(semantic=SemanticGuidance.for_concepts(2, [3.0, 2.0], [False, True], [0.9, 0.5], None, 1), c_edit=c_edit),
              'ledits': dict(semantic=SemanticGuidance.for_concepts(2, [3.0, 2.0], [False, True], [0.9, 0.5], None, 1, use_cross_attn_mask=True,
                                                                     edit_token_counts=[3, 1]), c_edit=c_edit)}
    for name, kw in noop.items():
        assert torch.equal(run(**kw), plain), name
    for name, kw in active.items():
        out = run(**kw)
        assert bool(torch.isfinite(out).all()) and not torch.equal(out, plain), name
        assert torch.equal(run(mask=m, **kw)[outside], x0[outside]), name
    unet.engine.set_mma_mode(0)
    try:
        plain0 = run()
        sega0 = run(semantic=SemanticGuidance.for_concepts(2, 0.0), c_edit=c_edit)
    finally:
        unet.engine.set_mma_mode(1)
    assert torch.equal(sega0, plain0)


def test_rejections(eng, unet):
    """What the loop cannot honour is CDX_E_INVALID at the C ABI, and an attention control with concepts is a ValueError"""
    from cycle_diffusion_b200.attn_control import PnPControl
    from cycle_diffusion_b200.engine import _ptr
    from cycle_diffusion_b200.semantic import SemanticGuidance
    sched = EditFriendlySchedule(6, 2)
    n = sched.refine_steps
    x0, c_src, c_tgt, uc, c_edit, noise = _inputs(n)
    xd, cs, ct, ud, nd = (t.cuda().contiguous() for t in (x0, c_src, c_tgt, uc, noise))
    out = torch.empty_like(xd)

    def raw(mutate=None, sampler=True):
        sp, keep = sched.sampler_struct()
        if mutate:
            mutate(sp, keep)
        return _cabi.lib.cdx_cycle_lockstep_sampler(unet.h, _ptr(xd), _ptr(cs), _ptr(ct), _ptr(ud), L, 1.0, 3.0, sched.coef_array(),
                                                    sched.t_array(), n, _ptr(nd), sched.sqrt_a_T, sched.sqrt_1ma_T, _ptr(out), None, B, 4, 16,
                                                    16, eng.stream, C.byref(sp) if sampler else None, None, None, None, None, None, None,
                                                    None, None)
    assert raw() == 0
    assert raw(sampler=False) == -1

    bad = [lambda sp, k: setattr(sp, 'kind', 3), lambda sp, k: setattr(sp, 'kind', -1),
           lambda sp, k: k[2][0].__setattr__('order', 2), lambda sp, k: k[2][1].__setattr__('order', 3),
           lambda sp, k: k[2][2].__setattr__('n', 0.0), lambda sp, k: k[0].__setitem__(0, k[0][0] * 1.5),
           lambda sp, k: k[1].__setitem__(0, 0.5), lambda sp, k: setattr(sp, 'qa', None), lambda sp, k: setattr(sp, 'dpm', None)]
    for i, fn in enumerate(bad):
        assert raw(fn) == -1, i
    assert raw() == 0
    with pytest.raises(ValueError):
        unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, semantic=SemanticGuidance.for_concepts(2, 1.0), c_edit=c_edit,
                            attn_control=PnPControl())


@pytest.mark.parametrize('inversion', ['ddpm', 'dpmsolver++'])
def test_pipeline_routes_to_the_loop(eng, inversion):
    """The pipeline's latents under inversion= equal UNet.cycle_lockstep under the EditFriendlySchedule, fed as the pipeline feeds it
    (the same generator draws as 'cycle'); 'cycle' with eta=None is 'cycle' at eta 0.1"""
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    g = _generator(eng)
    pipe = CycleDiffusionPipeline(g)
    image = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(4))
    kw = dict(strength=0.75, num_inference_steps=8, guidance_scale=3.0)
    lat = {}

    def run(tag, **extra):
        pipe(['a dog'] * 2, ['a cat'] * 2, image, generator=torch.Generator().manual_seed(9), callback=lambda i, t, x: lat.__setitem__(tag, x),
             **kw, **extra)
    run('ef', inversion=inversion)
    run('ef_eta1', inversion=inversion, eta=1.0)
    run('cycle_default')
    run('cycle_01', eta=0.1)
    gen = torch.Generator().manual_seed(9)
    c_tgt, c_src, uc = (g.get_learned_conditioning([p] * 2) for p in ('a dog', 'a cat', ''))
    sched = EditFriendlySchedule(8, 8 - 6, g.alphas_cumprod, solver=inversion)
    mom = g.encode_first_stage(eng.shift_scale(image, -0.5, 2.0))
    x0 = eng.vae_posterior(mom, torch.randn(2, 4, 16, 16, generator=gen), g.scale_factor)
    noise = torch.zeros(sched.refine_steps + 1, 2, 4, 16, 16)
    noise[0] = torch.randn(2, 4, 16, 16, generator=gen)
    for i in range(sched.refine_steps - 1):
        noise[1 + i] = torch.randn(2, 4, 16, 16, generator=gen)
    ref = g.unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1, 3.0, sched, noise)
    assert torch.equal(lat['ef'], ref) and torch.equal(lat['ef_eta1'], ref)
    assert torch.equal(lat['cycle_default'], lat['cycle_01']) and not torch.equal(lat['cycle_default'], ref)
