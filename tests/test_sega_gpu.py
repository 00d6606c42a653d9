"""Semantic guidance on the lock-step loop (cdx_cycle_lockstep_semantic, cdx_op_latent_chains stages 1 and 2): the threshold stage
and the step's concept terms bit for bit against tests/sega_oracle.py and tests/step_oracle.py, the no-op settings, the loop against
the CPU SEGA oracle, composition with a mask, the rejections, and the pipeline's routing."""
import itertools

import pytest
import torch

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.semantic import SemanticGuidance
from cycle_diffusion_b200.wrappers import encode_noise
from tests import step_oracle as so
from tests.common import NARROW, VAE_SMALL, maxdiff
from tests.sega_oracle import plane_thresholds, sega_cycle
from tests.test_step_kernels_gpu import GUARD, NAN, STEPS, SA_V, S1_V, chain_table, mask_of, same

pytestmark = pytest.mark.gpu

B, L = 2, 77


@pytest.fixture(scope='module')
def eng():
    from cycle_diffusion_b200.engine import Engine
    return Engine(0)


@pytest.fixture
def mode(eng):
    yield eng.set_mma_mode
    eng.set_mma_mode(1)


# ================================================================================================ one launch
def guarded(n, value=None, g=None):
    full = torch.full((n + 2 * GUARD,), NAN)
    if value is None:
        full[GUARD: GUARD + n] = torch.randn(n, generator=g)
    elif value is not NAN:
        full[GUARD: GUARD + n] = value
    return full


def inner(buf, n):
    return buf[GUARD: GUARD + n]


def layout(n_src, K, m, kind, shuffle, seed):
    """chain table and concept rows in the drivers' layout, renumbered together when shuffle"""
    chains, rows = chain_table(n_src, K, True, kind, False, seed)
    sg_rows = list(range(rows, rows + n_src * K * m))
    total = rows + n_src * K * m
    if shuffle:
        perm = torch.randperm(total, generator=torch.Generator().manual_seed(seed)).tolist()
        chains = [(perm[r], perm[r2] if r2 >= 0 else -1, s) for r, r2, s in chains]
        sg_rows = [perm[r] for r in sg_rows]
    return chains, sg_rows, total


def eout_values(rows, chw, hw, g, chains, sg_rows, n_src, K, m):
    """U-Net outputs with ties: values on a 1/8 grid, one concept row equal to its chain's uncond row (all-zero terms) and one its
    uncond row plus a constant (a constant plane)"""
    e = torch.round(torch.randn(rows * chw, generator=g) * 8) / 8
    for t in range(n_src * K):
        r, r2, _ = chains[n_src + t]
        ru = r2 if r2 >= 0 else r
        if m >= 2 and t % 2 == 0:
            e[sg_rows[t * m + 1] * chw: (sg_rows[t * m + 1] + 1) * chw] = e[ru * chw: (ru + 1) * chw]
        if m >= 3 and t % 3 == 0:
            e[sg_rows[t * m + 2] * chw: (sg_rows[t * m + 2] + 1) * chw] = e[ru * chw: (ru + 1) * chw] + 0.375
    return e


def oracle_thresholds(eout, chains, sg_rows, n_src, K, m, C, hw, scales, lambdas):
    chw = C * hw
    out = []
    for t in range(n_src * K):
        r, r2, _ = chains[n_src + t]
        ou = eout[(r2 if r2 >= 0 else r) * chw:][:chw]
        for k in range(m):
            ok = eout[sg_rows[t * m + k] * chw:][:chw]
            a = (so.f(scales[k]) * (ok - ou)).abs()
            out.append(plane_thresholds(a.reshape(1, C, hw, 1), lambdas[k]).reshape(C))
    return torch.cat(out)


PLANES = [(4, 4), (16, 24), (40, 24), (64, 64), (96, 96), (120, 120)]


@pytest.mark.parametrize('h,w', PLANES)
def test_threshold_stage_bit_exact(eng, h, w):
    """Stage 2 against the oracle's sort-and-lerp, bit for bit, every threshold in its guarded buffer: ties, all-zero and constant
    planes, zero and negative scales, lambda 0 / 0.5 / 0.9 / 0.999, target chains on one row (scale 0 or 1) and on two, in the
    drivers' row layout and renumbered."""
    C, n_src, K = 4, 2, 2
    hw, chw = h * w, 4 * h * w
    for n, (m, kind, shuffle) in enumerate(itertools.product((1, 3), ('cfg', 'mixed'), (False, True))):
        g = torch.Generator().manual_seed(n + hw)
        chains, sg_rows, rows = layout(n_src, K, m, kind, shuffle, n)
        scales = [2.5, -1.0, 0.0][:m] if m > 1 else [-3.0]
        lambdas = [0.9, 0.0, 0.999][:m] if n % 2 else [0.5, 0.9, 0.0][:m]
        eout = eout_values(rows, chw, hw, g, chains, sg_rows, n_src, K, m)
        n_thr = n_src * K * m * C
        want = oracle_thresholds(eout, chains, sg_rows, n_src, K, m, C, hw, scales, lambdas)
        thr = guarded(n_thr, NAN).cuda()
        ed = eout.cuda()
        eng.op_latent_chains(2, chains, chw, n_src, K, rows, src=1, eout=ed, hw=hw, sg_rows=sg_rows, sg_thr=inner(thr, n_thr),
                             sg_scale=scales, sg_lambda=lambdas)
        torch.cuda.synchronize()
        full = torch.full((n_thr + 2 * GUARD,), NAN)
        full[GUARD: GUARD + n_thr] = want
        assert same(thr.cpu(), full), f'{h}x{w} m={m} {kind} shuffle={shuffle}'


def sega_oracle_step(views, meta, sc, sg):
    """step_oracle.latent_step with each target chain's eps-hat plus its concept term G, then its concept rows and momentum"""
    n_src, K, chw = meta['n_src'], meta['K'], meta['chw']
    chains, m, hw = meta['chains'], len(sg['sg_scale']), sc['hw']
    C = chw // hw
    eout, thr, nu = views['eout'], views['sg_thr'], views['sg_nu']
    G_of = {}
    for t in range(n_src * K):
        r, r2, _ = chains[n_src + t]
        ou = eout[(r2 if r2 >= 0 else r) * chw:][:chw]
        S = None
        for k in range(m):
            ok = eout[sg['sg_rows'][t * m + k] * chw:][:chw]
            psi = so.f(sg['sg_scale'][k]) * (ok - ou)
            theta = thr[(t * m + k) * C:][:C].repeat_interleave(hw)
            keep = (psi.abs() >= theta) & bool((sg['sg_active'] >> k) & 1)
            gk = torch.where(keep, psi, torch.zeros_like(psi))
            S = gk if S is None else S + gk
        v = nu[t * chw:][:chw]
        G = S + so.f(sg['sg_mu']) * v
        v.copy_(so.f(sg['sg_beta']) * v + so.f(sg['sg_beta1']) * G)
        G_of[tuple(chains[n_src + t])] = G
    plain = so._eps_hat

    def eps_hat(e, ch, n):
        o = plain(e, ch, n)
        G = G_of.get(tuple(ch)) if ch in chains[n_src:] else None
        return o + G if G is not None and sg['sg_apply'] else o
    so._eps_hat = eps_hat
    try:
        so.latent_step(**meta, **sc, **views)
    finally:
        so._eps_hat = plain
    for t in range(n_src * K):
        for k in range(m):
            views['xin'][sg['sg_rows'][t * m + k] * chw:][:chw].copy_(views['y_out'][t * chw:][:chw])


STEP_CASES = [(pred, masked) for pred in (0, 1) for masked in (False, True)]


@pytest.mark.parametrize('pred,masked', STEP_CASES)
def test_step_bit_exact(eng, pred, masked):
    """Every new latent_chains_step<PRED, MASK, 1> instantiation: m = 1, 2, 3 with negative and zero scales; per-concept activity
    and the warmup flag on and off; target scales 0, 1 and 7.5 on one and two rows; three consecutive launches on one momentum
    buffer, every buffer guarded and compared bit for bit after each launch, in the drivers' layout and renumbered."""
    n_src, K, C, h, w = 3, 2, 4, 3, 5
    hw, chw = h * w, C * h * w
    for n, (m, kind, shuffle) in enumerate(itertools.product((1, 2, 3), ('cfg', 'pick', 'mixed'), (False, True))):
        g = torch.Generator().manual_seed(500 + n)
        chains, sg_rows, rows = layout(n_src, K, m, kind, shuffle, n)
        scales = [[1.5], [-2.0, 0.75], [3.0, 0.0, -1.25]][m - 1]
        lambdas = [[0.9], [0.5, 0.0], [0.999, 0.3, 0.9]][m - 1]
        nsrc = n_src * chw
        bufs = {'x0': guarded(nsrc, g=g), 'noise_next': guarded(nsrc, g=g), 'z_out': guarded(n_src * 3 * chw, NAN),
                'eout': guarded(rows * chw, eout_values(rows, chw, hw, g, chains, sg_rows, n_src, K, m)),
                'xt': guarded(nsrc, g=g), 'xn': guarded(nsrc, g=g), 'xn2': guarded(nsrc, NAN), 'yt': guarded(nsrc * K, g=g),
                'y_out': guarded(nsrc * K, NAN), 'xin': guarded(rows * chw, NAN), 'sg_nu': guarded(n_src * K * chw, 0.0)}
        if masked:
            bufs['mask'] = guarded(n_src * hw, mask_of('random', n_src, hw, n))
        n_thr = n_src * K * m * C
        views = lambda b: {k: b[k][GUARD: GUARD + (len(b[k]) - 2 * GUARD)] for k in b}
        thr_host = oracle_thresholds(inner(bufs['eout'], rows * chw), chains, sg_rows, n_src, K, m, C, hw, scales, lambdas)
        bufs['sg_thr'] = guarded(n_thr, thr_host)
        meta = dict(chains=chains, chw=chw, n_src=n_src, K=K, rows=rows)
        dev = {k: v.cuda() for k, v in bufs.items()}
        host = {k: v.clone() for k, v in bufs.items()}
        for launch in range(3):
            sched, i = STEPS[(n + launch) % len(STEPS)]
            c, cn = sched.coef[i], sched.coef[min(i + 1, sched.refine_steps - 1)]
            t = int(sched.t_loop[i])
            sc = dict(src=1, c=c, cnext=cn, next=1 + launch % 2, pred=pred, vsa=float(SA_V[t]), vs1=float(S1_V[t]), z_stride=3 * chw,
                      hw=hw)
            sg = dict(sg_rows=sg_rows, sg_scale=scales, sg_lambda=lambdas, sg_active=[0b111, 0b101, 0b010][launch],
                      sg_apply=launch != 1, sg_mu=0.3, sg_beta=0.4, sg_beta1=float(torch.tensor(1 - 0.4, dtype=torch.float32)))
            hv = views(host)
            sega_oracle_step(hv, meta, sc, sg)
            dv = views(dev)
            eng.op_latent_chains(1, **meta, **sc, **dv, **{k: (int(v) if k in ('sg_active', 'sg_apply') else v) for k, v in sg.items()})
            torch.cuda.synchronize()
            for name in bufs:
                assert same(dev[name].cpu(), host[name]), f'{name} after launch {launch}: m={m} {kind} shuffle={shuffle}'


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


@pytest.fixture(scope='module')
def sched():
    from cycle_diffusion_b200.schedule import DDIMSchedule
    return DDIMSchedule(6, 0.1, 2)


def _inputs(sched, h=16, w=16, seed=7, m=2):
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(B, 4, h, w, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(B, L, 48, generator=g) for _ in range(3))
    c_edit = torch.randn(B, m, L, 48, generator=g)
    torch.manual_seed(seed + 1)
    return x0, c_src, c_tgt, uc, c_edit, encode_noise(sched, sched.refine_steps, x0.shape)


def sg_of(scales, thresholds, cooldown, warmup, mu=0.3, beta=0.4):
    return SemanticGuidance.for_concepts(len(scales), [abs(s) for s in scales], [s < 0 for s in scales], thresholds, cooldown, warmup,
                                         mu, beta)


@pytest.mark.parametrize('mma', [1, 5, 0])
def test_no_op_settings(unet, sched, mode, mma):
    """Scale 0, warmup at or past the loop's steps, and every cooldown 0 give one output bit for bit.  Against the plain loop (no
    concept rows) the output and z stay within rel 1e-6: the extra rows share the fp16-split operands' one exponent per tensor."""
    mode(mma)
    x0, c_src, c_tgt, uc, c_edit, noise = _inputs(sched)
    n = sched.refine_steps
    outs = []
    for sg in (sg_of([0.0, -0.0], [0.9, 0.5], [None, None], 0), sg_of([3.0, -2.0], [0.9, 0.0], [None, None], n),
               sg_of([3.0, -2.0], [0.9, 0.0], [0, 0], 0)):
        outs.append(unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, semantic=sg, c_edit=c_edit))
    for o, z in outs[1:]:
        assert torch.equal(o, outs[0][0]) and torch.equal(z, outs[0][1])
    plain, zp = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True)
    ro = maxdiff(outs[0][0].cpu(), plain.cpu()) / float(plain.abs().max())
    rz = maxdiff(outs[0][1].cpu(), zp.cpu()) / float(zp.abs().max())
    print(f'mode {mma}: no-op SEGA vs plain loop rel|dx| {ro:.2e} rel|dz| {rz:.2e} bit-identical {ro == 0 and rz == 0}')
    # The target's guided output at scale 3 is e_uc + 3 (e_c - e_uc), which scales a per-row difference by up to 1 + 2 * 3.
    # Mode 1 (fp16-split): z within rel 1e-6, the latent within 7e-6.  Mode 5 (single-term fp16): the shared exponent moves the
    # rounding of every fp16 operand, so z stays within fp16's unit roundoff 2^-11 and the latent within 7 times it.  Mode 0 (exact
    # fp32 FFMA): the GEMM and attention partitions do not depend on the row count, so the outputs are the plain loop's bit for bit.
    if mma == 1:
        assert rz < 1e-6 and ro < 1e-6 * (1 + 2 * 3.0)
    elif mma == 5:
        assert rz < 2.0 ** -11 and ro < 2.0 ** -11 * (1 + 2 * 3.0)
    else:
        assert ro == 0 and rz == 0
    on = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, semantic=sg_of([3.0, -2.0], [0.9, 0.0], [None, 1], 1),
                             c_edit=c_edit)
    assert not torch.equal(on, outs[0][0])


ORACLE_CASES = [(pred, s, t, lam) for pred in ('eps', 'v') for s in (1.0, 2.0) for t in (1.0, 3.0) for lam in (0.0, 0.9)]
# seed 11 unless its oracle thresholds come within 1e-4 of a value they compare (the margin the test asserts): then the first seed
# that keeps it
SEEDS = {('eps', 1.0, 1.0, 0.9): 37, ('v', 1.0, 1.0, 0.9): 17}


@pytest.mark.parametrize('pred,src_scale,tgt_scale,lam', ORACLE_CASES)
def test_vs_sega_oracle(unet, usd, sched, with_prediction, pred, src_scale, tgt_scale, lam):
    """Engine against the CPU SEGA oracle within the PnP / mutual oracle bounds, the edit more than 10x the bound.  At lambda 0.9
    the oracle's thresholds sit more than 1e-4 (relative) from every value they compare, so no pass rests on a threshold landing
    inside the engine-oracle difference."""
    from oracle import unet_openai
    with_prediction(pred)
    seed = SEEDS.get((pred, src_scale, tgt_scale, lam), 11)
    x0, c_src, c_tgt, uc, c_edit, noise = _inputs(sched, seed=seed)
    sg = sg_of([2.0, -1.5], [lam, lam], [None, 3], 1)
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise, return_z=True, semantic=sg, c_edit=c_edit)
    plain = unet.cycle_lockstep(x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise)
    torch.manual_seed(seed + 1)                                                # the seed _inputs drew the noise under
    stats = {}
    fn = lambda x, t, c: unet_openai.unet_forward(usd, NARROW, x, t, c)
    with torch.no_grad():
        y_ref, z_ref = sega_cycle(fn, x0, c_src, c_tgt, uc, c_edit, 6, 0.1, 2, src_scale, tgt_scale, list(sg.signed_scales()),
                                  [lam, lam], [4, 3], 1, 0.3, 0.4, prediction=pred, stats=stats)
    z_ref = torch.stack(z_ref, dim=1)
    rz = maxdiff(z.cpu(), z_ref) / float(z_ref.abs().max())
    dx = maxdiff(out.cpu(), y_ref)
    dc = maxdiff(out.cpu(), plain.cpu())
    print(f'sega {pred} scales ({src_scale}, {tgt_scale}) lambda {lam}: rel|dz| {rz:.2e} |dx| {dx:.2e} |x - plain x| {dc:.2e} '
          f'threshold margin {stats["margin"]:.2e} over {stats["planes"]} planes')
    assert rz < 2e-4 and dx < 1e-3
    assert dc > 10 * dx
    if lam > 0:
        assert stats['margin'] > 1e-4


def test_composes_with_a_mask(unet, sched):
    """Box mask plus concepts: outside the box the latent is x0 bit for bit; inside it differs from the masked edit without them."""
    x0, c_src, c_tgt, uc, c_edit, noise = _inputs(sched)
    m = torch.zeros(B, 1, 16, 16)
    m[..., 4:12, 4:12] = 1.0
    sg = sg_of([3.0, -2.0], [0.9, 0.5], [None, None], 1)
    out = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=m, semantic=sg, c_edit=c_edit).cpu()
    masked = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=m).cpu()
    inside = m.expand_as(x0) == 1
    assert torch.equal(out[~inside], x0[~inside]) and not torch.equal(out[inside], masked[inside])


def test_rejections(eng, unet, sched):
    """What the engine cannot honour raises, at the C ABI (past the Python checks) and in Python."""
    import ctypes as C
    from cycle_diffusion_b200 import _cabi
    from cycle_diffusion_b200.attn_control import PnPControl
    from cycle_diffusion_b200.engine import UNet, _ptr
    x0, c_src, c_tgt, uc, c_edit, noise = _inputs(sched)
    sg = sg_of([3.0, -2.0], [0.9, 0.5], [None, None], 1)
    n = sched.refine_steps
    xd, cs, ct, ud, ce, nd = (t.cuda().contiguous() for t in (x0, c_src, c_tgt, uc, c_edit, noise))
    out = torch.empty_like(xd)

    def raw(s, uc_ptr=ud, ctx=ce):
        return _cabi.lib.cdx_cycle_lockstep_semantic(unet.h, _ptr(xd), _ptr(cs), _ptr(ct), _ptr(uc_ptr), L, 1.0, 3.0, sched.coef_array(),
                                                     sched.t_array(), n, _ptr(nd), sched.sqrt_a_T, sched.sqrt_1ma_T, _ptr(out), None, B, 4,
                                                     16, 16, eng.stream, None, _ptr(ctx), C.byref(s) if s is not None else None)
    assert raw(sg.c_struct(n)) == 0
    for field, value in (('m', 0), ('m', 9), ('threshold', 1.0), ('threshold', -0.5), ('threshold', float('nan'))):
        s = sg.c_struct(n)
        if field == 'm':
            s.m = value
        else:
            s.threshold[1] = value
        assert raw(s) == -1, (field, value)
    assert raw(sg.c_struct(n), uc_ptr=None) == -1                  # no uncond row to take the terms against
    assert raw(None) == -1 and raw(sg.c_struct(n), ctx=None) == -1
    with pytest.raises(ValueError):
        unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, semantic=sg, c_edit=c_edit, attn_control=PnPControl())
    with pytest.raises(ValueError):
        unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, semantic=sg, c_edit=c_edit[:, :1])
    # a context-free LDM U-Net
    cfg = dict(in_channels=4, out_channels=4, model_channels=32, attention_resolutions=(2, 4), num_res_blocks=1, channel_mult=(1, 2, 2),
               num_head_channels=16, context_dim=0)
    plain_net = UNet(eng, cfg, 'openai').load_state_dict(specs.synth_state_dict(specs.openai_unet_params(cfg), 41))
    ctx = torch.zeros(B, 1, 1)
    with pytest.raises(AssertionError):
        plain_net.cycle_lockstep(x0, ctx, ctx, ctx, 1.0, 3.0, sched, noise, semantic=sg, c_edit=torch.zeros(B, 2, 1, 1))
    # more rows than the GroupNorm statistics pool serves in one call: an error, not a fault
    nb, m = 96, 8
    g = torch.Generator().manual_seed(3)
    xb = torch.randn(nb, 4, 16, 16, generator=g)
    cb = torch.randn(nb, L, 48, generator=g)
    big = SemanticGuidance.for_concepts(m, 1.0)
    with pytest.raises(AssertionError, match='statistics'):
        unet.cycle_lockstep(xb, cb, cb, cb, 1.0, 3.0, sched, torch.randn(n + 1, nb, 4, 16, 16, generator=g), semantic=big,
                            c_edit=torch.randn(m, L, 48, generator=g))
    # the engine still runs afterwards
    assert torch.equal(unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, semantic=sg, c_edit=c_edit), out)


def _generator(eng):
    from cycle_diffusion_b200.wrappers import SDStochasticTextWrapper, SyntheticTextEncoder
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    vsd = specs.synth_state_dict(specs.kl_vae_params(VAE_SMALL), 21)
    sd = {'model.diffusion_model.' + k: v for k, v in usd.items()}
    sd.update({'first_stage_model.' + k: v for k, v in vsd.items()})
    w = SDStochasticTextWrapper('synthetic', engine=eng, state_dict=sd, cond_stage=SyntheticTextEncoder(48), unet_config=NARROW,
                                vae_config=VAE_SMALL, latent_size=16, resolution=128, custom_steps=4, eta=0.1, white_box_steps=5,
                                skip_steps=[0], encoder_unconditional_guidance_scales=[1], decoder_unconditional_guidance_scales=[3.0],
                                n_trials=1)
    return w.generator


@pytest.mark.parametrize('variant', ['plain', 'per_prompt2', 'auto_mask', 'autocast'])
def test_pipeline_routes_to_the_loop(eng, mode, variant):
    """The pipeline's latents equal UNet.cycle_lockstep(..., semantic=...) fed as the pipeline feeds it, exactly; without
    editing_prompt they are the plain loop's.  Two-phase and an attention edit_type are rejected."""
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    from cycle_diffusion_b200.schedule import DDIMSchedule
    g = _generator(eng)
    precision = 'autocast' if variant == 'autocast' else 'full'
    pipe = CycleDiffusionPipeline(g, precision=precision)
    image = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(4))
    per = 2 if variant == 'per_prompt2' else 1
    kw = dict(strength=0.75, num_inference_steps=8, guidance_scale=3.0, eta=0.1, num_images_per_prompt=per)
    edit = dict(editing_prompt=['glasses', 'a hat'], reverse_editing_direction=[False, True], edit_guidance_scale=[4.0, 2.0],
                edit_threshold=[0.8, 0.5], edit_cooldown_steps=[None, 4], edit_warmup_steps=1, edit_momentum_scale=0.2, edit_mom_beta=0.5)
    mask_arg = 'auto' if variant == 'auto_mask' else None
    lat = {}

    def run(tag, **extra):
        cb = lambda i, t, x: lat.__setitem__(tag, x)
        pipe(['a dog'] * 2, ['a cat'] * 2, image, generator=torch.Generator().manual_seed(9), callback=cb, mask_image=mask_arg, **kw, **extra)
    run('plain')
    run('sega', **edit)
    Bn = 2 * per
    gen = torch.Generator().manual_seed(9)
    mask = None
    if mask_arg == 'auto':
        mask = pipe.generate_mask(image, 'a cat', 'a dog', generator=gen, num_inference_steps=8)
    img = image.repeat_interleave(per, dim=0)
    with eng.precision(precision):
        if mask is not None:
            mask = eng.mask_pool(mask.repeat_interleave(per, dim=0).contiguous(), g.vae.down)
        c_tgt, c_src, uc = (g.get_learned_conditioning([p] * Bn) for p in ('a dog', 'a cat', ''))
        c_edit = g.get_learned_conditioning(['glasses', 'a hat'])
        sched = DDIMSchedule(8, 0.1, 8 - 6, g.alphas_cumprod)
        mom = g.encode_first_stage(eng.shift_scale(img, -0.5, 2.0))
        x0 = eng.vae_posterior(mom, torch.randn(Bn, 4, 16, 16, generator=gen), g.scale_factor)
        noise = torch.zeros(sched.refine_steps + 1, Bn, 4, 16, 16)
        noise[0] = torch.randn(Bn, 4, 16, 16, generator=gen)
        for i in range(sched.refine_steps - 1):
            noise[1 + i] = torch.randn(Bn, 4, 16, 16, generator=gen)
        sg = SemanticGuidance.for_concepts(2, [4.0, 2.0], [False, True], [0.8, 0.5], [None, 4], 1, 0.2, 0.5)
        ref = g.unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1, 3.0, sched, noise, mask=mask, semantic=sg, c_edit=c_edit)
        ref_plain = g.unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1, 3.0, sched, noise, mask=mask)
    assert torch.equal(lat['sega'], ref) and torch.equal(lat['plain'], ref_plain) and not torch.equal(ref, ref_plain)
    if variant == 'plain':
        call = lambda **k: pipe('a dog', 'a cat', image, num_inference_steps=4, editing_prompt='glasses', **k)
        for extra in (dict(two_phase=True), dict(cross_attention_kwargs={'edit_type': 'pnp'}), dict(edit_warmup_steps=[1]),
                      dict(edit_threshold=[0.5, 0.5])):
            with pytest.raises(ValueError):
                call(**extra)
