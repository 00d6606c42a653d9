"""LEDITS++'s implicit masks on the semantic-guidance loop (cdx_cycle_lockstep_semantic_attn): the cross-attention probe against
float64 on every attention route through cdx_op_attention_net, the threshold stage and the step kernel bit for bit against
tests/ledits_oracle.py, lambda = 0 against SEGA, the loop against the CPU oracle, composition, rejections and the pipeline."""
import itertools
import math

import pytest
import torch

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.semantic import SemanticGuidance
from tests import step_oracle as so
from tests.common import NARROW, WIDE, maxdiff
from tests.ledits_oracle import channel_sum, ledits_cycle, smooth
from tests.sega_oracle import quantile
from tests.test_sega_gpu import _generator, _inputs, eout_values, guarded, inner, layout
from tests.test_step_kernels_gpu import GUARD, NAN, STEPS, SA_V, S1_V, mask_of, same

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


# ================================================================================================ the probe
# representation error of the probed K (and q on the TF32 planes) relative to the fp32 operands, per route: fp32 operands exact; the
# fp16 hi + lo split keeps 22 bits; TF32 hi + lo 21 bits per operand; the one-term hi plane fp16's 11 bits
REP = {'generic': 0.0, 'unfused_tc': 0.0, 'fused_h16': 2.0 ** -21, 'fused_tf32': 2.0 ** -20, 'fused_one': 2.0 ** -10}
GRIDS = [(2, 2), (4, 6), (5, 3), (8, 8), (30, 30)]
PROBE_CASES = [(m, d) for m in (0, 1, 3, 4, 5) for d in (40, 64, 80, 160)]


def probe_bound(q, k, heads, span, rep, P):
    """Elementwise bound on the probe's map for one image, float64.  Logit s_j = scale * q.k_j: the operands' representation error
    plus the fp32 dot (d products, d - 1 adds) and the scale multiply give |ds_j| <= Delta = scale * max_j sum_c |q_c k_jc| *
    (rep + (d + 2) u), u = 2^-24; a shift of every logit by at most Delta moves a span ratio P by at most P (e^(2 Delta) - 1).
    Evaluating P in fp32 (L exponentials within 2 ulp, two sums of at most L terms, one division) adds P * 2 (L + 3) * 2u, and the
    sum over heads heads * u * sum P.  Twice that sum."""
    N, C = q.shape
    d = C // heads
    u = 2.0 ** -24
    scale = d ** -0.5
    total = torch.zeros(N, dtype=torch.float64)
    for h in range(heads):
        qa, ka = q[:, h * d:(h + 1) * d].abs(), k[:, h * d:(h + 1) * d].abs()
        delta = scale * (qa @ ka.T).amax(dim=-1) * (rep + (d + 2) * u)
        total += P[h] * (torch.expm1(2 * delta) + 2 * (L + 3) * 2 * u)
    return 2 * (total + heads * u * P.sum(dim=0))


@pytest.mark.parametrize('mma,d', PROBE_CASES)
def test_probe_vs_float64(eng, mode, mma, d):
    """The map of every listed row against a float64 softmax of the layer's fp32 q and K, within the derived bound, on each grid;
    spans 1 and L - 2, rows listed shuffled; the map's guards stay NaN, and the attention output is the one without the probe,
    bit for bit."""
    mode(mma)
    heads = 8 if d == 40 else 2
    C, nimg, Lp = heads * d, 3, 80
    for gi, (gh, gw) in enumerate(GRIDS):
        N = gh * gw
        g = torch.Generator().manual_seed(1000 * mma + 10 * d + gi)
        q = torch.randn(nimg * N, C, generator=g) * 1.5
        kv = torch.zeros(nimg * Lp, 2 * C)
        for b in range(nimg):
            kv[b * Lp: b * Lp + L] = torch.randn(L, 2 * C, generator=g)
        rows, spans = [2, 0, 1, 2], [1, L - 2, 5, L - 2]
        qd, kvd = q.cuda(), kv.cuda()
        out0 = torch.empty(nimg * N, C, device='cuda')
        out1 = torch.empty(nimg * N, C, device='cuda')
        n = len(rows) * N
        mp = guarded(n, NAN).cuda()
        plan = eng.op_attention_net('cross', out0, nimg, N, heads, d, d ** -0.5, q=qd, kv=kvd, L=L, ctx_lp=Lp)
        eng.op_attention_net('cross', out1, nimg, N, heads, d, d ** -0.5, q=qd, kv=kvd, L=L, ctx_lp=Lp, probe_rows=rows, probe_spans=spans,
                             probe_map=inner(mp, n))
        torch.cuda.synchronize()
        assert torch.equal(out0, out1)
        got = mp.cpu()
        assert torch.isnan(got[:GUARD]).all() and torch.isnan(got[GUARD + n:]).all()
        got = inner(got, n).reshape(len(rows), N).double()
        worst = 0.0
        for i, (b, sp) in enumerate(zip(rows, spans)):
            qb = q[b * N:(b + 1) * N].double()
            kb = kv[b * Lp: b * Lp + L, :C].double()
            P = torch.stack([torch.softmax(qb[:, h * d:(h + 1) * d] @ kb[:, h * d:(h + 1) * d].T * d ** -0.5, dim=-1)[:, 1:1 + sp].sum(-1)
                             for h in range(heads)])
            want = P.sum(dim=0)
            bound = probe_bound(qb, kb, heads, sp, REP[plan['route']], P)
            err = (got[i] - want).abs()
            assert (err <= bound).all(), f'row {b} span {sp} {gh}x{gw}: {float((err / bound).max()):.2f} of the bound'
            worst = max(worst, float((err / bound).max()))
        print(f'mode {mma} d {d} {gh}x{gw} route {plan["route"]}: worst error {worst:.3f} of the bound')


# ================================================================================================ one launch
def map_values(n_rows, gh, gw, g):
    """raw maps on a 1/8 grid (ties), one row constant"""
    A = torch.round(torch.rand(n_rows, gh * gw, generator=g) * 16) / 8
    A[0] = 0.625
    return A


def oracle_mask_thresholds(eout, amap, chains, sg_rows, n_src, K, m, C, h, w, scales, lambdas, gh, gw):
    chw = C * h * w
    out = []
    for t in range(n_src * K):
        r, r2, _ = chains[n_src + t]
        ou = eout[(r2 if r2 >= 0 else r) * chw:][:chw]
        for k in range(m):
            tq = t * m + k
            As = smooth(amap[tq].reshape(gh, gw))
            ok = eout[sg_rows[tq] * chw:][:chw]
            s = channel_sum((so.f(scales[k]) * (ok - ou)).reshape(1, C, h, w))
            out += [quantile(As.reshape(1, -1), lambdas[k]).reshape(1), quantile(s.reshape(1, -1), lambdas[k]).reshape(1)]
    return torch.cat(out)


@pytest.mark.parametrize('gh,gw', [(2, 2), (4, 6), (8, 8), (30, 30)])
def test_threshold_stage_bit_exact(eng, gh, gw):
    """Stage 2 in both mask modes against the oracle's smoothing and sort-and-lerp, bit for bit in guarded buffers: ties, constant
    maps and an all-zero term, lambda 0 / 0.5 / 0.9 / 0.999, in the drivers' row layout and renumbered.  Mode 1 leaves the
    channel-sum slots untouched."""
    C, n_src, K = 4, 2, 2
    h, w = 4 * gh, 4 * gw
    hw, chw = h * w, C * h * w
    for n, (m, kind, shuffle, sm) in enumerate(itertools.product((1, 3), ('cfg', 'mixed'), (False, True), (1, 2))):
        g = torch.Generator().manual_seed(n + hw)
        chains, sg_rows, rows = layout(n_src, K, m, kind, shuffle, n)
        scales = [2.5, -1.0, 0.0][:m] if m > 1 else [-3.0]
        lambdas = [0.9, 0.0, 0.999][:m] if n % 2 else [0.5, 0.9, 0.999][:m]
        eout = eout_values(rows, chw, hw, g, chains, sg_rows, n_src, K, m)
        nr = n_src * K * m
        amap = map_values(nr, gh, gw, g)
        want = oracle_mask_thresholds(eout, amap, chains, sg_rows, n_src, K, m, C, h, w, scales, lambdas, gh, gw)
        if sm == 1:
            want[1::2] = NAN
        thr = guarded(2 * nr, NAN).cuda()
        mapd = amap.reshape(-1).cuda()
        eng.op_latent_chains(2, chains, chw, n_src, K, rows, src=1, eout=eout.cuda(), hw=hw, sg_rows=sg_rows, sg_thr=inner(thr, 2 * nr),
                             sg_scale=scales, sg_lambda=lambdas, sg_mask=sm, sg_map=mapd, sg_gh=gh, sg_gw=gw, w=w)
        torch.cuda.synchronize()
        full = torch.full((2 * nr + 2 * GUARD,), NAN)
        full[GUARD: GUARD + 2 * nr] = want
        assert same(thr.cpu(), full), f'{gh}x{gw} m={m} {kind} shuffle={shuffle} mode {sm}'


def ledits_oracle_step(views, meta, sc, sg, gh, gw, w, intersect):
    """step_oracle.latent_step with each target chain's eps-hat plus its masked concept term G, then its concept rows and momentum"""
    n_src, K, chw = meta['n_src'], meta['K'], meta['chw']
    chains, m, hw = meta['chains'], len(sg['sg_scale']), sc['hw']
    C, h = chw // hw, hw // w
    eout, thr, nu, amap = views['eout'], views['sg_thr'], views['sg_nu'], views['sg_map']
    G_of = {}
    for t in range(n_src * K):
        r, r2, _ = chains[n_src + t]
        ou = eout[(r2 if r2 >= 0 else r) * chw:][:chw]
        S = None
        for k in range(m):
            tq = t * m + k
            ok = eout[sg['sg_rows'][tq] * chw:][:chw]
            psi = so.f(sg['sg_scale'][k]) * (ok - ou)
            M = smooth(amap[tq * gh * gw:][:gh * gw].reshape(gh, gw)) >= thr[2 * tq]
            M = M.repeat_interleave(4, dim=0).repeat_interleave(4, dim=1)
            if intersect:
                M = M & (channel_sum(psi.reshape(1, C, h, w))[0] >= thr[2 * tq + 1])
            keep = M.reshape(-1).repeat(C) & bool((sg['sg_active'] >> k) & 1)
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
        so.latent_step(**meta, **sc, **{k: v for k, v in views.items() if k != 'sg_map'})
    finally:
        so._eps_hat = plain
    for t in range(n_src * K):
        for k in range(m):
            views['xin'][sg['sg_rows'][t * m + k] * chw:][:chw].copy_(views['y_out'][t * chw:][:chw])


@pytest.mark.parametrize('pred,masked,sm', [(p, mk, sm) for p in (0, 1) for mk in (False, True) for sm in (1, 2)])
def test_step_bit_exact(eng, pred, masked, sm):
    """Every new latent_chains_step<PRED, MASK, 2 | 3> instantiation against the oracle step: m = 1, 2, 3, per-concept activity and
    the warmup flag on and off, three consecutive launches on one momentum buffer, every buffer guarded, compared after each launch,
    in the drivers' layout and renumbered."""
    n_src, K, C, gh, gw = 2, 2, 4, 2, 3
    h, w = 4 * gh, 4 * gw
    hw, chw = h * w, C * h * w
    for n, (m, kind, shuffle) in enumerate(itertools.product((1, 2, 3), ('cfg', 'mixed'), (False, True))):
        g = torch.Generator().manual_seed(700 + n)
        chains, sg_rows, rows = layout(n_src, K, m, kind, shuffle, n)
        scales = [[1.5], [-2.0, 0.75], [3.0, 0.0, -1.25]][m - 1]
        lambdas = [[0.9], [0.5, 0.0], [0.999, 0.3, 0.9]][m - 1]
        nsrc, nr = n_src * chw, n_src * K * m
        eout = eout_values(rows, chw, hw, g, chains, sg_rows, n_src, K, m)
        amap = map_values(nr, gh, gw, g)
        bufs = {'x0': guarded(nsrc, g=g), 'noise_next': guarded(nsrc, g=g), 'z_out': guarded(n_src * 3 * chw, NAN),
                'eout': guarded(rows * chw, eout), 'xt': guarded(nsrc, g=g), 'xn': guarded(nsrc, g=g), 'xn2': guarded(nsrc, NAN),
                'yt': guarded(nsrc * K, g=g), 'y_out': guarded(nsrc * K, NAN), 'xin': guarded(rows * chw, NAN),
                'sg_nu': guarded(n_src * K * chw, 0.0), 'sg_map': guarded(nr * gh * gw, amap.reshape(-1))}
        if masked:
            bufs['mask'] = guarded(n_src * hw, mask_of('random', n_src, hw, n))
        thr = oracle_mask_thresholds(eout, amap, chains, sg_rows, n_src, K, m, C, h, w, scales, lambdas, gh, gw)
        bufs['sg_thr'] = guarded(2 * nr, thr)
        meta = dict(chains=chains, chw=chw, n_src=n_src, K=K, rows=rows)
        dev = {k: v.cuda() for k, v in bufs.items()}
        host = {k: v.clone() for k, v in bufs.items()}
        views = lambda b: {k: b[k][GUARD: GUARD + (len(b[k]) - 2 * GUARD)] for k in b}
        for launch in range(3):
            sched, i = STEPS[(n + launch) % len(STEPS)]
            c, cn = sched.coef[i], sched.coef[min(i + 1, sched.refine_steps - 1)]
            t = int(sched.t_loop[i])
            sc = dict(src=1, c=c, cnext=cn, next=1 + launch % 2, pred=pred, vsa=float(SA_V[t]), vs1=float(S1_V[t]), z_stride=3 * chw,
                      hw=hw)
            sg = dict(sg_rows=sg_rows, sg_scale=scales, sg_lambda=lambdas, sg_active=[0b111, 0b101, 0b010][launch],
                      sg_apply=launch != 1, sg_mu=0.3, sg_beta=0.4, sg_beta1=float(torch.tensor(1 - 0.4, dtype=torch.float32)))
            ledits_oracle_step(views(host), meta, sc, sg, gh, gw, w, sm == 2)
            eng.op_latent_chains(1, **meta, **sc, **views(dev), **{k: (int(v) if k in ('sg_active', 'sg_apply') else v) for k, v in sg.items()},
                                 sg_mask=sm, sg_gh=gh, sg_gw=gw, w=w)
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


def sg_of(lam, cross=False, intersect=False, tokens=(3, 1)):
    return SemanticGuidance.for_concepts(2, [2.0, 1.5], [False, True], [lam, lam], [None, 3], 1, 0.3, 0.4, cross, intersect,
                                         list(tokens) if cross or intersect else None)


@pytest.mark.parametrize('mma', [0, 1, 5])
def test_lambda_zero_is_sega(unet, sched, mode, mma):
    """At lambda = 0 every mask is all ones: the attention-mask and intersect loops equal SEGA's at lambda = 0 bit for bit, latent
    and z.  The probe runs in every step of these loops, so this also shows it changes no U-Net output."""
    mode(mma)
    x0, c_src, c_tgt, uc, c_edit, noise = _inputs(sched)
    ref = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, semantic=sg_of(0.0), c_edit=c_edit)
    for cross, inter in ((True, False), (False, True)):
        o, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, semantic=sg_of(0.0, cross, inter), c_edit=c_edit)
        assert torch.equal(o, ref[0]) and torch.equal(z, ref[1]), (cross, inter)


ORACLE_CASES = [(p, s, t, i, (16, 16)) for p in ('eps', 'v') for (s, t) in ((1.0, 1.0), (2.0, 3.0)) for i in (False, True)]
ORACLE_CASES += [('eps', 2.0, 3.0, i, hw) for hw in ((16, 24), (32, 32)) for i in (False, True)]
# seed 11 unless the oracle's thresholds come within 1e-4 of a value they compare: then a seed that keeps them more than 1.2e-4 away
SEEDS = {('eps', 1.0, 1.0, True, (16, 16)): 12, ('eps', 2.0, 3.0, True, (16, 16)): 12, ('v', 1.0, 1.0, False, (16, 16)): 12,
         ('v', 1.0, 1.0, True, (16, 16)): 13, ('eps', 2.0, 3.0, False, (16, 24)): 15, ('eps', 2.0, 3.0, True, (16, 24)): 12,
         ('eps', 2.0, 3.0, False, (32, 32)): 45, ('eps', 2.0, 3.0, True, (32, 32)): 58}


@pytest.mark.parametrize('pred,src_scale,tgt_scale,intersect,hw', ORACLE_CASES)
def test_vs_ledits_oracle(unet, usd, sched, with_prediction, pred, src_scale, tgt_scale, intersect, hw):
    """Engine against the CPU oracle at lambda 0.9 within SEGA's bounds (rel z < 2e-4, |dx| < 1e-3), the oracle's threshold margins
    above 1e-4, and the result more than 10x the bound from SEGA's at the same settings."""
    with_prediction(pred)
    h, w = hw
    seed = SEEDS.get((pred, src_scale, tgt_scale, intersect, hw), 11)
    x0, c_src, c_tgt, uc, c_edit, noise = _inputs(sched, h, w, seed=seed)
    sg = sg_of(0.9, True, intersect)
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise, return_z=True, semantic=sg, c_edit=c_edit)
    sega = unet.cycle_lockstep(x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise, semantic=sg_of(0.9), c_edit=c_edit)
    torch.manual_seed(seed + 1)
    stats = {}
    with torch.no_grad():
        y_ref, z_ref = ledits_cycle(usd, NARROW, x0, c_src, c_tgt, uc, c_edit, 6, 0.1, 2, src_scale, tgt_scale, list(sg.signed_scales()),
                                    [0.9, 0.9], [4, 3], 1, 0.3, 0.4, [3, 1], intersect, prediction=pred, stats=stats)
    z_ref = torch.stack(z_ref, dim=1)
    rz = maxdiff(z.cpu(), z_ref) / float(z_ref.abs().max())
    dx = maxdiff(out.cpu(), y_ref)
    ds = maxdiff(out.cpu(), sega.cpu())
    print(f'ledits {pred} ({src_scale}, {tgt_scale}) intersect {intersect} {h}x{w}: rel|dz| {rz:.2e} |dx| {dx:.2e} |x - sega x| {ds:.2e} '
          f'margins {stats["margin1"]:.2e} {stats["margin2"]:.2e} layers {stats["layers"]}')
    assert stats['layers'] == 5
    assert rz < 2e-4 and dx < 1e-3
    assert ds > 10 * 1e-3
    assert stats['margin1'] > 1e-4 and (not intersect or stats['margin2'] > 1e-4)


@pytest.mark.parametrize('mma', [1, 5])
def test_composes_with_a_mask(eng, unet, sched, mode, mma):
    """Box mask plus masked concepts: outside the box the latent is x0 bit for bit; inside it differs from the masked loop without
    concepts.  Mode 5 is the pipeline's autocast."""
    mode(mma)
    x0, c_src, c_tgt, uc, c_edit, noise = _inputs(sched)
    m = torch.zeros(B, 1, 16, 16)
    m[..., 4:12, 4:12] = 1.0
    out = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=m, semantic=sg_of(0.9, True, True), c_edit=c_edit).cpu()
    masked = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=m).cpu()
    inside = m.expand_as(x0) == 1
    assert torch.equal(out[~inside], x0[~inside]) and not torch.equal(out[inside], masked[inside])


def test_rejections(eng, unet, sched):
    """At the C ABI (past the Python checks): token counts 0 and L - 1, a null mask struct, a latent side off a multiple of 4, and a
    net without 1/4-resolution cross-attention; in Python: counts out of range.  The engine runs on afterwards."""
    import ctypes as C
    from cycle_diffusion_b200 import _cabi
    from cycle_diffusion_b200.engine import UNet, _ptr
    x0, c_src, c_tgt, uc, c_edit, noise = _inputs(sched)
    sg = sg_of(0.9, True)
    n = sched.refine_steps
    xd, cs, ct, ud, ce, nd = (t.cuda().contiguous() for t in (x0, c_src, c_tgt, uc, c_edit, noise))
    out = torch.empty_like(xd)

    def raw(net, am, h=16, w=16):
        return _cabi.lib.cdx_cycle_lockstep_semantic_attn(net.h, _ptr(xd), _ptr(cs), _ptr(ct), _ptr(ud), L, 1.0, 3.0, sched.coef_array(),
                                                          sched.t_array(), n, _ptr(nd), sched.sqrt_a_T, sched.sqrt_1ma_T, _ptr(out), None, B,
                                                          4, h, w, eng.stream, None, _ptr(ce), C.byref(sg.c_struct(n)),
                                                          C.byref(am) if am is not None else None)
    assert raw(unet, sg.attn_mask_struct(L)) == 0
    for bad in (0, L - 1):
        am = sg.attn_mask_struct(L)
        am.n_tokens[1] = bad
        assert raw(unet, am) == -1, bad
    assert raw(unet, None) == -1
    assert raw(unet, sg.attn_mask_struct(L), 4, 16) == -1          # a 1-row map
    wide = UNet(eng, WIDE, 'openai').load_state_dict(specs.synth_state_dict(specs.openai_unet_params(WIDE), 5))
    g = torch.Generator().manual_seed(8)
    cw = torch.randn(B, L, 768, generator=g)
    with pytest.raises(AssertionError, match='no cross-attention'):
        wide.cycle_lockstep(x0, cw, cw, cw, 1.0, 3.0, sched, noise, semantic=sg, c_edit=torch.randn(2, L, 768, generator=g))
    with pytest.raises(ValueError):
        unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, semantic=sg_of(0.9, True, tokens=(3, L - 1)), c_edit=c_edit)
    assert torch.equal(unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, semantic=sg, c_edit=c_edit), out)


@pytest.mark.parametrize('variant', ['cross', 'intersect_per_prompt2', 'auto_mask', 'autocast'])
def test_pipeline_routes_to_the_loop(eng, mode, variant):
    """The pipeline's latents equal UNet.cycle_lockstep(..., semantic=...) with the synthetic encoder's word counts, exactly, and
    differ from SEGA's; an edit_type, two_phase and flags without editing_prompt are rejected."""
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    from cycle_diffusion_b200.schedule import DDIMSchedule
    g = _generator(eng)
    precision = 'autocast' if variant == 'autocast' else 'full'
    pipe = CycleDiffusionPipeline(g, precision=precision)
    image = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(4))
    per = 2 if variant == 'intersect_per_prompt2' else 1
    inter = variant == 'intersect_per_prompt2'
    kw = dict(strength=0.75, num_inference_steps=8, guidance_scale=3.0, eta=0.1, num_images_per_prompt=per)
    edit = dict(editing_prompt=['glasses', 'a red hat'], reverse_editing_direction=[False, True], edit_guidance_scale=[4.0, 2.0],
                edit_threshold=[0.8, 0.5], edit_cooldown_steps=[None, 4], edit_warmup_steps=1, edit_momentum_scale=0.2, edit_mom_beta=0.5)
    mask_arg = 'auto' if variant == 'auto_mask' else None
    lat = {}

    def run(tag, **extra):
        cb = lambda i, t, x: lat.__setitem__(tag, x)
        pipe(['a dog'] * 2, ['a cat'] * 2, image, generator=torch.Generator().manual_seed(9), callback=cb, mask_image=mask_arg, **kw, **extra)
    run('sega', **edit)
    run('ledits', **edit, use_cross_attn_mask=not inter, use_intersect_mask=inter)
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
        c_edit = g.get_learned_conditioning(['glasses', 'a red hat'])
        sched = DDIMSchedule(8, 0.1, 8 - 6, g.alphas_cumprod)
        mom = g.encode_first_stage(eng.shift_scale(img, -0.5, 2.0))
        x0 = eng.vae_posterior(mom, torch.randn(Bn, 4, 16, 16, generator=gen), g.scale_factor)
        noise = torch.zeros(sched.refine_steps + 1, Bn, 4, 16, 16)
        noise[0] = torch.randn(Bn, 4, 16, 16, generator=gen)
        for i in range(sched.refine_steps - 1):
            noise[1 + i] = torch.randn(Bn, 4, 16, 16, generator=gen)
        sg = SemanticGuidance.for_concepts(2, [4.0, 2.0], [False, True], [0.8, 0.5], [None, 4], 1, 0.2, 0.5, not inter, inter, [1, 3])
        ref = g.unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1, 3.0, sched, noise, mask=mask, semantic=sg, c_edit=c_edit)
    assert torch.equal(lat['ledits'], ref) and not torch.equal(lat['ledits'], lat['sega'])
    if variant == 'cross':
        call = lambda **k: pipe('a dog', 'a cat', image, num_inference_steps=4, **k)
        for extra in (dict(editing_prompt='glasses', use_cross_attn_mask=True, two_phase=True),
                      dict(editing_prompt='glasses', use_intersect_mask=True, cross_attention_kwargs={'edit_type': 'pnp'}),
                      dict(use_cross_attn_mask=True), dict(editing_prompt='glasses', use_cross_attn_mask=True, edit_token_counts=[1, 2])):
            with pytest.raises(ValueError):
                call(**extra)
