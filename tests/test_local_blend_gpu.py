"""Prompt-to-Prompt's LocalBlend on the lock-step loop (cdx_cycle_lockstep_blend): the weighted probe against float64 and against the
span form, the mask stage bit for bit against its fp32 restatement, the no-op settings bit for bit, the loop against
tests/local_blend_oracle.py, composition with a user mask and paste-back, and the interfaces."""
import ctypes as C

import pytest
import torch

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.attn_control import AttentionControl, LocalBlend, refine_token_map, replace_token_map
from cycle_diffusion_b200.wrappers import encode_noise
from tests.common import NARROW, VAE_SMALL, maxdiff
from tests.local_blend_oracle import blend_cycle, mask_stage_fp32, normalised
from tests.test_ledits_gpu import REP, probe_bound
from tests.test_sega_gpu import guarded, inner
from tests.test_step_kernels_gpu import GUARD, NAN

pytestmark = pytest.mark.gpu

B, L = 2, 77
BOS, EOS, A_, CAT, DOG, FLUFFY = 49406, 49407, 320, 2368, 1929, 21416
# the loop's relative |dz| bound (tests/test_attn_refine_gpu.py) times five: cells whose normalised map lies closer than this to the
# threshold may flip between the engine and the oracle and are left out of the comparison
MARGIN = 1e-3


@pytest.fixture(scope='module')
def eng():
    from cycle_diffusion_b200.engine import Engine
    return Engine(0)


@pytest.fixture
def mode(eng):
    yield eng.set_mma_mode
    eng.set_mma_mode(1)


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


def _sched(kind='cycle'):
    from cycle_diffusion_b200.schedule import DDIMSchedule, EditFriendlySchedule
    return DDIMSchedule(6, 0.1, 2) if kind == 'cycle' else EditFriendlySchedule(6, 2, solver=kind)


def _inputs(sched, h=16, w=16, seed=7):
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(B, 4, h, w, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(B, L, 48, generator=g) for _ in range(3))
    torch.manual_seed(seed + 1)
    return x0, c_src, c_tgt, uc, encode_noise(sched, sched.refine_steps, x0.shape)


def _words():
    a_src, a_tgt = torch.zeros(B, L), torch.zeros(B, L)
    a_src[:, 2] = 1.0
    a_tgt[:, 2:4] = 1.0
    return a_src, a_tgt


def _control(kind):
    """None, replace with an insertion's token map, or the pipeline's refine for it."""
    A = refine_token_map([BOS, A_, CAT, EOS], [BOS, A_, FLUFFY, CAT, EOS], L)
    if kind == 'none':
        return None
    if kind == 'replace':
        return AttentionControl(0.75, 0.5, 64, replace_token_map([BOS, A_, CAT, EOS], [BOS, A_, FLUFFY, CAT, EOS], L))
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    return CycleDiffusionPipeline._attn_control({'edit_type': 'refine', 'cross_replace_steps': 0.75, 'self_replace_steps': 0.5,
                                                 'self_replace_max_tokens': 64, 'token_map': A}, 1.0, False)


# ================================================================================================ the weighted probe
@pytest.mark.parametrize('mma,d', [(m, d) for m in (0, 1, 3, 4, 5) for d in (40, 64, 160)])
def test_weighted_probe_vs_float64(eng, mode, mma, d):
    """Every entry's map against a float64 softmax of the layer's q and K contracted with its weights, within probe_bound (the span
    sum replaced by the weighted sum, weights >= 0); 0/1 weights over tokens 1..n give the span form's map bit for bit; the attention
    output is the one without the probe, bit for bit; the map's guards stay NaN."""
    mode(mma)
    heads = 8 if d == 40 else 2
    C, nimg, Lp = heads * d, 3, 80
    for gi, (gh, gw) in enumerate([(4, 6), (8, 8), (16, 16)]):
        N = gh * gw
        g = torch.Generator().manual_seed(1000 * mma + 10 * d + gi)
        q = torch.randn(nimg * N, C, generator=g) * 1.5
        kv = torch.zeros(nimg * Lp, 2 * C)
        for b in range(nimg):
            kv[b * Lp: b * Lp + L] = torch.randn(L, 2 * C, generator=g)
        rows = [2, 0, 1, 2]
        wts = torch.rand(len(rows), L, generator=g) * (torch.rand(len(rows), L, generator=g) < 0.3)
        wts[0, 5] = 2.5
        qd, kvd = q.cuda(), kv.cuda()
        out0 = torch.empty(nimg * N, C, device='cuda')
        out1 = torch.empty(nimg * N, C, device='cuda')
        n = len(rows) * N
        mp = guarded(n, NAN).cuda()
        plan = eng.op_attention_net('cross', out0, nimg, N, heads, d, d ** -0.5, q=qd, kv=kvd, L=L, ctx_lp=Lp)
        eng.op_attention_net('cross', out1, nimg, N, heads, d, d ** -0.5, q=qd, kv=kvd, L=L, ctx_lp=Lp, probe_rows=rows, probe_weights=wts,
                             probe_map=inner(mp, n))
        spans = [1, L - 2, 5, 9]
        span_map = torch.empty(n, device='cuda')
        ones_map = torch.empty(n, device='cuda')
        ones = torch.zeros(len(rows), L)
        for i, sp in enumerate(spans):
            ones[i, 1: 1 + sp] = 1.0
        eng.op_attention_net('cross', out0.clone(), nimg, N, heads, d, d ** -0.5, q=qd, kv=kvd, L=L, ctx_lp=Lp, probe_rows=rows,
                             probe_spans=spans, probe_map=span_map)
        eng.op_attention_net('cross', out0.clone(), nimg, N, heads, d, d ** -0.5, q=qd, kv=kvd, L=L, ctx_lp=Lp, probe_rows=rows,
                             probe_weights=ones, probe_map=ones_map)
        torch.cuda.synchronize()
        assert torch.equal(out0, out1)
        assert torch.equal(span_map, ones_map)
        got = mp.cpu()
        assert torch.isnan(got[:GUARD]).all() and torch.isnan(got[GUARD + n:]).all()
        got = inner(got, n).reshape(len(rows), N).double()
        worst = 0.0
        for i, b in enumerate(rows):
            qb = q[b * N:(b + 1) * N].double()
            kb = kv[b * Lp: b * Lp + L, :C].double()
            P = torch.stack([torch.softmax(qb[:, h * d:(h + 1) * d] @ kb[:, h * d:(h + 1) * d].T * d ** -0.5, dim=-1) @ wts[i].double()
                             for h in range(heads)])
            want = P.sum(dim=0)
            bound = probe_bound(qb, kb, heads, 0, REP[plan['route']], P) + 1e-30
            err = (got[i] - want).abs()
            assert (err <= bound).all(), f'entry {i} {gh}x{gw}: {float((err / bound).max()):.2f} of the bound'
            worst = max(worst, float((err / bound).max()))
        print(f'mode {mma} d {d} {gh}x{gw} route {plan["route"]}: worst error {worst:.3f} of the bound')


# ================================================================================================ the mask stage
@pytest.mark.parametrize('gh,gw', [(16, 16), (16, 24)])
@pytest.mark.parametrize('n_vec,n_terms', [(2, 1), (2, 2), (4, 1), (4, 2)])
@pytest.mark.parametrize('user', [False, True])
def test_mask_stage_bit_exact(eng, gh, gw, n_vec, n_terms, user):
    """Four launches on one running buffer against mask_stage_fp32, bit for bit (the running sums and the mask): maps on a 1/8
    lattice (ties in the pool and the maximum), one image's target blend map and source subtract map zero at every launch
    (a zero maximum adds nothing), sparse maps, thresholds that land on lattice ratios."""
    G, h, w = gh * gw, 4 * gh, 4 * gw
    g = torch.Generator().manual_seed(gh * gw + 10 * n_vec + n_terms + user)
    run = torch.zeros(B * n_vec, G, device='cuda')
    ref_run = torch.zeros(B * n_vec, G)
    um = torch.rand(B, 1, h, w, generator=g) * (torch.rand(B, 1, h, w, generator=g) < 0.7) if user else None
    seen = set()
    for launch in range(4):
        maps = torch.round(torch.rand(B, n_vec, n_terms, G, generator=g) * 8) / 8 * (torch.rand(B, n_vec, n_terms, G, generator=g) < 0.15)
        maps[1, 1] = 0.0
        if n_vec == 4:
            maps[1, 2] = 0.0
        maps = maps.reshape(-1, G).contiguous()
        got = eng.op_local_blend_mask(maps.cuda(), n_terms, n_vec, run, h, w, 0.5, 0.75, um.cuda() if user else None).cpu()
        want = mask_stage_fp32(maps, n_terms, n_vec, ref_run, 0.5, 0.75, gh, gw, um)
        assert torch.equal(run.cpu(), ref_run), f'launch {launch}: running sums'
        assert torch.equal(got, want), f'launch {launch}: {int((got != want).sum())} mask values differ'
        seen.add(bool((want > 0).any()) and bool((want == 0).any()))
    assert True in seen                                           # neither empty nor full


# ================================================================================================ the loop
@pytest.mark.parametrize('mma', [1, 5])
@pytest.mark.parametrize('pred', ['eps', 'v'])
@pytest.mark.parametrize('kind', ['none', 'replace', 'refine'])
def test_no_op_settings_are_bit_identical(unet, mode, with_prediction, mma, pred, kind):
    """start_blend = 1 (no blended step) and th_blend = 0 without subtract (a mask of ones: probabilities are positive) give the loop
    without LocalBlend, latents and z bit for bit."""
    mode(mma)
    with_prediction(pred)
    sched = _sched()
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    ctl = _control(kind)
    a_src, a_tgt = _words()
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, attn_control=ctl)
    for lb in (LocalBlend(a_src, a_tgt, start_blend=1.0), LocalBlend(a_src, a_tgt, start_blend=0.0, threshold=(0.0, 0.3))):
        o, zz = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, attn_control=ctl, local_blend=lb)
        assert torch.equal(o, out) and torch.equal(zz, z)


def _threshold(rec):
    """A threshold from the oracle's last-step normalised blend maps: the midpoint of the widest gap between their sorted values
    inside the 30-70 % quantile range, so the mask is neither empty nor full and no cell lies near it."""
    R = rec[-1]['R']
    v = torch.cat([normalised(R[:, k], True).flatten() for k in (0, 1)]).sort().values
    lo, hi = int(0.3 * v.numel()), int(0.7 * v.numel())
    gaps = v[lo + 1: hi] - v[lo: hi - 1]
    k = int(gaps.argmax())
    return float((v[lo + k] + v[lo + k + 1]) / 2)


@pytest.mark.parametrize('pred', ['eps', 'v'])
@pytest.mark.parametrize('h,w', [(16, 16), (16, 24)])
@pytest.mark.parametrize('kind', ['none', 'replace', 'refine'])
def test_vs_oracle(unet, usd, with_prediction, pred, h, w, kind):
    """The loop blended at its last step (start_blend 0.75 of 4 steps) against the oracle, bounds of test_attn_refine_gpu, with a
    threshold from the oracle's own maps; cells within MARGIN of it are left out (reported).  The compared mask is neither empty nor
    full; outside it the output is x0 bit for bit."""
    with_prediction(pred)
    sched = _sched()
    x0, c_src, c_tgt, uc, noise = _inputs(sched, h, w, seed=11)
    ctl = _control(kind)
    a_src, a_tgt = _words()
    A = ctl.token_map.expand(B, L, L).contiguous() if ctl is not None and ctl.token_map is not None else None
    W = ctl.own_weight.expand(B, L).contiguous() if ctl is not None and ctl.own_weight is not None else None
    cs, ss = (3, 2) if ctl is not None else (0, 0)
    rec = []
    torch.manual_seed(12)
    with torch.no_grad():
        y_ref, z_ref = blend_cycle(usd, NARROW, x0, c_src, c_tgt, uc, 6, 0.1, 2, 1.0, 3.0, a_src, a_tgt, 4, 0.3, cross_steps=cs,
                                   self_steps=ss, self_max_tokens=64, token_map=A, own_weight=W, prediction=pred, record=rec)
    th = _threshold(rec)
    R = rec[-1]['R']
    vals = [normalised(R[:, k], True) for k in (0, 1)]
    keep = (vals[0] > th) | (vals[1] > th)                                       # [B, gh, gw]
    near = ((vals[0] - th).abs() < MARGIN * th) | ((vals[1] - th).abs() < MARGIN * th)
    m = keep.repeat_interleave(4, -2).repeat_interleave(4, -1).unsqueeze(1)
    y_want = torch.where(m, y_ref, x0)                                           # the last step's source x_{t-1} is x0
    lb = LocalBlend(a_src, a_tgt, start_blend=0.75, threshold=(th, 0.3))
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, attn_control=ctl, local_blend=lb)
    out = out.cpu()
    ok = ~near.repeat_interleave(4, -2).repeat_interleave(4, -1).unsqueeze(1).expand_as(x0)
    z_ref = torch.stack(z_ref, dim=1)
    rz = maxdiff(z.cpu(), z_ref) / float(z_ref.abs().max())
    dx = float((out - y_want).abs()[ok].max())
    frac = float(keep.double().mean())
    print(f'{kind} {pred} {h}x{w}: th {th:.4f} mask {frac:.2f} of the cells, {int(near.sum())} cells excluded; rel|dz| {rz:.2e} |dx| {dx:.2e}')
    assert 0.0 < frac < 1.0
    assert rz < 2e-4 and dx < 1e-3
    outside = (~m).expand_as(x0) & ok
    assert torch.equal(out[outside], x0[outside])


@pytest.mark.parametrize('inversion', ['cycle', 'dpmsolver++'])
def test_composes_with_a_user_mask(unet, inversion):
    """With a box mask_image the mask is the product: outside the box the output is x0 bit for bit; inside the box it is the box-only
    run where LocalBlend keeps the target (same trajectory before the last step) and x0 elsewhere; th = 0 gives the box-only run."""
    sched = _sched(inversion)
    x0, c_src, c_tgt, uc, noise = _inputs(sched, seed=3)
    box = torch.zeros(B, 1, 16, 16)
    box[..., 4:12, 2:14] = 1.0
    a_src, a_tgt = _words()
    ctl = _control('replace')
    only = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=box, attn_control=ctl).cpu()
    ones = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=box, attn_control=ctl,
                               local_blend=LocalBlend(a_src, a_tgt, start_blend=0.0, threshold=(0.0, 0.3))).cpu()
    assert torch.equal(ones, only)
    inside = box.expand_as(x0) == 1
    mixed = []
    for th in (0.5, 0.9, 0.95, 0.97, 0.98, 0.99):          # the synthetic maps are nearly flat: a mask inside the box at some of these
        out = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=box, attn_control=ctl,
                                  local_blend=LocalBlend(a_src, a_tgt, start_blend=0.75, threshold=(th, 0.3))).cpu()
        assert torch.equal(out[~inside], x0[~inside])
        same, orig = (out == only) & inside, (out == x0) & inside
        assert bool((same | orig)[inside].all())
        mixed.append(bool(same.any()) and bool((orig & ~same).any()))
    print(f'{inversion}: thresholds with a mask neither empty nor full inside the box: {mixed}')
    assert any(mixed)


# ================================================================================================ interfaces
def _sd_wrapper(eng, cond_stage):
    from cycle_diffusion_b200.wrappers import SDStochasticTextWrapper
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    vsd = specs.synth_state_dict(specs.kl_vae_params(VAE_SMALL), 21)
    sd = {'model.diffusion_model.' + k: v for k, v in usd.items()}
    sd.update({'first_stage_model.' + k: v for k, v in vsd.items()})
    return SDStochasticTextWrapper('synthetic', engine=eng, state_dict=sd, cond_stage=cond_stage, unet_config=NARROW, vae_config=VAE_SMALL,
                                   custom_steps=6, eta=0.1, white_box_steps=7, skip_steps=[2], encoder_unconditional_guidance_scales=[1.0],
                                   decoder_unconditional_guidance_scales=[3.0], n_trials=1)


class _ToyTokenizer:
    VOCAB = {'': [], 'a': [320], 'cat': [2368], 'dog': [1929], 'hotdog': [1929, 3], 'on': [525], 'grass': [4]}

    def __call__(self, texts):
        rows = []
        for t in texts:
            ids = [BOS] + [i for word in t.split() for i in self.VOCAB[word]] + [EOS]
            rows.append(ids + [0] * (L - len(ids)))
        return torch.tensor(rows)


def _toy_clip_stage(device):
    """A ClipTextCondStage whose tower is a fixed embedding of the token ids: routes words through the stage's own tokenizer."""
    from cycle_diffusion_b200.wrappers import ClipTextCondStage
    stage = object.__new__(ClipTextCondStage)
    stage.tokenizer = _ToyTokenizer()
    table = torch.randn(50000, 48, generator=torch.Generator().manual_seed(4))
    stage.encoder = lambda ids: table[ids % 50000].to(device)
    return stage


@pytest.mark.parametrize('stage', ['synthetic', 'clip'])
def test_pipeline_and_wrapper_route_words(eng, stage):
    """cross_attention_kwargs={'edit_type': 'replace', ..., 'local_blend': {'words': (...)}} runs end to end and equals the engine
    call with the LocalBlend the conditioning model's word_token_weights gives; start_blend 1 equals the run without LocalBlend;
    paste_back still holds the input image exactly where mask_image is 0; the wrapper's cycle() takes the same dict."""
    from cycle_diffusion_b200.attn_control import resolve_local_blend
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    from cycle_diffusion_b200.wrappers import SyntheticTextEncoder
    cond = SyntheticTextEncoder(48, device=eng.device) if stage == 'synthetic' else _toy_clip_stage(eng.device)
    wr = _sd_wrapper(eng, cond)
    pipe = CycleDiffusionPipeline(wr.generator)
    R = wr.resolution
    img = torch.rand(1, 3, R, R, generator=torch.Generator().manual_seed(2)).to(eng.device)
    src, tgt = ('a cat on grass', 'a hotdog on grass')
    base = {'edit_type': 'replace', 'cross_replace_steps': 0.5, 'self_replace_steps': 0.25, 'self_replace_max_tokens': 64}
    # the synthetic weights' maps are nearly flat, so P2P's default threshold 0.3 keeps every cell: 0.99 leaves part of the image
    kw = {**base, 'local_blend': {'words': ('cat', 'hotdog'), 'start_blend': 0.5, 'threshold': (0.99, 0.3)}}
    run = lambda k, **extra: pipe(tgt, src, img, strength=0.7, num_inference_steps=6, guidance_scale=3.0, source_guidance_scale=1.0,
                                  generator=torch.Generator().manual_seed(5), cross_attention_kwargs=k, output_type='pt', **extra).images
    a = run(kw)
    assert bool(torch.isfinite(a).all())
    late = run({**base, 'local_blend': {'words': ('cat', 'hotdog'), 'start_blend': 1.0}})
    assert torch.equal(late, run(base)) and not torch.equal(a, late)
    lb = resolve_local_blend(kw['local_blend'], cond, [src], [tgt])
    assert lb.alpha_src[0].nonzero().flatten().tolist() == [2] and int(lb.alpha_tgt[0].sum()) == (1 if stage == 'synthetic' else 2)
    mask = torch.zeros(1, 1, R, R, device=eng.device)
    mask[..., R // 4: 3 * R // 4, :] = 1.0
    pb = run(kw, mask_image=mask, paste_back=True)
    zero = (mask == 0).expand_as(img)
    assert torch.equal(pb[zero], img[zero])
    out = wr.cycle(img, [src], [tgt], attn_control=CycleDiffusionPipeline._attn_control(base, 1.0, False),
                   local_blend={'words': ('cat', 'hotdog')})
    assert bool(torch.isfinite(out).all())


def test_c_rejections(unet):
    """cdx_cycle_lockstep_blend: a null blend, a null alpha vector, one subtract vector alone, latent sides not multiples of 4, and
    semantic guidance alongside; the Python layer's own checks (sides, a control it cannot take)."""
    from cycle_diffusion_b200 import _cabi
    from cycle_diffusion_b200.attn_control import MutualSelfControl
    sched = _sched()
    a_src, a_tgt = _words()
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    dev = lambda t: t.cuda().contiguous()
    x0, c_src, c_tgt, uc, noise, a_src, a_tgt = map(dev, (x0, c_src, c_tgt, uc, noise, a_src, a_tgt))
    out = torch.empty_like(x0)
    n = sched.refine_steps

    def call(lb, h=16, w=16, sg=None):
        return _cabi.lib.cdx_cycle_lockstep_blend(unet.h, x0.data_ptr(), c_src.data_ptr(), c_tgt.data_ptr(), uc.data_ptr(), L, 1.0, 3.0,
                                                  sched.coef_array(), sched.t_array(), n, noise.data_ptr(), sched.sqrt_a_T, sched.sqrt_1ma_T,
                                                  out.data_ptr(), None, B, 4, h, w, unet.engine.stream, None, None, None, None, None, None,
                                                  None, sg, None, C.byref(lb) if lb is not None else None)
    ok = _cabi.LocalBlendC(a_src.data_ptr(), a_tgt.data_ptr(), None, None, 1, 0.3, 0.3)
    assert call(ok) == 0
    bad = [_cabi.LocalBlendC(None, a_tgt.data_ptr(), None, None, 1, 0.3, 0.3),
           _cabi.LocalBlendC(a_src.data_ptr(), a_tgt.data_ptr(), a_src.data_ptr(), None, 1, 0.3, 0.3),
           _cabi.LocalBlendC(a_src.data_ptr(), a_tgt.data_ptr(), None, None, n + 1, 0.3, 0.3),
           _cabi.LocalBlendC(a_src.data_ptr(), a_tgt.data_ptr(), None, None, 1, 1.0, 0.3)]
    for lb in bad:
        assert call(lb) != 0
    assert call(None) != 0
    x0 = dev(torch.randn(B, 4, 18, 16))
    out = torch.empty_like(x0)
    noise = dev(torch.randn(n + 1, B, 4, 18, 16))
    assert call(ok, h=18) != 0 and 'multiples of 4' in _cabi.lib.cdx_last_error().decode()
    with pytest.raises(ValueError):
        unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, local_blend=LocalBlend(a_src.cpu(), a_tgt.cpu()))
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    with pytest.raises(ValueError):
        unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, attn_control=MutualSelfControl(),
                            local_blend=LocalBlend(a_src.cpu(), a_tgt.cpu()))
    with pytest.raises(Exception):                                # the source chain at scale 0 has no source-prompt row
        unet.cycle_lockstep(x0, c_src, c_tgt, uc, 0.0, 3.0, sched, noise, local_blend=LocalBlend(a_src.cpu(), a_tgt.cpu()))
