"""Prompt-to-Prompt's refine edit on the lock-step loop (cdx_cycle_lockstep_refine, cdx_op_attention_accum): the fused kernel's
accumulating launch bit for bit, the no-op cases bit for bit, the engine against the CPU refine oracle, composition with a mask, and
the pipeline's cross_attention_kwargs."""
import pytest
import torch

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.attn_control import AttentionControl, refine_token_map
from cycle_diffusion_b200.wrappers import encode_noise
from tests.common import NARROW, VAE_SMALL, maxdiff
from tests.p2p_refine_oracle import p2p_refine_cycle

pytestmark = pytest.mark.gpu

B, L = 2, 77
BOS, EOS, A_, CAT, FLUFFY = 49406, 49407, 320, 2368, 21416


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


@pytest.fixture(scope='module')
def sched():
    from cycle_diffusion_b200.schedule import DDIMSchedule
    return DDIMSchedule(6, 0.1, 2)


def _inputs(sched, h=16, w=16, seed=7):
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(B, 4, h, w, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(B, L, 48, generator=g) for _ in range(3))
    torch.manual_seed(seed + 1)
    return x0, c_src, c_tgt, uc, encode_noise(sched, sched.refine_steps, x0.shape)


def _refine(eq=None, cross=0.75, self_=0.5, self_max_tokens=64):
    """The pipeline's refine control for an insertion ("a cat" -> "a fluffy cat"): A . diag(eq), w = (1 - colsum(A)) . eq."""
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    kw = {'edit_type': 'refine', 'cross_replace_steps': cross, 'self_replace_steps': self_, 'self_replace_max_tokens': self_max_tokens,
          'token_map': refine_token_map([BOS, A_, CAT, EOS], [BOS, A_, FLUFFY, CAT, EOS], L)}
    if eq is not None:
        kw['equalizer'] = eq
    return CycleDiffusionPipeline._attn_control(kw, 1.0, False)


def _attn_ref(q, k, v, heads, scale):
    Bq, N, C = q.shape
    d = C // heads
    sp = lambda x: x.double().view(Bq, x.shape[1], heads, d).transpose(1, 2)
    p = torch.softmax(sp(q) @ sp(k).transpose(-1, -2) * scale, dim=-1)
    return (p @ sp(v)).transpose(1, 2).reshape(Bq, N, C)


@pytest.mark.parametrize('mma,ds', [(1, (16, 32, 40, 64, 80, 160)), (5, (16, 32, 40, 64, 80, 160)), (3, (16, 32, 40, 64, 80))])
@pytest.mark.parametrize('N,Nk', [(256, 256), (200, 200), (256, 77), (200, 77)])
def test_accumulating_launch_is_exact(eng, mode, mma, ds, N, Nk):
    """op_attention(accumulate_rows=) adds, bit for bit, a plain launch's result for the listed images into out and leaves the other
    images untouched; against float64 the sum of the two attentions stays within twice the single-attention bound of
    test_attention_any_tokens_gpu (modes 1 and 3: 2e-5 absolute per term; mode 5: 4e-3 relative)."""
    mode(mma)
    rows = [2, 0]
    for d in ds:
        heads = 2
        g = torch.Generator().manual_seed(3 * d + N + Nk)
        q = torch.randn(3, N, heads * d, generator=g) * 1.5
        k, v, v2 = (torch.randn(3, Nk, heads * d, generator=g) for _ in range(3))
        q, k, v, v2 = q.cuda(), k.cuda(), v.cuda(), v2.cuda()
        scale = d ** -0.5
        first = eng.op_attention(q, k, v, heads, scale)
        eng.profile(True)
        got = eng.op_attention(q, k, v2, heads, scale, accumulate_rows=rows, out=first.clone())
        fam = eng.profile_read()
        eng.profile(False)
        assert fam['batched_tc']['launches'] == 1 and 'softmax' not in fam, sorted(fam)
        second = eng.op_attention(q, k, v2, heads, scale)
        want = first.clone()
        want[rows] = first[rows] + second[rows]
        assert torch.equal(got, want), f'mode {mma} d={d} N={N} Nk={Nk}: max |diff| {maxdiff(got.cpu(), want.cpu()):.3e}'
        assert torch.equal(got[1], first[1])
        ref = (_attn_ref(q, k, v, heads, scale) + _attn_ref(q, k, v2, heads, scale))[rows]
        err = float((got[rows].double() - ref).abs().max())
        if mma == 5:
            assert err / float(ref.abs().max()) < 2 * 4e-3, f'd={d}: rel {err / float(ref.abs().max()):.2e}'
        else:
            assert err < 2 * 2e-5, f'mode {mma} d={d} N={N} Nk={Nk}: max abs err {err:.2e}'
    with pytest.raises(AssertionError):                          # a row outside the batch
        eng.op_attention(q, k, v2, heads, d ** -0.5, accumulate_rows=[3], out=first.clone())
    if mma == 3:
        with pytest.raises(AssertionError):                      # TF32 planes have no d = 160 fused kernel: no silent fall-back
            x = torch.randn(3, N, 320).cuda()
            eng.op_attention(x, x, x, 2, 0.1, accumulate_rows=rows, out=torch.zeros_like(x))


@pytest.mark.parametrize('mma', [1, 5])
@pytest.mark.parametrize('pred', ['eps', 'v'])
def test_no_op_refines_are_bit_identical(unet, sched, mode, with_prediction, mma, pred):
    """Refine with an identity map (own weight zero) equals replace with no map, and refine with no controlled step equals the
    uncontrolled run, bit for bit (latents and the source chain's z)."""
    mode(mma)
    with_prediction(pred)
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True)
    for ctl in (AttentionControl(0.0, 0.0, token_map=_refine().token_map, own_weight=_refine().own_weight),
                AttentionControl(0.1, 0.1, token_map=torch.eye(L), own_weight=torch.ones(L))):     # int(0.1 * 4) == 0
        o, zz = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, attn_control=ctl)
        assert torch.equal(o, out) and torch.equal(zz, z)
    replace, zr = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, attn_control=AttentionControl(1.0, 1.0))
    ident, zi = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True,
                                    attn_control=AttentionControl(1.0, 1.0, token_map=torch.eye(L), own_weight=torch.zeros(L)))
    assert torch.equal(ident, replace) and torch.equal(zi, zr) and not torch.equal(replace, out)


def test_own_attention_alone_is_the_uncontrolled_run(unet, sched):
    """A == 0 and w == 1 on cross-attention only: the controlled row's attention is its own, through V'' planes and the summed range
    slot instead of V and the K | V slot -- close to the uncontrolled run, not bit for bit (bounds of test_vs_refine_oracle)."""
    x0, c_src, c_tgt, uc, noise = _inputs(sched, seed=5)
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True)
    ctl = AttentionControl(1.0, 0.0, token_map=torch.zeros(L, L), own_weight=torch.ones(L))
    o, zz = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, attn_control=ctl)
    rz, dx = maxdiff(zz.cpu(), z.cpu()) / float(z.abs().max()), maxdiff(o.cpu(), out.cpu())
    print(f'refine A = 0, w = 1 vs uncontrolled: rel|dz| {rz:.2e}  |dx| {dx:.2e}')
    assert rz < 2e-4 and dx < 1e-3


@pytest.mark.parametrize('pred', ['eps', 'v'])
@pytest.mark.parametrize('h,w', [(16, 16), (16, 24)])
@pytest.mark.parametrize('equalize', [False, True])
def test_vs_refine_oracle(unet, usd, sched, with_prediction, pred, h, w, equalize):
    """Engine (remapped Q / K tiles over V', plus the accumulating launch over V'') against the CPU oracle (probabilities replaced
    literally) for an insertion alignment, bounds of test_vs_p2p_oracle.  The equalizer case scales the inserted token by 8 and its
    neighbour by 3, so max |V'| + max |V''| is well above max |V|: the output's range slot is the sum, and the result stays finite."""
    with_prediction(pred)
    x0, c_src, c_tgt, uc, noise = _inputs(sched, h, w, seed=11)
    eq = None
    if equalize:
        eq = torch.ones(L)
        eq[2], eq[3] = 8.0, 3.0
    ctl = _refine(eq)
    A = ctl.token_map.expand(B, L, L).contiguous()
    W = ctl.own_weight.expand(B, L).contiguous()
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, attn_control=ctl)
    assert bool(torch.isfinite(out).all()) and bool(torch.isfinite(z).all())
    torch.manual_seed(12)                                                       # the seed _inputs drew the noise under
    with torch.no_grad():
        y_ref, z_ref = p2p_refine_cycle(usd, NARROW, x0, c_src, c_tgt, uc, 6, 0.1, 2, 1.0, 3.0, 3, 2, 64, A, W, prediction=pred)
    z_ref = torch.stack(z_ref, dim=1)
    rz = maxdiff(z.cpu(), z_ref) / float(z_ref.abs().max())
    dx = maxdiff(out.cpu(), y_ref)
    print(f'refine {pred} {h}x{w} eq={equalize} vs oracle: rel|dz| {rz:.2e}  |dx| {dx:.2e}')
    assert rz < 2e-4 and dx < 1e-3
    replace = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, attn_control=AttentionControl(0.75, 0.5, 64, ctl.token_map))
    assert not torch.equal(replace, out)                                        # the own term is there


def test_composes_with_a_mask(unet, sched):
    """Box mask plus refine: outside the box the latent is x0 bit for bit; inside it differs from the masked replace edit."""
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    m = torch.zeros(B, 1, 16, 16)
    m[..., 4:12, 4:12] = 1.0
    ctl = _refine()
    out = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=m, attn_control=ctl).cpu()
    rep = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=m,
                              attn_control=AttentionControl(0.75, 0.5, 64, ctl.token_map)).cpu()
    inside = m.expand_as(x0) == 1
    assert torch.equal(out[~inside], x0[~inside]) and not torch.equal(out[inside], rep[inside])


def _sd_wrapper(eng):
    from cycle_diffusion_b200.wrappers import SDStochasticTextWrapper, SyntheticTextEncoder
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    vsd = specs.synth_state_dict(specs.kl_vae_params(VAE_SMALL), 21)
    sd = {'model.diffusion_model.' + k: v for k, v in usd.items()}
    sd.update({'first_stage_model.' + k: v for k, v in vsd.items()})
    return SDStochasticTextWrapper('synthetic', engine=eng, state_dict=sd, cond_stage=SyntheticTextEncoder(48), unet_config=NARROW,
                                   vae_config=VAE_SMALL, latent_size=16, resolution=128, custom_steps=4, eta=0.1, white_box_steps=5,
                                   skip_steps=[0], encoder_unconditional_guidance_scales=[1], decoder_unconditional_guidance_scales=[3.0],
                                   n_trials=1)


def test_pipeline_and_wrapper_route_refine(eng, unet, sched, mode):
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    from cycle_diffusion_b200.schedule import DDIMSchedule
    w = _sd_wrapper(eng)
    pipe = CycleDiffusionPipeline(w.generator)
    image = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(4))
    kw = dict(strength=0.75, num_inference_steps=8, guidance_scale=3.0, eta=0.1)
    lat = {}

    def run(tag, **extra):
        cb = lambda i, t, x: lat.__setitem__(tag, x)
        return pipe('a fluffy dog', 'a dog', image, generator=torch.Generator().manual_seed(9), callback=cb, **kw, **extra).images

    A = refine_token_map([BOS, A_, CAT, EOS], [BOS, A_, FLUFFY, CAT, EOS], L)
    eq = torch.ones(L)
    eq[2] = 2.0
    p2p = {'cross_replace_steps': 0.8, 'self_replace_steps': 0.4, 'token_map': A, 'equalizer': eq}
    run('refine', cross_attention_kwargs={'edit_type': 'refine', **p2p})
    run('reweight', cross_attention_kwargs={'edit_type': 'reweight', **p2p})
    # the same control straight on the U-Net: the pipeline's latents exactly
    g = w.generator
    gen = torch.Generator().manual_seed(9)
    c_tgt, c_src, uc = (g.get_learned_conditioning([p] * 2) for p in ('a fluffy dog', 'a dog', ''))
    sch = DDIMSchedule(8, 0.1, 8 - 6, g.alphas_cumprod)
    mom = g.encode_first_stage(eng.shift_scale(image, -0.5, 2.0))
    x0 = eng.vae_posterior(mom, torch.randn(2, 4, 16, 16, generator=gen), g.scale_factor)
    noise = torch.zeros(sch.refine_steps + 1, 2, 4, 16, 16)
    noise[0] = torch.randn(2, 4, 16, 16, generator=gen)
    for i in range(sch.refine_steps - 1):
        noise[1 + i] = torch.randn(2, 4, 16, 16, generator=gen)
    ctl = AttentionControl(0.8, 0.4, token_map=A * eq, own_weight=(1 - A.sum(0)) * eq)
    ref = g.unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1, 3.0, sch, noise, attn_control=ctl)
    assert torch.equal(lat['refine'], ref) and not torch.equal(lat['refine'], lat['reweight'])
    # the text wrapper's cycle takes the same value
    out_w = w.cycle(image, ['a dog'] * 2, ['a fluffy dog'] * 2, attn_control=ctl)
    assert out_w.shape == (2, 3, 128, 128) and bool(torch.isfinite(out_w).all())
    # rejections
    call = lambda **k: pipe('a fluffy dog', 'a dog', image, num_inference_steps=4, **k)
    ok = {'edit_type': 'refine', 'cross_replace_steps': 0.5, 'self_replace_steps': 0.5, 'token_map': A}
    for kwargs in ({k: v for k, v in ok.items() if k != 'token_map'}, {**ok, 'token_map': A * 2}, {**ok, 'token_map': -A}):
        with pytest.raises(ValueError):
            call(cross_attention_kwargs=kwargs)
    with pytest.raises(ValueError):
        call(cross_attention_kwargs=ok, two_phase=True)
    x0s, c_s, c_t, ucs, nz = _inputs(sched)
    for bad in (torch.ones(L + 1), torch.ones(B + 1, L)):
        with pytest.raises(ValueError):
            unet.cycle_lockstep(x0s, c_s, c_t, ucs, 1.0, 3.0, sched, nz, attn_control=AttentionControl(0.5, 0.5, token_map=A, own_weight=bad))
    for m in (0, 2):
        mode(m)
        with pytest.raises(AssertionError):
            call(cross_attention_kwargs=ok)
        with pytest.raises(AssertionError):
            unet.cycle_lockstep(x0s, c_s, c_t, ucs, 1.0, 3.0, sched, nz, attn_control=_refine())
    mode(1)
