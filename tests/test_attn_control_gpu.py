"""Prompt-to-Prompt attention control on the lock-step loop (cdx_cycle_lockstep_ctl, cdx_op_attention_rows): the fused kernel's
row remap bit for bit, the no-op cases bit for bit, the engine against the CPU P2P oracle, composition with a mask, and the
pipeline's cross_attention_kwargs."""
import pytest
import torch

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.attn_control import AttentionControl
from cycle_diffusion_b200.wrappers import encode_noise
from tests.common import NARROW, VAE_SMALL, maxdiff
from tests.p2p_oracle import p2p_cycle

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


def _swap_map():
    """P2P's token mapper for a one-token swap at positions 2 <-> 3 of sample 1 (identity for sample 0), times an equalizer that
    doubles token 4 and halves token 5."""
    A = torch.eye(L).repeat(B, 1, 1)
    A[1, 2, 2] = A[1, 3, 3] = 0.0
    A[1, 2, 3] = A[1, 3, 2] = 1.0
    eq = torch.ones(L)
    eq[4], eq[5] = 2.0, 0.5
    return A * eq


@pytest.mark.parametrize('mma,ds', [(1, (16, 32, 40, 64, 80, 160)), (5, (16, 32, 40, 64, 80, 160)), (3, (16, 32, 40, 64, 80))])
@pytest.mark.parametrize('N,Nk', [(256, 256), (200, 200), (256, 77), (200, 77)])
def test_row_remap_is_exact(eng, mode, mma, ds, N, Nk):
    """op_attention with a row table equals op_attention on the remapped q and k with v unchanged, bit for bit.  The largest |q| and
    |k| sit in row 0, which maps to itself, so both sides take the same fp16-split exponents."""
    mode(mma)
    rows = [0, 0, 1]
    for d in ds:
        heads = 2
        g = torch.Generator().manual_seed(d + N + Nk)
        q, k, v = torch.randn(3, N, heads * d, generator=g), torch.randn(3, Nk, heads * d, generator=g), torch.randn(3, Nk, heads * d, generator=g)
        q[0, 0, 0], k[0, 0, 0] = 6.0, -6.0
        q, k, v = q.cuda(), k.cuda(), v.cuda()
        got = eng.op_attention(q, k, v, heads, d ** -0.5, qk_rows=rows)
        ref = eng.op_attention(q[rows], k[rows], v, heads, d ** -0.5)
        assert torch.equal(got, ref), f'mode {mma} d={d} N={N} Nk={Nk}: max |diff| {maxdiff(got.cpu(), ref.cpu()):.3e}'
        assert not torch.equal(got[2], eng.op_attention(q, k, v, heads, d ** -0.5)[2])
    if mma == 3:
        with pytest.raises(AssertionError):                      # TF32 planes have no d = 160 fused kernel: no silent fall-back
            eng.op_attention(torch.randn(3, N, 320).cuda(), torch.randn(3, Nk, 320).cuda(), torch.randn(3, Nk, 320).cuda(), 2, 0.1, qk_rows=rows)


@pytest.mark.parametrize('mma', [1, 5])
@pytest.mark.parametrize('pred', ['eps', 'v'])
def test_no_op_controls_are_bit_identical(unet, sched, mode, with_prediction, mma, pred):
    """Zero controlled steps (with or without a token map), and an identity token map with every step controlled against no token
    map, change nothing bit for bit."""
    mode(mma)
    with_prediction(pred)
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True)
    for ctl in (AttentionControl(0.0, 0.0), AttentionControl(0.1, 0.1, token_map=_swap_map())):   # int(0.1 * 4) == 0
        o, zz = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, attn_control=ctl)
        assert torch.equal(o, out) and torch.equal(zz, z)
    plain = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, attn_control=AttentionControl(1.0, 1.0))
    ident = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, attn_control=AttentionControl(1.0, 1.0, token_map=torch.eye(L)))
    assert torch.equal(ident, plain) and not torch.equal(plain, out)


@pytest.mark.parametrize('pred', ['eps', 'v'])
@pytest.mark.parametrize('h,w', [(16, 16), (16, 24)])
def test_vs_p2p_oracle(unet, usd, sched, with_prediction, pred, h, w):
    """Engine (remapped Q / K tiles, A . c_tgt projected) against the CPU oracle (probabilities replaced literally) with a swap
    mapper times an equalizer (bounds of test_soft_mask_vs_masked_oracle).  The source chain's z stays with the uncontrolled
    loop's: the rows share one U-Net call whose fp16-split operands take one exponent per tensor."""
    with_prediction(pred)
    x0, c_src, c_tgt, uc, noise = _inputs(sched, h, w, seed=11)
    A = _swap_map()
    ctl = AttentionControl(0.75, 0.5, self_max_tokens=64, token_map=A)          # 3 and 2 of the 4 steps; self: levels of <= 64 tokens
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, attn_control=ctl)
    _, z_plain = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True)
    rs = maxdiff(z.cpu(), z_plain.cpu()) / float(z_plain.abs().max())
    torch.manual_seed(12)                                                       # the seed _inputs drew the noise under
    with torch.no_grad():
        y_ref, z_ref = p2p_cycle(usd, NARROW, x0, c_src, c_tgt, uc, 6, 0.1, 2, 1.0, 3.0, 3, 2, 64, A, prediction=pred)
    z_ref = torch.stack(z_ref, dim=1)
    rz = maxdiff(z.cpu(), z_ref) / float(z_ref.abs().max())
    dx = maxdiff(out.cpu(), y_ref)
    print(f'p2p {pred} {h}x{w} vs oracle: rel|dz| {rz:.2e}  |dx| {dx:.2e}; source z vs uncontrolled rel {rs:.2e}')
    assert rz < 2e-4 and dx < 1e-3 and rs < 1e-6


def test_composes_with_a_mask(unet, sched):
    """Box mask plus control: outside the box the latent is x0 bit for bit; inside it differs from the uncontrolled masked edit."""
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    m = torch.zeros(B, 1, 16, 16)
    m[..., 4:12, 4:12] = 1.0
    ctl = AttentionControl(0.75, 0.5, self_max_tokens=64, token_map=_swap_map())
    out = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=m, attn_control=ctl).cpu()
    masked = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=m).cpu()
    inside = m.expand_as(x0) == 1
    assert torch.equal(out[~inside], x0[~inside]) and not torch.equal(out[inside], masked[inside])


def test_rejections(unet, sched, mode):
    """Control the engine cannot honour raises instead of running uncontrolled."""
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    ctl = AttentionControl(0.5, 0.5)
    for m in (0, 2):
        mode(m)
        with pytest.raises(AssertionError):
            unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, attn_control=ctl)
    mode(1)
    with pytest.raises(AssertionError):                          # a source chain at scale 0 has no source-prompt row
        unet.cycle_lockstep(x0, c_src, c_tgt, uc, 0.0, 3.0, sched, noise, attn_control=ctl)
    with pytest.raises(ValueError):
        unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, attn_control=AttentionControl(0.5, 0.5, token_map=torch.eye(L - 1)))


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


def test_pipeline_and_wrapper_route_to_the_control(eng, mode):
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    w = _sd_wrapper(eng)
    pipe = CycleDiffusionPipeline(w.generator)
    image = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(4))
    kw = dict(strength=0.75, num_inference_steps=8, guidance_scale=3.0, eta=0.1)
    lat = {}

    def run(tag, **extra):
        cb = lambda i, t, x: lat.__setitem__(tag, x)
        return pipe('a dog', 'a cat', image, generator=torch.Generator().manual_seed(9), callback=cb, **kw, **extra).images

    swap = torch.eye(L)[[0, 2, 1] + list(range(3, L))]
    p2p = {'edit_type': 'reweight', 'cross_replace_steps': 0.8, 'self_replace_steps': 0.4, 'token_map': swap, 'equalizer': torch.ones(L) * 1.5}
    plain = run('plain')
    assert torch.equal(run('ignored', cross_attention_kwargs={'scale': 0.5}), plain)
    run('p2p', cross_attention_kwargs=p2p)
    # the same control straight on the U-Net: the pipeline's latents exactly
    g = w.generator
    gen = torch.Generator().manual_seed(9)
    c_tgt, c_src, uc = g.get_learned_conditioning(['a dog'] * 2), g.get_learned_conditioning(['a cat'] * 2), g.get_learned_conditioning([''] * 2)
    from cycle_diffusion_b200.schedule import DDIMSchedule
    sched = DDIMSchedule(8, 0.1, 8 - 6, g.alphas_cumprod)
    mom = g.encode_first_stage(eng.shift_scale(image, -0.5, 2.0))
    x0 = eng.vae_posterior(mom, torch.randn(2, 4, 16, 16, generator=gen), g.scale_factor)
    noise = torch.zeros(sched.refine_steps + 1, 2, 4, 16, 16)
    noise[0] = torch.randn(2, 4, 16, 16, generator=gen)
    for i in range(sched.refine_steps - 1):
        noise[1 + i] = torch.randn(2, 4, 16, 16, generator=gen)
    ref = g.unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1, 3.0, sched, noise,
                                attn_control=AttentionControl(0.8, 0.4, token_map=swap * 1.5))
    assert torch.equal(lat['p2p'], ref) and not torch.equal(lat['p2p'], lat['plain'])
    # the text wrapper's cycle takes the same value
    out_w = w.cycle(image, ['a cat'] * 2, ['a dog'] * 2, attn_control=AttentionControl(0.8, 0.4))
    assert out_w.shape == (2, 3, 128, 128) and bool(torch.isfinite(out_w).all())
    call = lambda **k: pipe('a dog', 'a cat', image, num_inference_steps=4, **k)
    ok = {'edit_type': 'replace', 'cross_replace_steps': 0.5, 'self_replace_steps': 0.5}
    for kwargs in ({**ok, 'edit_type': 'refine'}, {**ok, 'cross_replace_steps': 2.0}, {**ok, 'token_map': torch.eye(L + 1)}):
        with pytest.raises(ValueError):
            call(cross_attention_kwargs=kwargs)
    with pytest.raises(ValueError):
        call(cross_attention_kwargs=ok, two_phase=True)
    for m in (0, 2):
        mode(m)
        with pytest.raises(AssertionError):
            call(cross_attention_kwargs=ok)
    mode(1)
