"""Mutual self-attention control (MasaCtrl) on the lock-step loop (cdx_cycle_lockstep_mutual, cdx_op_attention_kv_rows): the fused
kernel's K / V row remap bit for bit, the no-op controls bit for bit, the engine against the CPU mutual oracle, composition with a
mask, the rejections, and the routing from the pipeline's cross_attention_kwargs and the SD wrapper."""
import pytest
import torch

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.attn_control import MutualSelfControl
from cycle_diffusion_b200.wrappers import encode_noise
from tests.common import NARROW, VAE_SMALL, maxdiff
from tests.mutual_oracle import mutual_cycle

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


def _check_kv_remap(eng, rows, N, heads, d, tag):
    """op_attention with a K / V row table equals op_attention on the remapped k and v with q unchanged, bit for bit.  The largest
    |k| and |v| sit in row 0, which maps to itself, so both sides take the same fp16-split exponents."""
    n = len(rows)
    g = torch.Generator().manual_seed(d + N + n)
    q, k, v = (torch.randn(n, N, heads * d, generator=g) for _ in range(3))
    k[0, 0, 0], v[0, 1, 1] = -6.0, 6.0
    q, k, v = q.cuda(), k.cuda(), v.cuda()
    got = eng.op_attention(q, k, v, heads, d ** -0.5, kv_rows=rows)
    ref = eng.op_attention(q, k[rows], v[rows], heads, d ** -0.5)
    assert torch.equal(got, ref), f'{tag}: max |diff| {maxdiff(got.cpu(), ref.cpu()):.3e}'
    moved = [b for b in range(n) if rows[b] != b]
    assert not torch.equal(got[moved], eng.op_attention(q, k, v, heads, d ** -0.5)[moved])


@pytest.mark.parametrize('mma,ds', [(1, (16, 32, 40, 64, 80, 160)), (5, (16, 32, 40, 64, 80, 160)), (3, (16, 32, 40, 64, 80))])
@pytest.mark.parametrize('N', [256, 200])
def test_kv_remap_is_exact(eng, mode, mma, ds, N):
    mode(mma)
    for d in ds:
        _check_kv_remap(eng, [0, 0, 1], N, 2, d, f'mode {mma} d={d} N={N}')
    if mma == 3:
        with pytest.raises(AssertionError):                      # TF32 planes have no d = 160 fused kernel: no silent fall-back
            eng.op_attention(torch.randn(3, N, 320).cuda(), torch.randn(3, N, 320).cuda(), torch.randn(3, N, 320).cuda(), 2, 0.1,
                             kv_rows=[0, 0, 1])
    with pytest.raises(AssertionError):                          # one row table per launch
        x = torch.randn(3, N, 64).cuda()
        eng.op_attention(x, x, x, 2, 0.1, qk_rows=[0, 0, 1], kv_rows=[0, 0, 1])


@pytest.mark.parametrize('mma', [1, 5, 3])
@pytest.mark.parametrize('N,d', [(4096, 40), (1024, 80)])
def test_kv_remap_is_exact_at_sd_shapes(eng, mode, mma, N, d):
    """The self-attention shapes of a 12-row SD v1 512^2 lock-step call (batch 4, source scale 1: rows [source cond | target uncond |
    target cond]) under the driver's row table."""
    mode(mma)
    _check_kv_remap(eng, [0, 1, 2, 3] * 3, N, 8, d, f'mode {mma} N={N} d={d}')        # 8 heads of 320 / 640 channels


@pytest.mark.parametrize('mma', [1, 5])
@pytest.mark.parametrize('pred', ['eps', 'v'])
def test_no_op_controls_are_bit_identical(unet, sched, mode, with_prediction, mma, pred):
    """start_step at the loop's step count, or start_layer at the net's 16 SpatialTransformers, changes nothing bit for bit."""
    mode(mma)
    with_prediction(pred)
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True)
    for ctl in (MutualSelfControl(sched.refine_steps, 0), MutualSelfControl(0, 16), MutualSelfControl(9, 99)):
        o, zz = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, attn_control=ctl)
        assert torch.equal(o, out) and torch.equal(zz, z), ctl
    o = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, attn_control=MutualSelfControl(sched.refine_steps - 1, 15))
    assert not torch.equal(o, out)                               # one step, one layer


@pytest.mark.parametrize('scales', [(1.0, 3.0), (2.0, 3.0)])
@pytest.mark.parametrize('start', [(1, 10), (0, 0)])
@pytest.mark.parametrize('h,w', [(16, 16), (16, 24)])
def test_vs_mutual_oracle(unet, usd, sched, scales, start, h, w):
    """Engine (redirected K / V^T tiles) against the CPU oracle (K and V replaced literally), within the bounds of the P2P oracle
    test.  (0, 0) reaches every level, the middle block included; source scale 2 runs a source uncond row, so the target's uncond
    row maps to it.  The source chain's z stays with the uncontrolled loop's: the rows share one U-Net call whose fp16-split operands
    take one exponent per tensor."""
    x0, c_src, c_tgt, uc, noise = _inputs(sched, h, w, seed=11)
    ctl = MutualSelfControl(*start)
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, *scales, sched, noise, return_z=True, attn_control=ctl)
    plain, z_plain = unet.cycle_lockstep(x0, c_src, c_tgt, uc, *scales, sched, noise, return_z=True)
    rs = maxdiff(z.cpu(), z_plain.cpu()) / float(z_plain.abs().max())
    torch.manual_seed(12)                                                       # the seed _inputs drew the noise under
    with torch.no_grad():
        y_ref, z_ref = mutual_cycle(usd, NARROW, x0, c_src, c_tgt, uc, 6, 0.1, 2, *scales, *start)
    z_ref = torch.stack(z_ref, dim=1)
    rz = maxdiff(z.cpu(), z_ref) / float(z_ref.abs().max())
    dx = maxdiff(out.cpu(), y_ref)
    dc = maxdiff(out.cpu(), plain.cpu())
    print(f'mutual {start} scales {scales} {h}x{w} vs oracle: rel|dz| {rz:.2e}  |dx| {dx:.2e}; source z vs uncontrolled rel {rs:.2e}; '
          f'|x - uncontrolled x| {dc:.2e}')
    assert rz < 2e-4 and dx < 1e-3 and rs < 1e-6
    assert dc > 10 * dx                                          # the control is visible above the oracle bound


def test_composes_with_a_mask(unet, sched):
    """Box mask plus control: outside the box the latent is x0 bit for bit; inside it differs from the uncontrolled masked edit."""
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    m = torch.zeros(B, 1, 16, 16)
    m[..., 4:12, 4:12] = 1.0
    out = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=m, attn_control=MutualSelfControl(0, 0)).cpu()
    masked = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=m).cpu()
    inside = m.expand_as(x0) == 1
    assert torch.equal(out[~inside], x0[~inside]) and not torch.equal(out[inside], masked[inside])


def test_rejections(eng, unet, sched, mode):
    """Control the engine cannot honour raises instead of running uncontrolled."""
    from cycle_diffusion_b200.engine import UNet
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    ctl = MutualSelfControl(0, 10)
    for m in (0, 2):
        mode(m)
        with pytest.raises(AssertionError):
            unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, attn_control=ctl)
    mode(1)
    # a context-free LDM U-Net (AttentionBlocks, no SpatialTransformer)
    cfg = dict(in_channels=4, out_channels=4, model_channels=32, attention_resolutions=(2, 4), num_res_blocks=1, channel_mult=(1, 2, 2),
               num_head_channels=16, context_dim=0)
    plain_net = UNet(eng, cfg, 'openai').load_state_dict(specs.synth_state_dict(specs.openai_unet_params(cfg), 41))
    ctx = torch.zeros(B, 1, 1)
    with pytest.raises(AssertionError):
        plain_net.cycle_lockstep(x0, ctx, ctx, None, 1.0, 1.0, sched, noise, attn_control=ctl)


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
    from cycle_diffusion_b200.schedule import DDIMSchedule
    w = _sd_wrapper(eng)
    g = w.generator
    pipe = CycleDiffusionPipeline(g)
    image = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(4))
    kw = dict(strength=0.75, num_inference_steps=8, guidance_scale=3.0, eta=0.1)
    lat = {}

    def run(tag, **extra):
        cb = lambda i, t, x: lat.__setitem__(tag, x)
        return pipe('a dog', 'a cat', image, generator=torch.Generator().manual_seed(9), callback=cb, **kw, **extra).images

    run('plain')
    run('default', cross_attention_kwargs={'edit_type': 'mutual_self'})
    run('mutual', cross_attention_kwargs={'edit_type': 'mutual_self', 'start_step': 1, 'start_layer': 7})
    # the same controls straight on the U-Net: the pipeline's latents exactly
    gen = torch.Generator().manual_seed(9)
    c_tgt, c_src, uc = g.get_learned_conditioning(['a dog'] * 2), g.get_learned_conditioning(['a cat'] * 2), g.get_learned_conditioning([''] * 2)
    sched = DDIMSchedule(8, 0.1, 8 - 6, g.alphas_cumprod)
    mom = g.encode_first_stage(eng.shift_scale(image, -0.5, 2.0))
    x0 = eng.vae_posterior(mom, torch.randn(2, 4, 16, 16, generator=gen), g.scale_factor)
    noise = torch.zeros(sched.refine_steps + 1, 2, 4, 16, 16)
    noise[0] = torch.randn(2, 4, 16, 16, generator=gen)
    for i in range(sched.refine_steps - 1):
        noise[1 + i] = torch.randn(2, 4, 16, 16, generator=gen)
    for tag, ctl in (('default', MutualSelfControl()), ('mutual', MutualSelfControl(1, 7))):
        ref = g.unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1, 3.0, sched, noise, attn_control=ctl)
        assert torch.equal(lat[tag], ref) and not torch.equal(lat[tag], lat['plain']), tag
    # with a mask, a tensor or one made from the prompts
    box = torch.zeros(1, 1, 128, 128)
    box[..., 32:96, 32:96] = 1.0
    mutual = {'edit_type': 'mutual_self', 'start_step': 1, 'start_layer': 7}
    for m in (box, 'auto'):
        img = run('masked', cross_attention_kwargs=mutual, mask_image=m)
        assert img.shape == (2, 3, 128, 128) and bool(torch.isfinite(img).all())
    # the text wrapper's cycle hands the same value to UNet.cycle_lockstep, whose latent it decodes
    calls = []
    real = g.unet.cycle_lockstep

    def spy(*a, **k):
        calls.append((a, k, real(*a, **k)))
        return calls[-1][2]

    ctl = MutualSelfControl(1, 7)
    g.unet.cycle_lockstep = spy
    try:
        out_w = w.cycle(image, ['a cat'] * 2, ['a dog'] * 2, attn_control=ctl)
    finally:
        del g.unet.cycle_lockstep
    (a, k, sample), = calls
    assert k['attn_control'] is ctl
    assert torch.equal(real(*a, **k), sample)
    assert not torch.equal(real(*a, **{**k, 'attn_control': None}), sample)
    assert torch.equal(out_w, eng.shift_scale(g.decode_first_stage(sample), 1.0, 0.5))
    # rejections at the pipeline
    call = lambda **k: pipe('a dog', 'a cat', image, num_inference_steps=4, **k)
    for kwargs in ({**mutual, 'cross_replace_steps': 0.5}, {**mutual, 'start_steps': 2}, {**mutual, 'start_layer': -1}):
        with pytest.raises(ValueError):
            call(cross_attention_kwargs=kwargs)
    with pytest.raises(ValueError):
        call(cross_attention_kwargs=mutual, two_phase=True)
    for m in (0, 2):
        mode(m)
        with pytest.raises(AssertionError):
            call(cross_attention_kwargs=mutual)
    mode(1)

