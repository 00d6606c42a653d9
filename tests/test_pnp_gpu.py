"""Plug-and-Play injection on the lock-step loop (cdx_cycle_lockstep_pnp, cdx_op_groupnorm_rows): the row-mapped GroupNorm bit for
bit in every form the executors use, the no-op controls bit for bit, the engine against the CPU PnP oracle, composition with a
mask, the rejections, and the routing from the pipeline's cross_attention_kwargs and the SD wrapper."""
import pytest
import torch

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.attn_control import PnPControl
from cycle_diffusion_b200.wrappers import encode_noise
from tests.common import NARROW, VAE_SMALL, maxdiff
from tests.pnp_oracle import pnp_cycle

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


# (C1, C2, H, W): single sources and the [h | skip] concat of the output blocks, C from 64 to 2560, HW from 16 to 4096, with the
# rectangular and non-power-of-two maps of test_sizes_gpu.py
SHAPES = [(64, 0, 4, 4), (320, 0, 64, 64), (2560, 0, 8, 8), (640, 640, 16, 16), (1280, 1280, 8, 8), (960, 320, 24, 40),
          (128, 64, 6, 10), (64, 64, 40, 24)]


@pytest.mark.parametrize('rows', [[0, 0, 1], [0, 1, 2, 3] * 3], ids=['3rows', 'lockstep12'])
@pytest.mark.parametrize('C1,C2,H,W', SHAPES)
def test_groupnorm_rows_is_exact(eng, rows, C1, C2, H, W):
    """Image b of the mapped norm is image rows[b] of the plain norm bit for bit, and its range slot is the max over the images it
    wrote: SiLU off and on, and the scale-shift norm (scale / shift the two halves of one [B, 2C] projection)."""
    n, C = len(rows), C1 + C2
    g = torch.Generator(device='cuda').manual_seed(C * 7 + H * W + n)
    x1 = torch.randn(n, H, W, C1, generator=g, device='cuda') * 1.5 + 0.3
    x2 = torch.randn(n, H, W, C2, generator=g, device='cuda') * 0.7 - 0.2 if C2 else None
    gamma, beta = torch.rand(C, generator=g, device='cuda') + 0.5, torch.randn(C, generator=g, device='cuda') * 0.1
    emb = torch.randn(n, 2 * C, generator=g, device='cuda') * 0.3
    for silu, ss in ((False, False), (True, False), (True, True)):
        kw = dict(scale=emb[:, :C], shift=emb[:, C:]) if ss else {}
        y, amax, y_rows, amax_rows = eng.op_groupnorm_rows(x1, x2, gamma, beta, 1e-5, silu, rows, **kw)
        tag = f'C={C1}+{C2} {H}x{W} rows={rows} silu={silu} scale_shift={ss}'
        assert torch.equal(y_rows, y[rows]), f'{tag}: max |diff| {maxdiff(y_rows.cpu(), y[rows].cpu()):.3e}'
        assert float(amax_rows) == float(y_rows.abs().max()), tag
        assert float(amax) == float(y.abs().max()), tag
    with pytest.raises(AssertionError):
        eng.op_groupnorm_rows(x1, x2, gamma, beta, 1e-5, True, [0] * (n - 1) + [n])        # a row outside [0, B)


@pytest.mark.parametrize('mma', [1, 5])
@pytest.mark.parametrize('pred', ['eps', 'v'])
def test_no_op_controls_are_bit_identical(unet, sched, mode, with_prediction, mma, pred):
    """No controlled step, or no controlled block and layer (the net has 16 SpatialTransformers), changes nothing bit for bit."""
    mode(mma)
    with_prediction(pred)
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True)
    for ctl in (PnPControl(0.0, 0.0), PnPControl(feature_blocks=(), attention_start_layer=16), PnPControl(0.2, 0.2, (0, 11), 0)):
        o, zz = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, attn_control=ctl)
        assert torch.equal(o, out) and torch.equal(zz, z), ctl                 # (0.2 of 4 steps: int(0.8) = 0)
    for ctl in (PnPControl(0.25, 0.0, (11,)), PnPControl(0.0, 0.25, (), 15)):  # one step, one block or one layer
        o = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, attn_control=ctl)
        assert not torch.equal(o, out), ctl


@pytest.mark.parametrize('case', ['defaults', 'features', 'attention', 'src2', 'src0'])
@pytest.mark.parametrize('h,w', [(16, 16), (16, 24)])
def test_vs_pnp_oracle(unet, usd, sched, case, h, w):
    """Engine (row-mapped out_layers norm, redirected Q / K tiles) against the CPU oracle (features and Q / K replaced literally),
    within the bounds of the mutual oracle test.  Source scale 2 runs a source uncond row, so the target's uncond row maps to it;
    source scale 0 runs the source as its uncond row alone (PnP's unconditional source branch).  The source chain's z stays with
    the uncontrolled loop's: the rows share one U-Net call whose fp16-split operands take one exponent per tensor."""
    ctl, scales = {'defaults': (PnPControl(), (1.0, 3.0)), 'features': (PnPControl(0.8, 0.0), (1.0, 3.0)),
                   'attention': (PnPControl(0.0, 0.5), (1.0, 3.0)), 'src2': (PnPControl(), (2.0, 3.0)),
                   'src0': (PnPControl(), (0.0, 3.0))}[case]
    x0, c_src, c_tgt, uc, noise = _inputs(sched, h, w, seed=11)
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, *scales, sched, noise, return_z=True, attn_control=ctl)
    plain, z_plain = unet.cycle_lockstep(x0, c_src, c_tgt, uc, *scales, sched, noise, return_z=True)
    rs = maxdiff(z.cpu(), z_plain.cpu()) / float(z_plain.abs().max())
    nf, na = ctl.steps(sched.refine_steps)
    torch.manual_seed(12)                                                       # the seed _inputs drew the noise under
    with torch.no_grad():
        y_ref, z_ref = pnp_cycle(usd, NARROW, x0, c_src, c_tgt, uc, 6, 0.1, 2, *scales, nf, na, ctl.feature_blocks,
                                 ctl.attention_start_layer)
    z_ref = torch.stack(z_ref, dim=1)
    rz = maxdiff(z.cpu(), z_ref) / float(z_ref.abs().max())
    dx = maxdiff(out.cpu(), y_ref)
    dc = maxdiff(out.cpu(), plain.cpu())
    print(f'pnp {case} scales {scales} {h}x{w} vs oracle: rel|dz| {rz:.2e}  |dx| {dx:.2e}; source z vs uncontrolled rel {rs:.2e}; '
          f'|x - uncontrolled x| {dc:.2e}')
    assert rz < 2e-4 and dx < 1e-3 and rs < 1e-6
    assert dc > 10 * dx                                          # the control is visible above the oracle bound


def test_composes_with_a_mask(unet, sched):
    """Box mask plus control: outside the box the latent is x0 bit for bit; inside it differs from the uncontrolled masked edit."""
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    m = torch.zeros(B, 1, 16, 16)
    m[..., 4:12, 4:12] = 1.0
    out = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=m, attn_control=PnPControl()).cpu()
    masked = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=m).cpu()
    inside = m.expand_as(x0) == 1
    assert torch.equal(out[~inside], x0[~inside]) and not torch.equal(out[inside], masked[inside])


def test_rejections(eng, unet, sched, mode):
    """Control the engine cannot honour raises instead of running uncontrolled."""
    from cycle_diffusion_b200.engine import UNet
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    run = lambda ctl: unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, attn_control=ctl)
    for m in (0, 2):
        mode(m)
        with pytest.raises(AssertionError):
            run(PnPControl())
    mode(1)
    with pytest.raises(AssertionError):                          # NARROW has 12 output blocks, 0 .. 11
        run(PnPControl(feature_blocks=(4, 12)))
    dup = PnPControl(feature_blocks=(4, 5))
    object.__setattr__(dup, 'feature_blocks', (4, 4))            # past the Python check: the C ABI rejects it too
    with pytest.raises(AssertionError):
        run(dup)
    # a context-free LDM U-Net (AttentionBlocks, no SpatialTransformer)
    cfg = dict(in_channels=4, out_channels=4, model_channels=32, attention_resolutions=(2, 4), num_res_blocks=1, channel_mult=(1, 2, 2),
               num_head_channels=16, context_dim=0)
    plain_net = UNet(eng, cfg, 'openai').load_state_dict(specs.synth_state_dict(specs.openai_unet_params(cfg), 41))
    ctx = torch.zeros(B, 1, 1)
    with pytest.raises(AssertionError):
        plain_net.cycle_lockstep(x0, ctx, ctx, None, 1.0, 1.0, sched, noise, attn_control=PnPControl(feature_blocks=(1,)))


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

    pnp = {'edit_type': 'pnp', 'feature_steps': 0.5, 'attention_steps': 0.5, 'feature_blocks': [3, 4], 'attention_start_layer': 7}
    run('plain')
    run('default', cross_attention_kwargs={'edit_type': 'pnp'})
    run('pnp', cross_attention_kwargs=pnp)
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
    for tag, ctl in (('default', PnPControl()), ('pnp', PnPControl(0.5, 0.5, (3, 4), 7))):
        ref = g.unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1, 3.0, sched, noise, attn_control=ctl)
        assert torch.equal(lat[tag], ref) and not torch.equal(lat[tag], lat['plain']), tag
    # with a mask, a tensor or one made from the prompts
    box = torch.zeros(1, 1, 128, 128)
    box[..., 32:96, 32:96] = 1.0
    for m in (box, 'auto'):
        img = run('masked', cross_attention_kwargs=pnp, mask_image=m)
        assert img.shape == (2, 3, 128, 128) and bool(torch.isfinite(img).all())
    # PnP's unconditional source branch: an empty source prompt at source scale 0
    img = pipe('a dog', '', image, generator=torch.Generator().manual_seed(9), source_guidance_scale=0, cross_attention_kwargs=pnp,
               **kw).images
    assert img.shape == (2, 3, 128, 128) and bool(torch.isfinite(img).all())
    # the text wrapper's cycle hands the same value to UNet.cycle_lockstep, whose latent it decodes
    calls = []
    real = g.unet.cycle_lockstep

    def spy(*a, **k):
        calls.append((a, k, real(*a, **k)))
        return calls[-1][2]

    ctl = PnPControl(0.5, 0.5, (3, 4), 7)
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
    for kwargs in ({**pnp, 'cross_replace_steps': 0.5}, {**pnp, 'start_step': 2}, {**pnp, 'feature_steps': 1.5},
                   {**pnp, 'feature_blocks': (4, 4)}, {**pnp, 'attention_start_layer': -1}):
        with pytest.raises(ValueError):
            call(cross_attention_kwargs=kwargs)
    with pytest.raises(ValueError):
        call(cross_attention_kwargs=pnp, two_phase=True)
    for m in (0, 2):
        mode(m)
        with pytest.raises(AssertionError):
            call(cross_attention_kwargs=pnp)
    mode(1)
