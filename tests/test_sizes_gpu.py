"""Image sizes other than powers of two, and rectangular images, on the GPU.

The conv3x3 tensor-core path tiles maps whose sides are not powers of two with boxes that overhang the map (their outside rows
are masked in the epilogue), so no such layer falls back to the FFMA tiles.  The first stage and the pipeline take H != W.
Bounds are those of the square tests: 2e-5 relative per op, 2e-4 through a network, 1e-3 on pipeline images."""
import math

import pytest
import torch
import torch.nn.functional as F

from cycle_diffusion_b200 import specs
from tests.common import NARROW, VAE_SMALL, WIDE, golden, maxdiff

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module', params=[1, 3], ids=['h16', 'tf32'])
def eng(request):
    from cycle_diffusion_b200.engine import Engine
    e = Engine(0)
    e.set_mma_mode(request.param)
    return e


@pytest.fixture(scope='module')
def eng1():
    from cycle_diffusion_b200.engine import Engine
    return Engine(0)


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / max(1e-30, float(b.double().abs().max())))


def relmax(a, b):
    return float((a.double() - b.double()).abs().max() / max(1.0, float(b.double().abs().max())))


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


def run_conv(e, x, w, b, stride, pad_lo):
    e.profile(True)
    y = nchw(e.op_conv3x3(nhwc(x).cuda(), w.cuda(), b.cuda(), stride, pad_lo, 1).cpu())
    fam = e.profile_read()
    e.profile(False)
    assert 'conv3x3_tc' in fam and 'conv3x3_ffma' not in fam, f'tensor-core path was not taken: {sorted(fam)}'
    return y


@pytest.mark.parametrize('B,Cin,Cout,H,W', [
    (2, 64, 64, 24, 40), (2, 64, 64, 40, 24), (1, 128, 96, 96, 96),       # rectangular / non-power-of-two maps
    (1, 64, 128, 16, 40), (2, 96, 64, 10, 80),                            # widths above 16, not multiples of 16
    (8, 64, 64, 3, 5), (8, 128, 96, 6, 10),                               # tiny maps, several images per 128-row tile
    (2, 1280, 640, 6, 10),                                                # K-heavy: split-K partials of masked tiles
    (3, 64, 100, 24, 40), (2, 160, 36, 12, 20)])                          # ragged N tiles
def test_conv3x3_tc_any_size(eng, B, Cin, Cout, H, W):
    g = torch.Generator().manual_seed(Cin * 1000 + Cout + H * 7 + W)
    x = torch.randn(B, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / math.sqrt(9 * Cin)
    b = torch.randn(Cout, generator=g)
    y = run_conv(eng, x, w, b, 1, 1)
    r = rel(y, F.conv2d(x, w, b, padding=1))
    print(f'conv_tc B{B} {Cin}->{Cout} @{H}x{W}: rel {r:.2e}')
    assert r < 2e-5


@pytest.mark.parametrize('pad', [1, 0], ids=['oai_pad1', 'vae_pad0101'])
def test_conv3x3_tc_downsample_any_size(eng, pad):
    """Stride-2 downsample of a 48x80 map: OAI Downsample (padding 1) and the VAE's asymmetric (0,1,0,1) pad then padding 0."""
    g = torch.Generator().manual_seed(48 + pad)
    x = torch.randn(2, 64, 48, 80, generator=g)
    w = torch.randn(64, 64, 3, 3, generator=g) / math.sqrt(9 * 64)
    b = torch.randn(64, generator=g)
    y = run_conv(eng, x, w, b, 2, pad)
    ref = F.conv2d(x, w, b, stride=2, padding=1) if pad == 1 else F.conv2d(F.pad(x, (0, 1, 0, 1)), w, b, stride=2)
    assert y.shape == ref.shape == (2, 64, 24, 40)
    r = rel(y, ref)
    print(f'downsample pad {pad} 48x80: rel {r:.2e}')
    assert r < 2e-5


def test_conv3x3_tc_after_materialised_upsample(eng):
    """The networks' Upsample on the tensor-core path: nearest-2x of a 12x20 map materialised, then the plain conv at 24x40."""
    g = torch.Generator().manual_seed(1220)
    x = torch.randn(2, 128, 12, 20, generator=g)
    w = torch.randn(64, 128, 3, 3, generator=g) / math.sqrt(9 * 128)
    b = torch.randn(64, generator=g)
    xu = F.interpolate(x, scale_factor=2.0, mode='nearest')
    y = run_conv(eng, xu, w, b, 1, 1)
    r = rel(y, F.conv2d(xu, w, b, padding=1))
    print(f'upsampled 12x20 -> 24x40: rel {r:.2e}')
    assert r < 2e-5


def _conv_ffma(e, net, x, t, ctx):
    e.profile(True)
    y = net(x, t, ctx).cpu()
    fam = e.profile_read()
    e.profile(False)
    return y, fam.get('conv3x3_ffma', {}).get('launches', 0)


@pytest.mark.parametrize('name,cfg', [('unet_sd_rect', NARROW), ('unet_sd_wide_rect', WIDE)])
def test_unet_rect_vs_reference_fixture(eng, name, cfg):
    """SD-topology U-Nets at latent 24x40 (960-token self-attention: ragged query blocks) against the reference UNetModel."""
    from cycle_diffusion_b200.engine import UNet
    g = golden(name)
    sd = specs.synth_state_dict(specs.openai_unet_params(cfg), int(g['seed']))
    net = UNet(eng, cfg, 'openai').load_state_dict(sd)
    y, _ = _conv_ffma(eng, net, g['x'], g['t'], g['ctx'])
    r = relmax(y, g['y'])
    print(f'{name}: rel max err vs reference fixture {r:.3e}')
    assert r < 2e-4
    # no conv of the 24x40 call leaves the tensor cores for a reason the 32x32 call does not have (batch 3: both sizes fall on the
    # same side of the small-problem rule, M < 2048 rows with fewer than 32 output channels)
    gen = torch.Generator().manual_seed(7)
    t = torch.tensor([501., 11., 3.])
    ctx = torch.randn(3, 77, cfg['context_dim'], generator=gen)
    _, n_rect = _conv_ffma(eng, net, torch.randn(3, 4, 24, 40, generator=gen), t, ctx)
    _, n_sq = _conv_ffma(eng, net, torch.randn(3, 4, 32, 32, generator=gen), t, ctx)
    print(f'{name}: conv3x3_ffma launches 24x40 {n_rect}, 32x32 {n_sq}')
    assert n_rect <= n_sq


def test_vae_rect_vs_reference_fixture(eng1):
    from cycle_diffusion_b200.engine import VAE
    g = golden('vae_rect')
    sd = specs.synth_state_dict(specs.kl_vae_params(VAE_SMALL), int(g['seed']))
    vae = VAE(eng1, VAE_SMALL).load_state_dict(sd)
    m = vae.encode_moments(g['img']).cpu()
    r = vae.decode(g['z']).cpu()
    assert m.shape == g['moments'].shape and r.shape == g['rec'].shape == (1, 3, 96, 160)
    print(f'vae 96x160: moments {relmax(m, g["moments"]):.3e} rec {relmax(r, g["rec"]):.3e}')
    assert relmax(m, g['moments']) < 2e-4
    assert relmax(r, g['rec']) < 2e-4
    with pytest.raises(AssertionError, match='multiples of 8'):      # CDX_E_INVALID: sides must be multiples of 8 here
        vae.encode_moments(torch.zeros(1, 3, 96, 156))


def _sd_wrapper(eng, cond):
    from cycle_diffusion_b200.wrappers import SDStochasticTextWrapper
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    vsd = specs.synth_state_dict(specs.kl_vae_params(VAE_SMALL), 21)
    sd = {'model.diffusion_model.' + k: v for k, v in usd.items()}
    sd.update({'first_stage_model.' + k: v for k, v in vsd.items()})
    w = SDStochasticTextWrapper('synthetic', custom_steps=4, eta=0.1, white_box_steps=5, skip_steps=[0], encoder_unconditional_guidance_scales=[1],
                                decoder_unconditional_guidance_scales=[1], n_trials=1, engine=eng, state_dict=sd, cond_stage=cond,
                                unet_config=NARROW, vae_config=VAE_SMALL, latent_size=16, resolution=128)
    return w, usd, vsd


def test_pipeline_rect_identity_cycle(eng1):
    """Same prompt, guidance 1, on a 192x320 image (latent 24x40): the output is decode(encode(image))."""
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    from cycle_diffusion_b200.wrappers import SyntheticTextEncoder
    w, _, _ = _sd_wrapper(eng1, SyntheticTextEncoder(48))
    pipe = CycleDiffusionPipeline.from_wrapper(w)
    image = torch.rand(1, 3, 192, 320, generator=torch.Generator().manual_seed(4))
    out = pipe('a cat', 'a cat', image, strength=0.75, num_inference_steps=8, guidance_scale=1.0, source_guidance_scale=1.0, eta=0.1,
               generator=torch.Generator().manual_seed(9))
    g = w.generator
    gen = torch.Generator().manual_seed(9)
    mom = g.encode_first_stage(eng1.shift_scale(image, -0.5, 2.0))
    assert mom.shape == (1, 8, 24, 40)
    x0 = eng1.vae_posterior(mom, torch.randn(1, 4, 24, 40, generator=gen), 0.18215)
    rec = eng1.shift_scale(g.decode_first_stage(x0), 1.0, 0.5).clamp(0, 1)
    assert out.images.shape == (1, 3, 192, 320)
    d = maxdiff(out.images.cpu(), rec.cpu())
    print(f'pipeline 192x320 identity cycle: |d img| {d:.2e}')
    assert d < 1e-3
    with pytest.raises(ValueError, match='multiples of 64'):
        pipe('a', 'b', torch.rand(1, 3, 200, 320))


def test_pipeline_rect_vs_oracle(eng1):
    """A translating call on two 192x320 images against the oracle's restatement (VAE encode -> posterior sample -> DPM-Encoder
    under the source prompt -> CFG decode under the target prompt -> VAE decode), same generator seed."""
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    from cycle_diffusion_b200.wrappers import SyntheticTextEncoder
    from oracle import dpm_encoder, unet_openai, vae_kl
    cond = SyntheticTextEncoder(48)
    w, usd, vsd = _sd_wrapper(eng1, cond)
    pipe = CycleDiffusionPipeline.from_wrapper(w)
    image = torch.rand(2, 3, 192, 320, generator=torch.Generator().manual_seed(4))
    S, strength, gs, sgs = 8, 0.75, 4.0, 1.0
    src, tgt = ['a cat', 'a blue car'], ['a dog', 'a red car']
    out = pipe(tgt, src, image, strength=strength, num_inference_steps=S, guidance_scale=gs, source_guidance_scale=sgs, eta=0.1,
               generator=torch.Generator().manual_seed(9)).images.cpu()
    skip = S - int(S * strength)
    unet_fn = lambda x, t, c: unet_openai.unet_forward(usd, NARROW, x, t, c)
    sf = 0.18215
    torch.manual_seed(9)
    with torch.no_grad():
        mean, logvar = torch.chunk(vae_kl.encode_moments(vsd, VAE_SMALL, (image - 0.5) * 2.0), 2, dim=1)
        std = torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0))
        x0 = sf * (mean + std * torch.randn(mean.shape))
        uc, c = cond(2 * ['']), cond(src)
        z = torch.stack(dpm_encoder.latent_encode(unet_fn, x0, c, uc, S, 0.1, skip, S + 1, sgs), dim=1)
        uc, c = cond(2 * ['']), cond(tgt)
        sample = dpm_encoder.latent_decode(unet_fn, z[:, 0], z[:, 1:], c, uc, S, 0.1, skip, gs)
        ref = ((vae_kl.decode(vsd, VAE_SMALL, 1. / sf * sample) + 1.0) / 2.0).clamp(0, 1)
    d = maxdiff(out, ref)
    print(f'pipeline 192x320 vs oracle: |d img| {d:.2e}')
    assert out.shape == ref.shape == (2, 3, 192, 320)
    assert d < 1e-3
