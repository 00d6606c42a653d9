"""Parity at the REAL shapes of the BASELINE configurations (not the reduced test topologies): the networks the bench is
quoted on are compared with the CPU oracle on the box's host cores, through the same C ABI the bench uses.

  (i)   SD v1-4 U-Net (859 M params, specs.sd_unet_config(768)), latent 64x64, B=2 distinct contexts      OAI:710-742
  (ii)  KL-f8 VAE encode + decode of one 512x512 image (d=512 / N=4096 attention, asym-pad s2 convs)       AEM:434-459, 535-568
  (iii) improved-DDPM 256x256 U-Net forward                                                               IU:639-668
  (iv)  LDM text2img-large U-Net (context 1280), latent 32x32                                              OAI:710-742
  (v)   a short (2+2 steps) BASELINE config-2 cycle through SDStochasticTextWrapper                        SDW:169-249, BASELINE.md section 3
  (vi)  UnsupervisedTranslation with two improved-DDPM 256x256 wrappers (config 5 API)                     unsupervised_translation.py:27-55

Tolerances: 2e-4 relative to the output's max magnitude for single forwards, 1e-3 absolute on decoded images / latents
(the north-star bar).  Every check prints its measured error."""
import pytest
import torch

from cycle_diffusion_b200 import specs
from tests.common import maxdiff

pytestmark = pytest.mark.gpu
TOL = 2e-4


@pytest.fixture(scope='module')
def eng():
    from cycle_diffusion_b200.engine import Engine
    return Engine(0)


def relmax(a, b):
    return float((a.double() - b.double()).abs().max() / max(1e-30, float(b.double().abs().max())))


@pytest.fixture(scope='module')
def sd_unet(eng):
    from cycle_diffusion_b200.engine import UNet
    cfg = specs.sd_unet_config(768)
    sd = specs.synth_state_dict(specs.openai_unet_params(cfg), 1234)
    return cfg, sd, UNet(eng, cfg, 'openai').load_state_dict(sd)


@pytest.fixture(scope='module')
def kl_f8(eng):
    from cycle_diffusion_b200.engine import VAE
    cfg = specs.kl_f8_config()
    sd = specs.synth_state_dict(specs.kl_vae_params(cfg), 1235)
    return cfg, sd, VAE(eng, cfg).load_state_dict(sd)


def _families(eng, fn):
    eng.profile(True)
    out = fn()
    fam = eng.profile_read()
    eng.profile(False)
    return out, fam


def test_sd_v14_unet_full_size(eng, sd_unet):
    """(i) the 859 M-parameter U-Net at the CFG launch shape (two samples, distinct contexts and timesteps)."""
    from oracle import unet_openai
    cfg, sd, net = sd_unet
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 64, 64, generator=g)
    ctx = torch.randn(2, 77, 768, generator=g)
    t = torch.tensor([981., 21.])
    y, fam = _families(eng, lambda: net(x, t, ctx).cpu())
    with torch.no_grad():
        ref = unet_openai.unet_forward(sd, cfg, x, t.long(), ctx)
    r = relmax(y, ref)
    print(f'SD v1-4 U-Net 64x64 B2: rel max err vs oracle {r:.3e}  (|ref|max {float(ref.abs().max()):.3f}) families {sorted(fam)}')
    assert 'conv3x3_tc' in fam and 'dense_tc' in fam, f'tensor-core path not taken: {fam}'
    assert not [k for k in fam if k.endswith('ffma') and fam[k]['flops'] > 0.02 * fam['conv3x3_tc']['flops']], f'large FFMA share: {fam}'
    assert r < TOL


def test_kl_f8_vae_512(eng, kl_f8):
    """(ii) one 512x512 image through the full-width VAE; the mid-block attention (d=512, 4096 tokens) must run on tensor cores."""
    from oracle import vae_kl
    cfg, sd, vae = kl_f8
    g = torch.Generator().manual_seed(1)
    img = torch.rand(1, 3, 512, 512, generator=g) * 2 - 1
    z = torch.randn(1, 4, 64, 64, generator=g)
    (m, rec), fam = _families(eng, lambda: (vae.encode_moments(img).cpu(), vae.decode(z).cpu()))
    with torch.no_grad():
        m_ref = vae_kl.encode_moments(sd, cfg, img)
        rec_ref = vae_kl.decode(sd, cfg, z)
    rm, rr = relmax(m, m_ref), relmax(rec, rec_ref)
    print(f'KL-f8 @512: moments rel {rm:.3e}  decode rel {rr:.3e}  abs {maxdiff(rec, rec_ref):.3e}  families {sorted(fam)}')
    assert 'batched_ffma' not in fam, f'the d=512 attention fell back to the FFMA path: {sorted(fam)}'
    assert rm < TOL and rr < TOL


def test_iddpm_256_unet(eng):
    """(iii) the 256x256 improved-DDPM U-Net of BASELINE config 5."""
    from cycle_diffusion_b200.engine import UNet
    from oracle import unet_iddpm
    cfg = specs.iddpm_config(256)
    sd = specs.synth_state_dict(specs.iddpm_unet_params(cfg), 4321)
    net = UNet(eng, cfg, 'iddpm').load_state_dict(sd)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1, 3, 256, 256, generator=g)
    t = torch.tensor([612.])
    y = net(x, t).cpu()
    with torch.no_grad():
        ref = unet_iddpm.unet_forward(sd, cfg, x, t)
    r = relmax(y, ref)
    print(f'i-DDPM 256 U-Net: rel max err vs oracle {r:.3e}')
    assert y.shape == (1, 6, 256, 256)
    assert r < TOL


def test_ldm_text2img_large_unet(eng):
    """(iv) LDM text2img-large: same U-Net topology with context_dim 1280, latent 32x32 (BASELINE config 4)."""
    from cycle_diffusion_b200.engine import UNet
    from oracle import unet_openai
    cfg = specs.sd_unet_config(1280)
    sd = specs.synth_state_dict(specs.openai_unet_params(cfg), 99)
    net = UNet(eng, cfg, 'openai').load_state_dict(sd)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 4, 32, 32, generator=g)
    ctx = torch.randn(2, 77, 1280, generator=g)
    t = torch.tensor([501., 1.])
    y = net(x, t, ctx).cpu()
    with torch.no_grad():
        ref = unet_openai.unet_forward(sd, cfg, x, t.long(), ctx)
    r = relmax(y, ref)
    print(f'LDM text2img-large U-Net 32x32 B2: rel max err vs oracle {r:.3e}')
    assert r < TOL


def test_sd_config2_short_cycle(eng, sd_unet, kl_f8):
    """(v) BASELINE config 2 with 2+2 steps (BASELINE.md section 3): VAE encode + posterior sample + DPM-Encoder under the source
    prompt + CFG-7.5 decode under the target prompt + VAE decode, through the drop-in wrapper, against the oracle's wrapper."""
    from cycle_diffusion_b200.wrappers import SDStochasticTextWrapper, SyntheticTextEncoder, _LatentGenerator
    from oracle import dpm_encoder, unet_openai, vae_kl
    ucfg, usd, unet = sd_unet
    vcfg, vsd, vae = kl_f8
    cond = SyntheticTextEncoder(768)
    kw = dict(custom_steps=2, eta=0.1, white_box_steps=3, skip_steps=[0], encoder_unconditional_guidance_scales=[1.0],
              decoder_unconditional_guidance_scales=[7.5], n_trials=1)
    gen = _LatentGenerator(eng, unet, vae, cond, 4, 64, 0.18215, True)
    w = SDStochasticTextWrapper('synthetic', generator=gen, **kw)
    image = torch.rand(1, 3, 512, 512, generator=torch.Generator().manual_seed(0))
    src, tgt = ['a photo of a cat'], ['a photo of a dog']
    torch.manual_seed(7)
    z_ens = w.encode(image, src)
    img = w(z_ens, image, src, tgt).cpu()
    ora = dpm_encoder.LatentCycle(lambda x, t, c: unet_openai.unet_forward(usd, ucfg, x, t, c),
                                  lambda im: vae_kl.encode_moments(vsd, vcfg, im), lambda zz: vae_kl.decode(vsd, vcfg, zz), cond,
                                  channels=4, latent_size=64, resolution=512, **kw)
    torch.manual_seed(7)
    with torch.no_grad():
        z_ref = ora.encode(image, src)
        img_ref = ora.forward_all(z_ref, tgt)[0]
    rz = maxdiff(z_ens[0].cpu(), z_ref[0]) / float(z_ref[0].abs().max())
    di = maxdiff(img, img_ref)
    print(f'config-2 short cycle: z {tuple(z_ens[0].shape)} rel|dz| {rz:.2e}  |d img| {di:.2e}  (|img|max {float(img_ref.abs().max()):.2f})')
    assert z_ens[0].shape == z_ref[0].shape == (1, 3 * 4 * 64 * 64)
    assert rz < TOL
    assert di < 1e-3


def test_unsupervised_translation_two_iddpm_256(eng):
    """(vi) BASELINE config 5's API: UnsupervisedTranslation.forward with a source and a target 256x256 improved-DDPM wrapper
    (different weights), encode under the source model, decode under the target model."""
    from cycle_diffusion_b200.models import UnsupervisedTranslation
    from oracle import dpm_encoder, unet_iddpm
    cfg = specs.iddpm_config(256)
    sd_src = specs.synth_state_dict(specs.iddpm_unet_params(cfg), 1234)
    sd_tgt = specs.synth_state_dict(specs.iddpm_unet_params(cfg), 4321)
    gan = dict(gan_type='DDPM_DDIM', source_model_type='cat256', target_model_type='dog256', sample_type='ddim', custom_steps=4, es_steps=4,
               eta=0.1)
    m = UnsupervisedTranslation(dict(gan=gan), source_kwargs=dict(engine=eng, state_dict=sd_src, image_size=256),
                                target_kwargs=dict(engine=eng, state_dict=sd_tgt, image_size=256)).eval()
    image = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(5))
    torch.manual_seed(11)
    (orig, img), loss, losses = m(torch.tensor([0, 1]), None, image)
    img = img.cpu()
    kw = dict(sample_type='ddim', custom_steps=4, es_steps=4, eta=0.1, resolution=256)
    src = dpm_encoder.PixelCycle(lambda x, t: unet_iddpm.unet_forward(sd_src, cfg, x, t), **kw)
    tgt = dpm_encoder.PixelCycle(lambda x, t: unet_iddpm.unet_forward(sd_tgt, cfg, x, t), **kw)
    torch.manual_seed(11)
    with torch.no_grad():
        z_ref = src.encode(image)
        img_ref = tgt.forward(z_ref)
    di = maxdiff(img, img_ref)
    print(f'UnsupervisedTranslation 2x i-DDPM 256: |d img| {di:.2e}  (|img|max {float(img_ref.abs().max()):.2f})')
    assert orig is image and img.shape == (2, 3, 256, 256) and loss.shape == (2,) and losses == {}
    assert di < 1e-3
