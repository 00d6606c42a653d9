#!/usr/bin/env python
"""Generate the rectangular-image golden fixtures by running the REAL reference modules (CPU, fp32).

Run in the build container only (``/root/reference`` is not present on the GPU box):

    python tests/golden/make_golden_rect.py

Same modules, shims, synthetic weights and save format as ``make_golden.py`` (whose helpers it imports), at sizes whose sides are
not powers of two and not equal:
  * unet_sd_rect.npz / unet_sd_wide_rect.npz: the NARROW / WIDE SD-topology UNetModel at latent 24x40 (960 tokens at the first
    attention level);
  * vae_rect.npz: the small KL VAE Encoder on a 96x160 image and Decoder on a 12x20 latent.
Nothing from the reference is copied into the repo; only numeric outputs are stored.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402
from make_golden import NARROW, VAE_SMALL, WIDE, _quiet, build_ref_unet, save, sd_checksum, specs  # noqa: E402


def golden_unets_rect():
    for name, cfg, seed, B in (('unet_sd_rect', NARROW, 11, 2), ('unet_sd_wide_rect', WIDE, 12, 1)):
        sd = specs.synth_state_dict(specs.openai_unet_params(cfg), seed)
        m = build_ref_unet(cfg)
        m.load_state_dict(sd, strict=True)
        g = torch.Generator().manual_seed(300 + seed)
        x = torch.randn(B, cfg['in_channels'], 24, 40, generator=g)
        ctx = torch.randn(B, 77, cfg['context_dim'], generator=g)
        t = torch.tensor([901, 21][:B], dtype=torch.long)
        with torch.no_grad():
            y = m(x, t, context=ctx)
        save(name, x=x, t=t, ctx=ctx, y=y, seed=seed, wsum=sd_checksum(sd))


def golden_vae_rect():
    from ldm.modules.diffusionmodules.model import Encoder, Decoder
    cfg = VAE_SMALL
    sd = specs.synth_state_dict(specs.kl_vae_params(cfg), 21)
    dd = dict(double_z=True, z_channels=cfg['z_channels'], resolution=64, in_channels=3, out_ch=3, ch=cfg['ch'],
              ch_mult=list(cfg['ch_mult']), num_res_blocks=cfg['num_res_blocks'], attn_resolutions=[], dropout=0.0)
    with _quiet():
        enc, dec = Encoder(**dd).eval(), Decoder(**dd).eval()
    enc.load_state_dict({k[len('encoder.'):]: v for k, v in sd.items() if k.startswith('encoder.')}, strict=True)
    dec.load_state_dict({k[len('decoder.'):]: v for k, v in sd.items() if k.startswith('decoder.')}, strict=True)
    quant = torch.nn.Conv2d(2 * cfg['z_channels'], 2 * cfg['embed_dim'], 1)
    post = torch.nn.Conv2d(cfg['embed_dim'], cfg['z_channels'], 1)
    quant.load_state_dict({'weight': sd['quant_conv.weight'], 'bias': sd['quant_conv.bias']})
    post.load_state_dict({'weight': sd['post_quant_conv.weight'], 'bias': sd['post_quant_conv.bias']})
    g = torch.Generator().manual_seed(321)
    img = torch.rand(1, 3, 96, 160, generator=g) * 2 - 1
    z = torch.randn(1, 4, 12, 20, generator=g)
    with torch.no_grad():
        moments = quant(enc(img))           # AutoencoderKL.encode
        rec = dec(post(z))                  # AutoencoderKL.decode
    save('vae_rect', img=img, z=z, moments=moments, rec=rec, seed=21, wsum=sd_checksum(sd))


if __name__ == '__main__':
    mg._shim_omegaconf()
    sys.path.insert(0, os.path.join(mg.REF, 'model/lib/stable_diffusion'))
    golden_unets_rect()
    golden_vae_rect()
