#!/usr/bin/env python
"""Generate the SD 2.x fixtures (CPU, fp32), the same way make_golden.py does; run in the build container:

    python tests/golden/make_golden_sd2.py

  * unet_sd2_narrow.npz  a narrow SD 2-shaped U-Net (num_head_channels 32: 2 and 4 heads per level, Linear proj_in / proj_out
                         stored [C, C], context width 40) through the reference's own UNetModel(num_head_channels=...), with the
                         projection weights reshaped to its 1x1-conv [C, C, 1, 1] layout; also pins tests/sd2_oracle.unet_forward.
  * openclip_text.npz    a reduced OpenCLIP text tower through transformers.CLIPTextModel(hidden_act="gelu"): output
                         final_layer_norm(hidden_states[-2]); the weights are stored under OpenCLIP names (one extra, unused block)
                         so that the OpenCLIP -> HF mapping is exercised.
  * ddim_cycle_v.npz     an encode / decode cycle of the narrow U-Net under prediction='v' with the tests/sd2_oracle restatement
                         (the reference has no v-prediction sampler): z, the same-condition reconstruction and a target decode.
Only numbers are stored.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from cycle_diffusion_b200 import specs  # noqa: E402
from make_golden import REF, _quiet, _shim_omegaconf, save, sd_checksum  # noqa: E402
from tests import sd2_oracle  # noqa: E402

torch.set_num_threads(8)

NARROW2 = dict(in_channels=4, out_channels=4, model_channels=64, attention_resolutions=(4, 2, 1), num_res_blocks=1,
               channel_mult=(1, 2, 2), num_head_channels=32, context_dim=40, use_linear_in_transformer=True)
OPENCLIP_SMALL = specs.openclip_h14_text_config(layers=2, total_layers=3, vocab_size=1000, width=64, heads=4, mlp_width=256)


def golden_unet_sd2():
    from ldm.modules.diffusionmodules.openaimodel import UNetModel
    cfg = NARROW2
    sd = specs.synth_state_dict(specs.openai_unet_params(cfg), 31)
    with _quiet():
        m = UNetModel(image_size=32, in_channels=4, out_channels=4, model_channels=cfg['model_channels'],
                      attention_resolutions=list(cfg['attention_resolutions']), num_res_blocks=cfg['num_res_blocks'],
                      channel_mult=list(cfg['channel_mult']), num_head_channels=cfg['num_head_channels'], use_spatial_transformer=True,
                      transformer_depth=1, context_dim=cfg['context_dim'], use_checkpoint=False, legacy=False).eval()
    m.load_state_dict(sd2_conv_view(sd), strict=True)
    g = torch.Generator().manual_seed(131)
    x = torch.randn(2, 4, 16, 16, generator=g)
    ctx = torch.randn(2, 77, cfg['context_dim'], generator=g)
    t = torch.tensor([901, 21], dtype=torch.long)
    with torch.no_grad():
        y = m(x, t, context=ctx)
        y_or = sd2_oracle.unet_forward(sd, cfg, x, t, ctx)
    print(f'unet_sd2_narrow: |y|max {y.abs().max():.3f}, oracle max|diff| {(y - y_or).abs().max():.2e}')
    save('unet_sd2_narrow', x=x, t=t, ctx=ctx, y=y, seed=31, wsum=sd_checksum(sd))


def sd2_conv_view(sd):
    return {k: (v[:, :, None, None] if k.endswith(('.proj_in.weight', '.proj_out.weight')) else v) for k, v in sd.items()}


def golden_openclip_text():
    from transformers import CLIPTextConfig, CLIPTextModel
    c = OPENCLIP_SMALL
    hf = CLIPTextConfig(vocab_size=c['vocab_size'], hidden_size=c['width'], intermediate_size=c['mlp_width'],
                        num_hidden_layers=c['total_layers'], num_attention_heads=c['heads'], max_position_embeddings=c['max_len'],
                        hidden_act='gelu', layer_norm_eps=1e-5)
    m = CLIPTextModel(hf).eval()
    oc = specs.synth_state_dict(specs.openclip_text_params(c), 41, gain=2.0)
    full = specs.openclip_to_hf(oc, c['total_layers'])
    want = {k for k in m.state_dict() if not k.endswith('position_ids')}
    assert want == set(full), sorted(want ^ set(full))[:6]
    m.load_state_dict(full, strict=False)
    g = torch.Generator().manual_seed(43)
    ids = torch.randint(0, c['vocab_size'], (3, 77), generator=g)
    with torch.no_grad():
        hs = m(input_ids=ids, output_hidden_states=True).hidden_states
        y = m.text_model.final_layer_norm(hs[-2])            # FrozenOpenCLIPEmbedder layer="penultimate"
    print(f'openclip_text: out {tuple(y.shape)} |y|max {y.abs().max():.3f}')
    save('openclip_text', ids=ids, out=y, seed=41, gain=2.0,
         cfg=np.asarray([c[k] for k in ('vocab_size', 'width', 'layers', 'total_layers', 'heads', 'max_len', 'mlp_width')], dtype=np.int64))


def golden_ddim_cycle_v():
    cfg = NARROW2
    sd = specs.synth_state_dict(specs.openai_unet_params(cfg), 31)
    fn = lambda x, t, cc: sd2_oracle.unet_forward(sd, cfg, x, t, cc)
    g = torch.Generator().manual_seed(151)
    B, S, skip, eta, enc_scale, dec_scale = 2, 8, 2, 0.1, 2.0, 3.0
    x0 = torch.randn(B, 4, 16, 16, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(B, 77, cfg['context_dim'], generator=g) for _ in range(3))
    torch.manual_seed(1200)
    with torch.no_grad():
        z = torch.stack(sd2_oracle.latent_encode(fn, x0, c_src, uc, S, eta, skip, enc_scale, 'v'), dim=1)
        same = sd2_oracle.latent_decode(fn, z[:, 0], z[:, 1:], c_src, uc, S, eta, skip, enc_scale, 'v')
        tgt = sd2_oracle.latent_decode(fn, z[:, 0], z[:, 1:], c_tgt, uc, S, eta, skip, dec_scale, 'v')
    print(f'ddim_cycle_v: same-condition max|x0_hat-x0| = {(same - x0).abs().max():.3e}, |z|max = {z.abs().max():.2f}')
    save('ddim_cycle_v', x0=x0, c_src=c_src, c_tgt=c_tgt, uc=uc, z=z, same=same, tgt=tgt, seed=31, noise_seed=1200,
         cfg=np.asarray([S, skip, eta, enc_scale, dec_scale], dtype=np.float64))


if __name__ == '__main__':
    _shim_omegaconf()
    sys.path.insert(0, os.path.join(REF, 'model/lib/stable_diffusion'))
    golden_unet_sd2()
    golden_openclip_text()
    golden_ddim_cycle_v()
