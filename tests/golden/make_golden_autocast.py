#!/usr/bin/env python
"""Generate the mixed-precision ("autocast") golden fixtures by running the REAL reference modules on the CPU under CUDA
autocast's cast policy.

Run in the build container only (``/root/reference`` is not present on the GPU box):

    python tests/golden/make_golden_autocast.py

The reference's SD wrapper and txt2img.py run encode / generate inside ``torch.autocast("cuda")`` when ``precision ==
"autocast"``.  CPU ``torch.autocast`` is not the same policy (it leaves softmax, GroupNorm and LayerNorm in fp16), so the
reference modules run here under ``CudaAutocastPolicy``, a TorchFunctionMode that applies the CUDA policy to CPU tensors:
  * convolutions, linear, matmul / mm / bmm / baddbmm / einsum: floating inputs cast to fp16 (fp16 output);
  * softmax / log_softmax / group_norm / layer_norm / exp / log / pow / sum and the rest of CUDA autocast's fp32 list:
    floating inputs cast to fp32 (fp32 output);
  * every other op: normal type promotion (so GroupNorm32's ``.type(x.dtype)`` returns fp16, as on the GPU).
This reproduces the policy -- which op sees which dtype -- not cuDNN's or cuBLAS's summation order.

Every fixture stores the fp32 output and the policy's output of the same inputs (same modules, shims and synthetic weights
as ``make_golden.py``):
  * unet_sd_autocast.npz: the WIDE SD-topology UNetModel at latent 32x32 (d = 40 at 1024 tokens, d = 80 at 256 tokens) and
    the NARROW one at 32x32 with B = 2;
  * vae_autocast.npz: the small KL VAE, encode (64x64 image) and decode (8x8 latent);
  * ddim_cycle_autocast.npz: a NARROW latent cycle through DDIMSampler (every step recovered, CFG on the target chain), torch-seeded
    noise as in make_golden.golden_ddim_cycle.
Nothing from the reference is copied into the repo; only numeric outputs are stored.
"""
import os
import sys

import numpy as np
import torch
from torch.overrides import TorchFunctionMode

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402
from make_golden import NARROW, VAE_SMALL, WIDE, _LatentStandIn, _quiet, build_ref_unet, save, sd_checksum, specs  # noqa: E402

# CUDA autocast's lower-precision list (the ops these modules reach) and its fp32 lists (fp32, fp32_set_opt_dtype, fp32_append_dtype)
F16_OPS = {'conv1d', 'conv2d', 'conv3d', 'conv_transpose1d', 'conv_transpose2d', 'conv_transpose3d', 'convolution', 'linear', 'matmul',
           '__matmul__', 'mm', 'mv', 'bmm', 'baddbmm', 'addmm', 'addmv', 'addbmm', 'addr', 'einsum', 'chain_matmul', 'prelu',
           'scaled_dot_product_attention'}
F32_OPS = {'softmax', 'log_softmax', 'group_norm', 'layer_norm', 'exp', 'expm1', 'log', 'log10', 'log2', 'log1p', 'pow', '__pow__',
           '__rpow__', 'reciprocal', 'rsqrt', 'acos', 'asin', 'cosh', 'sinh', 'tan', 'erfinv', 'softplus', 'sum', 'prod', 'cumsum',
           'cumprod', 'logsumexp', 'norm', 'frobenius_norm', 'nuclear_norm', 'cosine_similarity', 'dist', 'pdist', 'cdist', 'renorm',
           'mse_loss', 'l1_loss', 'smooth_l1_loss', 'huber_loss', 'kl_div', 'nll_loss', 'binary_cross_entropy_with_logits'}


def _cast(x, dt):
    if torch.is_tensor(x):
        return x.to(dt) if x.dtype in (torch.float16, torch.float32) and x.dtype != dt else x
    if isinstance(x, (list, tuple)):
        return type(x)(_cast(v, dt) for v in x)
    return x


class CudaAutocastPolicy(TorchFunctionMode):
    def __torch_function__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        name = getattr(func, '__name__', '')
        dt = torch.float16 if name in F16_OPS else torch.float32 if name in F32_OPS else None
        if dt is None:
            return func(*args, **kwargs)
        return func(*_cast(args, dt), **{k: _cast(v, dt) for k, v in kwargs.items()})


def both(fn):
    """(fp32 output, policy output as fp32) of fn()."""
    with torch.no_grad():
        y32 = fn()
        with CudaAutocastPolicy():
            yac = fn()
    return y32, yac.float()


def rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


def golden_unets_autocast():
    out = {}
    for tag, cfg, seed, B in (('wide', WIDE, 12, 1), ('narrow', NARROW, 11, 2)):
        sd = specs.synth_state_dict(specs.openai_unet_params(cfg), seed)
        m = build_ref_unet(cfg)
        m.load_state_dict(sd, strict=True)
        g = torch.Generator().manual_seed(500 + seed)
        x = torch.randn(B, cfg['in_channels'], 32, 32, generator=g)
        ctx = torch.randn(B, 77, cfg['context_dim'], generator=g)
        t = torch.tensor([901, 21][:B], dtype=torch.long)
        y32, yac = both(lambda: m(x, t, context=ctx))
        print(f'unet[{tag}]: autocast vs fp32 rel {rel(yac, y32):.2e}')
        out.update({f'x_{tag}': x, f't_{tag}': t, f'ctx_{tag}': ctx, f'y32_{tag}': y32, f'yac_{tag}': yac, f'seed_{tag}': seed,
                    f'wsum_{tag}': sd_checksum(sd)})
    save('unet_sd_autocast', **out)


def golden_vae_autocast():
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
    g = torch.Generator().manual_seed(621)
    img = torch.rand(2, 3, 64, 64, generator=g) * 2 - 1
    z = torch.randn(2, 4, 8, 8, generator=g)
    m32, mac = both(lambda: quant(enc(img)))          # AutoencoderKL.encode
    r32, rac = both(lambda: dec(post(z)))             # AutoencoderKL.decode
    print(f'vae: autocast vs fp32 rel moments {rel(mac, m32):.2e} rec {rel(rac, r32):.2e}')
    save('vae_autocast', img=img, z=z, moments32=m32, momentsac=mac, rec32=r32, recac=rac, seed=21, wsum=sd_checksum(sd))


def golden_ddim_cycle_autocast():
    from ldm.models.diffusion.ddim import DDIMSampler

    class CPUSampler(DDIMSampler):
        def register_buffer(self, name, attr):      # stock one forces .to("cuda"), ddim.py:19-23
            setattr(self, name, attr)

    cfg = NARROW
    sd = specs.synth_state_dict(specs.openai_unet_params(cfg), 11)
    unet = build_ref_unet(cfg)
    unet.load_state_dict(sd, strict=True)
    model = _LatentStandIn(unet)
    g = torch.Generator().manual_seed(641)
    B, S, skip, wb, enc_scale, dec_scale, seed = 2, 10, 3, 11, 1.0, 3.0, 1010
    x0 = torch.randn(B, 4, 16, 16, generator=g) * 0.8
    c_src = torch.randn(B, 77, 48, generator=g)
    c_tgt = torch.randn(B, 77, 48, generator=g)
    uc = torch.randn(B, 77, 48, generator=g)

    def cycle():
        torch.manual_seed(seed)
        with _quiet():
            z_list = CPUSampler(model).ddpm_ddim_encoding(S, conditioning=c_src, batch_size=B, shape=(4, 16, 16), eta=0.1,
                                                          white_box_steps=wb, skip_steps=skip, verbose=False, x0=x0,
                                                          unconditional_guidance_scale=enc_scale, unconditional_conditioning=uc)
            z = torch.stack(z_list, dim=1).view(B, -1)                       # SDW:203
            eps_list = z.view(B, wb - skip, 4, 16, 16)                         # SDW:150
            tgt, _ = CPUSampler(model).sample_with_eps(S, eps_list[:, 1:], conditioning=c_tgt, batch_size=B, shape=(4, 16, 16),
                                                       eta=0.1, verbose=False, x_T=eps_list[:, 0], skip_steps=skip,
                                                       unconditional_guidance_scale=dec_scale, unconditional_conditioning=uc)
        return z.float(), tgt.float()

    with torch.no_grad():
        z32, t32 = cycle()
        with CudaAutocastPolicy():
            zac, tac = cycle()
    print(f'ddim_cycle: autocast vs fp32 rel z {rel(zac, z32):.2e} tgt {rel(tac, t32):.2e}')
    save('ddim_cycle_autocast', x0=x0, c_src=c_src, c_tgt=c_tgt, uc=uc, z32=z32, zac=zac, tgt32=t32, tgtac=tac,
         cfg=np.asarray([S, skip, wb, enc_scale, dec_scale, seed], dtype=np.float64))


if __name__ == '__main__':
    mg._shim_omegaconf()
    sys.path.insert(0, os.path.join(mg.REF, 'model/lib/stable_diffusion'))
    golden_unets_autocast()
    golden_vae_autocast()
    golden_ddim_cycle_autocast()
