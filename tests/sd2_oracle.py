"""CPU fp32 restatements of the SD 2.x additions, for the tests and tests/golden/make_golden_sd2.py (test infrastructure only).

  * unet_forward: SD 2 UNetModel.forward (v2-inference.yaml unet_config): the oracle.unet_openai network with the head count
    derived per level as C / num_head_channels and the Linear proj_in / proj_out weights [C, C] applied as the 1x1 convolutions
    they are equivalent to on NCHW (GroupNorm -> rearrange -> Linear == 1x1 conv -> rearrange).
  * latent_encode / latent_decode with prediction='v': oracle.dpm_encoder's loops with the U-Net output read as v.  After the
    guidance combine (ddim.py:550-559) the output of a step at timestep t becomes
        e_t     = sa_v[t] * v + s1_v[t] * x_t
        pred_x0 = sa_v[t] * x_t - s1_v[t] * v
    with sa_v = fp32(sqrt(abar)), s1_v = fp32(sqrt(1 - abar)) of the float64 abar (LatentDiffusion.predict_eps_from_z_and_v /
    predict_start_from_z_and_v over register_schedule's buffers); compute_eps and p_sample_ddim_with_eps are otherwise unchanged.
    Every product is a separate fp32 torch op, as the engine's step kernels round them.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import unet_openai as U
from oracle.dpm_encoder import _coeffs, _guided_eps, latent_sample_xt_next
from oracle.schedules import DDIMTables


def _conv_proj(sd):
    return {k: (v[:, :, None, None] if k.endswith(('.proj_in.weight', '.proj_out.weight')) and v.dim() == 2 else v) for k, v in sd.items()}


def unet_forward(sd, cfg, x, timesteps, context):
    """x [B,4,h,w], timesteps [B], context [B,L,D] -> [B,4,h,w] under an SD 2-shaped config (num_head_channels, Linear projections)."""
    sd = _conv_proj(sd)
    hc = cfg['num_head_channels']
    inp, mid, outb = U.plan(cfg)
    emb = U._lin(sd, 'time_embed.2', F.silu(U._lin(sd, 'time_embed.0', U.timestep_embedding(timesteps, cfg['model_channels']))))

    def run(block, bp, h):
        for li, kind in enumerate(block):
            p = f'{bp}.{li}'
            if kind == 'conv':
                h = U._conv(sd, p, h)
            elif kind == 'res':
                h = U._resblock(sd, p, h, emb)
            elif kind == 'st':
                h = U._spatial_transformer(sd, p, h, context, h.shape[1] // hc)
            elif kind == 'down':
                h = U._conv(sd, p + '.op', h, stride=2, padding=1)
            elif kind == 'up':
                h = U._conv(sd, p + '.conv', F.interpolate(h, scale_factor=2, mode='nearest'))
        return h

    hs, h = [], x
    for i, block in enumerate(inp):
        h = run(block, f'input_blocks.{i}', h)
        hs.append(h)
    h = run(mid, 'middle_block', h)
    for i, block in enumerate(outb):
        h = run(block, f'output_blocks.{i}', torch.cat([h, hs.pop()], dim=1))
    return U._conv(sd, 'out.2', F.silu(U._gn(sd, 'out.0', h, 1e-5)))


def v_tables():
    """fp32(sqrt(abar_t)), fp32(sqrt(1 - abar_t)) of the LDM linear schedule's float64 abar (0.00085 -> 0.012, 1000 steps)."""
    betas = np.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=np.float64) ** 2
    ac = np.cumprod(1.0 - betas)
    return torch.tensor(np.sqrt(ac), dtype=torch.float32), torch.tensor(np.sqrt(1.0 - ac), dtype=torch.float32)


def _eps_x0(out, x, t, index, tab, b, prediction):
    """(e_t, pred_x0) of one step from the guidance-combined output."""
    a_t, _, _, sqrt_1m_at = _coeffs(tab, index, b)
    if prediction == 'eps':
        return out, (x - sqrt_1m_at * out) / a_t.sqrt()
    SA, S1 = v_tables()
    sa, s1 = torch.full((b, 1, 1, 1), float(SA[t])), torch.full((b, 1, 1, 1), float(S1[t]))
    return sa * out + s1 * x, sa * x - s1 * out


def latent_encode(unet_fn, x0, c, uc, S, eta, skip_steps, scale, prediction='eps'):
    """_ddpm_ddim_encoding with every step recovered -> z_list = [x_T, eps_0, ..., eps_last]."""
    tab = DDIMTables(S, eta)
    b = x0.shape[0]
    refine_steps = tab.timesteps.shape[0] - skip_steps
    at = tab.alphas[refine_steps - 1]
    xt = at.sqrt() * x0 + (1 - at).sqrt() * torch.randn(x0.shape)
    z_list = [xt]
    for i, step in enumerate(np.flip(tab.timesteps)[-refine_steps:]):
        index = refine_steps - i - 1
        xt_next = latent_sample_xt_next(tab, x0, xt, index)
        out = _guided_eps(unet_fn, xt, torch.full((b,), int(step), dtype=torch.long), c, uc, scale)
        e_t, pred_x0 = _eps_x0(out, xt, int(step), index, tab, b, prediction)
        _, a_prev, sigma_t, _ = _coeffs(tab, index, b)
        dir_xt = (1. - a_prev - sigma_t ** 2).sqrt() * e_t
        z_list.append((xt_next - a_prev.sqrt() * pred_x0 - dir_xt) / sigma_t / 1.0)
        xt = xt_next
    return z_list


def latent_decode(unet_fn, x_T, eps_list, c, uc, S, eta, skip_steps, scale, prediction='eps'):
    """ddim_sampling_with_eps: eps_list [B, n, C, h, w] (n == the refine steps) -> x0."""
    tab = DDIMTables(S, eta)
    b = x_T.shape[0]
    refine_steps = tab.timesteps.shape[0] - skip_steps
    img = x_T
    for i, step in enumerate(np.flip(tab.timesteps)[-refine_steps:]):
        index = refine_steps - i - 1
        out = _guided_eps(unet_fn, img, torch.full((b,), int(step), dtype=torch.long), c, uc, scale)
        e_t, pred_x0 = _eps_x0(out, img, int(step), index, tab, b, prediction)
        _, a_prev, sigma_t, _ = _coeffs(tab, index, b)
        dir_xt = (1. - a_prev - sigma_t ** 2).sqrt() * e_t
        img = a_prev.sqrt() * pred_x0 + dir_xt + sigma_t * eps_list[:, i] * 1.0
    return img
