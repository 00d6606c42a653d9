"""CPU fp32 restatement of mask-guided local editing on the lock-step loop (test infrastructure only).

The reference has no masking, so this loop is pinned indirectly: it is oracle.dpm_encoder's latent_encode and latent_decode
arithmetic stepped together (the source chain's DPM-Encoder step, then each target chain's p_sample_ddim_with_eps step with the
noise just recovered), and after every step each target x_{t-1} is blended with the source chain's x_{t-1}:

    m == 1  -> target value;   m == 0 -> source value;   else  x + m * (y - x)    (each op a separate fp32 torch op)

with m [B,1,h,w] broadcast over the channels.  With a mask of ones it is latent_encode followed by latent_decode bit for bit; with a
mask of zeros it ends at x0 (the source chain's last x_{t-1} is x0 itself, ddim.py:583-584).  Random draws are made in
latent_encode's order, so ``torch.manual_seed(s)`` before a call matches the engine fed with wrappers.encode_noise under the same seed.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.dpm_encoder import _coeffs, _guided_eps, latent_compute_eps, latent_sample_xt_next
from oracle.schedules import DDIMTables


def blend(y, x, m):
    return torch.where(m == 1, y, torch.where(m == 0, x, x + m * (y - x)))


def masked_cycle(unet_fn, x0, c_src, c_tgt, uc, S, eta, skip_steps, src_scale, tgt_scales, mask, alphas_cumprod=None):
    """One source chain (c_src at src_scale) driving one target chain per entry of tgt_scales (c_tgt), every step recovered.
    mask [B,1,h,w] or None (unmasked).  -> (list of target latents [B,C,h,w], z_list as latent_encode returns it)."""
    assert eta > 0
    tab = DDIMTables(S, eta, alphas_cumprod)
    b = x0.shape[0]
    refine_steps = tab.timesteps.shape[0] - skip_steps
    at = tab.alphas[refine_steps - 1]
    xt = at.sqrt() * x0 + (1 - at).sqrt() * torch.randn(x0.shape)
    z_list, ys = [xt], [xt] * len(tgt_scales)
    for i, step in enumerate(np.flip(tab.timesteps)[-refine_steps:]):
        index = refine_steps - i - 1
        ts = torch.full((b,), int(step), dtype=torch.long)
        xt_next = latent_sample_xt_next(tab, x0, xt, index)
        eps = latent_compute_eps(tab, unet_fn, xt, xt_next, c_src, uc, ts, index, src_scale)
        z_list.append(eps)
        a_t, a_prev, sigma_t, sqrt_1m_at = _coeffs(tab, index, b)
        for k, scale in enumerate(tgt_scales):
            img = ys[k]
            e_t = _guided_eps(unet_fn, img, ts, c_tgt, uc, scale)
            pred_x0 = (img - sqrt_1m_at * e_t) / a_t.sqrt()
            dir_xt = (1. - a_prev - sigma_t ** 2).sqrt() * e_t
            y = a_prev.sqrt() * pred_x0 + dir_xt + sigma_t * eps * 1.
            ys[k] = y if mask is None else blend(y, xt_next, mask)
        xt = xt_next
    return ys, z_list


def masked_search(ora, image01, encode_text, decode_text, mask01, factor):
    """The ensemble of oracle.dpm_encoder.LatentCycle member by member, every member's target chains under the image-resolution
    mask pooled to the latent grid (avg_pool2d over factor x factor blocks).  Same draws in the same order as ora.encode.
    -> post-processed candidates (x + 1) / 2 in candidate order (member * n_dec + k)."""
    x0 = ora.first_stage_encode(image01)
    m = F.avg_pool2d(mask01, factor)
    bsz = image01.shape[0]
    imgs = []
    for _ in range(ora.n_trials):
        for enc_scale in ora.enc_scales:
            for skip in ora.skip_steps:
                uc = ora.cond_fn(bsz * [""])
                c_src, c_tgt = ora.cond_fn(encode_text), ora.cond_fn(decode_text)
                ys, _ = masked_cycle(ora.unet_fn, x0, c_src, c_tgt, uc, ora.custom_steps, ora.eta, skip, enc_scale, ora.dec_scales, m,
                                     ora.alphas_cumprod)
                imgs += [(ora.vae_decode_fn(1. / ora.scale_factor * y) + 1.0) / 2.0 for y in ys]
    return imgs
