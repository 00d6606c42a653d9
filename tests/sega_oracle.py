"""CPU fp32 restatement of semantic guidance (SEGA) on the lock-step cycle (test infrastructure only).

The reference has no semantic guidance, so this loop is pinned only by its definition (include/cdx.h, cdx_cycle_lockstep_semantic),
as masked_oracle.py is.  It is masked_oracle.masked_cycle's loop with one target chain and concept rows added: the source and target
U-Net calls are exactly masked_cycle's, and the concept rows (with the target's uncond row when the target runs at scale 1) are
evaluated in a U-Net call of their own, so a CPU convolution that picks its algorithm by batch size sees masked_cycle's batches.

Per step i, with o_uc the target's uncond output and o_k concept k's, every op a separate fp32 torch op:

    psi_k = s_k * (o_k - o_uc);  a_k = |psi_k|;  theta = quantile(a_k over each (image, channel) plane, lambda_k)
    g_k = psi_k where (i < cooldown_k and a_k >= theta) else 0;  S = g_1 + g_2 + ...;  G = S + mu * nu;  nu = beta * nu + beta1 * G
    o-hat = o-hat + G   when i >= warmup

quantile() sorts with torch.sort and interpolates with ATen's scalar lerp; torch.quantile's own CPU lerp is vectorised and may fuse
its multiply-add, so it can differ in the last bit.
"""
import numpy as np
import torch

from oracle.dpm_encoder import _coeffs, latent_sample_xt_next
from oracle.schedules import DDIMTables
from tests.masked_oracle import blend
from tests.sd2_oracle import _eps_x0

F32 = torch.float32


def quantile(a, lam):
    """The lam-quantile of each row of a [..., n] (fp32): r = fp32(lam) * fp32(n - 1), the floor(r)-th and ceil(r)-th smallest
    values, w = r - floor(r), then w < 0.5 ? lo + w (hi - lo) : hi - (hi - lo)(1 - w).  -> [...]."""
    n = a.shape[-1]
    v = torch.sort(a, dim=-1).values
    r = torch.tensor(lam, dtype=F32) * torch.tensor(float(n - 1), dtype=F32)
    lo_f = torch.floor(r)
    w = r - lo_f
    lo, hi = int(lo_f), int(torch.ceil(r))
    v_lo, v_hi = v[..., lo], v[..., hi]
    d = v_hi - v_lo
    if float(w) < 0.5:
        return v_lo + w * d
    return v_hi - d * (torch.tensor(1.0, dtype=F32) - w)


def plane_thresholds(a, lam):
    """a [b, C, h, w] -> theta [b, C, 1, 1], the lam-quantile of each (image, channel) plane."""
    b, c = a.shape[:2]
    return quantile(a.reshape(b, c, -1), lam).reshape(b, c, 1, 1)


def _guided(unet_fn, x, t, c, uc, scale):
    """oracle.dpm_encoder._guided_eps with the same U-Net calls, also returning the uncond output when the call made one."""
    if uc is None or scale == 1.0:
        return unet_fn(x, t, c), None
    if scale == 0:
        e = unet_fn(x, t, uc)
        return e, e
    e_uc, e_c = unet_fn(torch.cat([x] * 2), torch.cat([t] * 2), torch.cat([uc, c])).chunk(2)
    return e_uc + scale * (e_c - e_uc), e_uc


def sega_cycle(unet_fn, x0, c_src, c_tgt, uc, c_edit, S, eta, skip_steps, src_scale, tgt_scale, scales, thresholds, cooldown, warmup,
               momentum_scale, beta, mask=None, prediction='eps', alphas_cumprod=None, stats=None):
    """One source chain (c_src at src_scale) driving one target chain (c_tgt at tgt_scale) with m concepts c_edit [B, m, L, D]:
    signed scales, thresholds and cooldowns (lists of m), one warmup, momentum scale and beta.  mask as in masked_cycle.  stats
    (optional dict): receives 'margin', the smallest |a - theta| / theta over every active plane and step, and 'planes'.
    -> (target latent [B,C,h,w], z_list as latent_encode returns it)."""
    assert eta > 0 and uc is not None
    tab = DDIMTables(S, eta, alphas_cumprod)
    b, m = x0.shape[0], c_edit.shape[1]
    sc = [torch.tensor(s, dtype=F32) for s in scales]
    mu, be = torch.tensor(momentum_scale, dtype=F32), torch.tensor(beta, dtype=F32)
    be1 = torch.tensor(float(np.float32(1.0 - float(beta))), dtype=F32)
    refine_steps = tab.timesteps.shape[0] - skip_steps
    at = tab.alphas[refine_steps - 1]
    xt = at.sqrt() * x0 + (1 - at).sqrt() * torch.randn(x0.shape)
    z_list, y = [xt], xt
    nu = torch.zeros_like(x0)
    margin, planes = float('inf'), 0
    for i, step in enumerate(np.flip(tab.timesteps)[-refine_steps:]):
        index = refine_steps - i - 1
        ts = torch.full((b,), int(step), dtype=torch.long)
        xt_next = latent_sample_xt_next(tab, x0, xt, index)
        e_src, _ = _guided(unet_fn, xt, ts, c_src, uc, src_scale)
        a_t, a_prev, sigma_t, _ = _coeffs(tab, index, b)
        e_t, pred_x0 = _eps_x0(e_src, xt, int(step), index, tab, b, prediction)
        dir_xt = (1. - a_prev - sigma_t ** 2).sqrt() * e_t
        eps = (xt_next - a_prev.sqrt() * pred_x0 - dir_xt) / sigma_t / 1.0
        z_list.append(eps)
        o_hat, o_uc = _guided(unet_fn, y, ts, c_tgt, uc, tgt_scale)
        # the concept rows (and the target's uncond row when its own call made none) in a call of their own
        extra = 1 if o_uc is None else 0
        cs = ([uc] if extra else []) + [c_edit[:, k] for k in range(m)]
        out = unet_fn(torch.cat([y] * (extra + m)), torch.cat([ts] * (extra + m)), torch.cat(cs)).chunk(extra + m)
        if extra:
            o_uc = out[0]
        S_ = None
        for k in range(m):
            psi = sc[k] * (out[extra + k] - o_uc)
            a = psi.abs()
            theta = plane_thresholds(a, thresholds[k])
            active = i < cooldown[k]
            if active:
                planes += theta.numel()
                rel = ((a - theta).abs() / theta).reshape(b, a.shape[1], -1).amin(dim=-1)
                margin = min(margin, float(rel.min()))
            g = torch.where((a >= theta) & active, psi, torch.zeros_like(psi))
            S_ = g if S_ is None else S_ + g
        G = S_ + mu * nu
        nu = be * nu + be1 * G
        if i >= warmup:
            o_hat = o_hat + G
        e_t, pred_x0 = _eps_x0(o_hat, y, int(step), index, tab, b, prediction)
        dir_xt = (1. - a_prev - sigma_t ** 2).sqrt() * e_t
        y_new = a_prev.sqrt() * pred_x0 + dir_xt + sigma_t * eps * 1.
        y = y_new if mask is None else blend(y_new, xt_next, mask)
        xt = xt_next
    if stats is not None:
        stats.update(margin=margin, planes=planes)
    return y, z_list
