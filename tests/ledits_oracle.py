"""CPU fp32 restatement of LEDITS++'s implicit masks on the semantic-guidance loop (test infrastructure only).

The reference has no semantic guidance, so this loop is pinned only by its definition (include/cdx.h,
cdx_cycle_lockstep_semantic_attn), as sega_oracle.py is.  It is sega_oracle.sega_cycle's loop (the same source, target and concept
U-Net calls) with SEGA's per-channel rule replaced by the masks.  During the concept call oracle.unet_openai's ``_attention`` is
substituted, as p2p_oracle.py and mutual_oracle.py substitute it, and records for every cross-attention of the input and output
blocks whose token count is (h/4)(w/4) the concept rows' probabilities softmax(q k^T d^-1/2) over all L keys, summed over heads and
over the concept's tokens 1..n_k, and over those layers.  Then, per concept k, every op a separate fp32 torch op in the kernel's order:

    As     = smooth(A)                                     (3x3, reflect padding 1, products row-major, added left to right)
    M1     = As(y/4, x/4) >= quantile(As over the grid, lambda_k)
    s      = |psi_k[0]| + |psi_k[1]| + ...                 (channels ascending)
    M      = M1 and s >= quantile(s over h*w, lambda_k)     with intersect, else M1
    g_k    = psi_k where (i < cooldown_k and M) else 0

The sum over concepts, the momentum and the warmup are sega_cycle's.
"""
import contextlib
import math

import numpy as np
import torch

from oracle import unet_openai
from oracle.dpm_encoder import _coeffs, latent_sample_xt_next
from oracle.schedules import DDIMTables
from tests.masked_oracle import blend
from tests.sd2_oracle import _eps_x0
from tests.sega_oracle import _guided, quantile

F32 = torch.float32


def smoothing_weights():
    """diffusers' GaussianSmoothing(kernel_size=3, sigma=0.5) as the engine states it: w_ab = fp32(g_a g_b / (sum g)^2), g = (e^-1, 1,
    e^-1) in double -> [3, 3] fp32."""
    g = [math.exp(-1.0), 1.0, math.exp(-1.0)]
    s = sum(g)
    return torch.tensor([[g[a] * g[b] / (s * s) for b in range(3)] for a in range(3)], dtype=torch.float64).to(F32)


def smooth(A):
    """A [..., gh, gw] fp32 -> the smoothed map, the kernel's order: the nine products row-major, each rounded, added left to right."""
    gh, gw = A.shape[-2:]
    ry = torch.tensor([1] + list(range(gh)) + [gh - 2])
    rx = torch.tensor([1] + list(range(gw)) + [gw - 2])
    P = A[..., ry, :][..., rx]
    W = smoothing_weights()
    s = None
    for a in range(3):
        for b in range(3):
            pr = W[a, b] * P[..., a: a + gh, b: b + gw]
            s = pr if s is None else s + pr
    return s


def channel_sum(psi):
    """|psi| summed over channels ascending, one rounded add each: [b, C, h, w] -> [b, h, w]."""
    s = psi[:, 0].abs()
    for c in range(1, psi.shape[1]):
        s = s + psi[:, c].abs()
    return s


def head_span_probs(q, k, heads, span):
    """q [b, N, C], k [b, L, C] -> [b, N]: sum over heads of the softmax probabilities of tokens 1..span[r] of row r (fp32 torch)."""
    b, n, inner = q.shape
    d = inner // heads
    qh = q.reshape(b, n, heads, d).permute(0, 2, 1, 3)
    kh = k.reshape(b, k.shape[1], heads, d).permute(0, 2, 1, 3)
    p = (torch.einsum('bhid,bhjd->bhij', qh, kh) * d ** -0.5).softmax(dim=-1)
    out = torch.zeros(b, n)
    for r in range(b):
        out[r] = p[r, :, :, 1: 1 + span[r]].sum(dim=-1).sum(dim=0)
    return out


@contextlib.contextmanager
def record_maps(tokens, span, maps):
    """Within the block, every cross-attention of the input and output blocks over `tokens` queries adds its rows' span sums into
    maps['A'] ([b, tokens]); maps['layers'] counts them."""
    plain = unet_openai._attention

    def attention(sd, p, x, context, heads):
        if context is not None and x.shape[1] == tokens and (p.startswith('input_blocks.') or p.startswith('output_blocks.')):
            q = unet_openai._lin(sd, p + '.to_q', x)
            k = unet_openai._lin(sd, p + '.to_k', context)
            a = head_span_probs(q, k, heads, span)
            maps['A'] = a if maps.get('A') is None else maps['A'] + a
            maps['layers'] = maps.get('layers', 0) + 1
        return plain(sd, p, x, context, heads)

    unet_openai._attention = attention
    try:
        yield
    finally:
        unet_openai._attention = plain


def rel_margin(v, theta):
    return float(((v - theta).abs() / theta).min()) if float(theta) > 0 else 0.0


def ledits_cycle(sd, cfg, x0, c_src, c_tgt, uc, c_edit, S, eta, skip_steps, src_scale, tgt_scale, scales, thresholds, cooldown, warmup,
                 momentum_scale, beta, n_tokens, intersect, mask=None, prediction='eps', alphas_cumprod=None, stats=None):
    """sega_cycle's arguments (the U-Net given as its state dict and config) plus n_tokens (list of m spans) and intersect.  stats
    (optional dict): 'margin1' / 'margin2', the smallest |v - theta| / theta of the attention and channel-sum thresholds over every
    active concept and step, and 'layers', the probed layers per call.  -> (target latent [B,C,h,w], z_list)."""
    assert eta > 0 and uc is not None
    unet_fn = lambda x, t, c: unet_openai.unet_forward(sd, cfg, x, t, c)
    tab = DDIMTables(S, eta, alphas_cumprod)
    b, m = x0.shape[0], c_edit.shape[1]
    h, w = x0.shape[2:]
    gh, gw = h // 4, w // 4
    sc = [torch.tensor(s, dtype=F32) for s in scales]
    mu, be = torch.tensor(momentum_scale, dtype=F32), torch.tensor(beta, dtype=F32)
    be1 = torch.tensor(float(np.float32(1.0 - float(beta))), dtype=F32)
    refine_steps = tab.timesteps.shape[0] - skip_steps
    at = tab.alphas[refine_steps - 1]
    xt = at.sqrt() * x0 + (1 - at).sqrt() * torch.randn(x0.shape)
    z_list, y = [xt], xt
    nu = torch.zeros_like(x0)
    m1 = m2 = float('inf')
    layers = None
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
        extra = 1 if o_uc is None else 0
        cs = ([uc] if extra else []) + [c_edit[:, k] for k in range(m)]
        span = [1] * (extra * b) + [n_tokens[k] for k in range(m) for _ in range(b)]
        maps = {}
        with record_maps(gh * gw, span, maps):
            out = unet_fn(torch.cat([y] * (extra + m)), torch.cat([ts] * (extra + m)), torch.cat(cs)).chunk(extra + m)
        layers = maps.get('layers', 0)
        A = maps['A'].reshape(extra + m, b, gh, gw)
        if extra:
            o_uc = out[0]
        S_ = None
        for k in range(m):
            psi = sc[k] * (out[extra + k] - o_uc)
            As = smooth(A[extra + k])
            th1 = quantile(As.reshape(b, -1), thresholds[k]).reshape(b, 1, 1)
            M = (As >= th1).repeat_interleave(4, dim=-2).repeat_interleave(4, dim=-1)
            active = i < cooldown[k]
            if active:
                m1 = min(m1, min(rel_margin(As[j], th1[j]) for j in range(b)))
            if intersect:
                s = channel_sum(psi)
                th2 = quantile(s.reshape(b, -1), thresholds[k]).reshape(b, 1, 1)
                M = M & (s >= th2)
                if active:
                    m2 = min(m2, min(rel_margin(s[j], th2[j]) for j in range(b)))
            keep = M.unsqueeze(1).expand_as(psi) & active
            g = torch.where(keep, psi, torch.zeros_like(psi))
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
        stats.update(margin1=m1, margin2=m2, layers=layers)
    return y, z_list
