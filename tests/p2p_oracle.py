"""CPU fp32 restatement of Prompt-to-Prompt's "replace" attention control on the lock-step cycle (test infrastructure only).

The reference has no attention control, so this loop is pinned only by its definition, as masked_oracle.py is.  It states P2P in the
probability domain (Hertz et al., 2022): oracle.unet_openai's ``_attention`` is substituted for the duration of a U-Net call, and
on a controlled row (the target chain's cond row of sample b) the softmax probabilities are replaced before they meet V:

    cross-attention, step i < cross_steps:                   attn = einsum('hpw,wn->hpn', attn_src, A_b)
    self-attention, step i < self_steps, tokens <= max:      attn = attn_src

attn_src being the probabilities of the source chain's cond row of the same sample (same layer, all heads), and V the controlled row's
own.  The engine instead remaps the Q / K tiles and projects A . c_tgt, so the two routes share nothing but the definition.

The loop runs every chain's rows in one U-Net call per step, [source (uncond, cond) | target (uncond, cond)], a chain contributing
an uncond row only when its scale is neither 0 nor 1 (ddim.py:550-559), and makes its random draws in latent_encode's order, so
``torch.manual_seed(s)`` before a call matches the engine fed with wrappers.encode_noise under the same seed.
"""
import contextlib

import numpy as np
import torch

from oracle import unet_openai
from oracle.dpm_encoder import _coeffs, latent_sample_xt_next
from oracle.schedules import DDIMTables
from tests.masked_oracle import blend
from tests.sd2_oracle import _eps_x0


@contextlib.contextmanager
def controlled_attention(pairs, cross, self_, self_max_tokens, A):
    """Within the block, unet_openai's attention replaces the probabilities of row r by those of row s for each (r, s, b) in pairs:
    cross-attention (when `cross`) through A[b] [L, L], self-attention (when `self_` and at most self_max_tokens tokens) as they are."""
    plain = unet_openai._attention

    def attention(sd, p, x, context, heads):
        if not (cross if context is not None else (self_ and x.shape[1] <= self_max_tokens)):
            return plain(sd, p, x, context, heads)
        q = unet_openai._lin(sd, p + '.to_q', x)
        ctx = x if context is None else context
        k = unet_openai._lin(sd, p + '.to_k', ctx)
        v = unet_openai._lin(sd, p + '.to_v', ctx)
        b, n, inner = q.shape
        d = inner // heads

        def split(t):
            return t.reshape(b, t.shape[1], heads, d).permute(0, 2, 1, 3)

        q, k, v = split(q), split(k), split(v)
        attn = (torch.einsum('bhid,bhjd->bhij', q, k) * d ** -0.5).softmax(dim=-1).clone()
        for r, s, j in pairs:
            attn[r] = torch.einsum('hpw,wn->hpn', attn[s], A[j]) if context is not None else attn[s]
        out = torch.einsum('bhij,bhjd->bhid', attn, v).permute(0, 2, 1, 3).reshape(b, n, inner)
        return unet_openai._lin(sd, p + '.to_out.0', out)

    unet_openai._attention = attention
    try:
        yield
    finally:
        unet_openai._attention = plain


def _rows(uc, scale):
    return 1 if uc is None or scale == 1.0 else 2


def p2p_cycle(sd, cfg, x0, c_src, c_tgt, uc, S, eta, skip_steps, src_scale, tgt_scale, cross_steps, self_steps, self_max_tokens=256,
              token_map=None, prediction='eps', mask=None):
    """One source chain (c_src at src_scale) driving one target chain (c_tgt at tgt_scale) under attention control; cross_steps /
    self_steps are step counts of the refine_steps-step loop; token_map [B, L, L] or None (identity).  mask as in masked_cycle.
    -> (target latent [B,C,h,w], z_list as latent_encode returns it)."""
    assert eta > 0 and src_scale != 0 and tgt_scale != 0
    tab = DDIMTables(S, eta)
    b, L = x0.shape[0], c_src.shape[1]
    A = token_map if token_map is not None else torch.eye(L).expand(b, L, L)
    ns, nt = _rows(uc, src_scale), _rows(uc, tgt_scale)
    src_cond, tgt_cond = (ns - 1) * b, (ns + nt - 1) * b           # first cond row of each block
    pairs = [(tgt_cond + j, src_cond + j, j) for j in range(b)]
    refine_steps = tab.timesteps.shape[0] - skip_steps
    at = tab.alphas[refine_steps - 1]
    xt = at.sqrt() * x0 + (1 - at).sqrt() * torch.randn(x0.shape)
    z_list, y = [xt], xt
    for i, step in enumerate(np.flip(tab.timesteps)[-refine_steps:]):
        index = refine_steps - i - 1
        xt_next = latent_sample_xt_next(tab, x0, xt, index)
        xs = [xt] * ns + [y] * nt
        cs = ([uc] if ns == 2 else []) + [c_src] + ([uc] if nt == 2 else []) + [c_tgt]
        x_in, c_in = torch.cat(xs), torch.cat(cs)
        t_in = torch.full((x_in.shape[0],), int(step), dtype=torch.long)
        with controlled_attention(pairs, i < cross_steps, i < self_steps, self_max_tokens, A):
            out = unet_openai.unet_forward(sd, cfg, x_in, t_in, c_in).chunk(ns + nt)
        e_src = out[0] + src_scale * (out[1] - out[0]) if ns == 2 else out[0]          # _guided_eps
        e_tgt = out[ns] + tgt_scale * (out[ns + 1] - out[ns]) if nt == 2 else out[ns]
        a_t, a_prev, sigma_t, _ = _coeffs(tab, index, b)
        e_t, pred_x0 = _eps_x0(e_src, xt, int(step), index, tab, b, prediction)
        dir_xt = (1. - a_prev - sigma_t ** 2).sqrt() * e_t
        eps = (xt_next - a_prev.sqrt() * pred_x0 - dir_xt) / sigma_t / 1.0
        z_list.append(eps)
        e_t, pred_x0 = _eps_x0(e_tgt, y, int(step), index, tab, b, prediction)
        dir_xt = (1. - a_prev - sigma_t ** 2).sqrt() * e_t
        y_new = a_prev.sqrt() * pred_x0 + dir_xt + sigma_t * eps * 1.
        y = y_new if mask is None else blend(y_new, xt_next, mask)
        xt = xt_next
    return y, z_list
