"""CPU fp32 restatement of Prompt-to-Prompt's "refine" attention control on the lock-step cycle (test infrastructure only).

Refine in the probability domain (Hertz et al., 2022): on a controlled row (the target chain's cond row of sample b), at a
controlled cross-attention step, the softmax probabilities become

    attn = einsum('hpw,wn->hpn', attn_src, A_b) + attn_own * w_b          (w_b [L] scales key n of the row's own map)

attn_src being the source chain's cond row's probabilities (same layer, all heads) and attn_own the row's own; self-attention is
controlled as for replace (attn = attn_src).  With w = None this is tests/p2p_oracle.py's replace edit, whose loop runs it (one
U-Net call per step on [source (uncond, cond) | target (uncond, cond)], random draws in latent_encode's order).  The engine instead
runs a second, accumulating attention launch over V'' = diag(w) . c_tgt projected, so the two routes share only the definition.
"""
import contextlib

import torch

from oracle import unet_openai
from tests import p2p_oracle


@contextlib.contextmanager
def refined_attention(pairs, cross, self_, self_max_tokens, A, W):
    """Within the block, unet_openai's attention replaces the probabilities of row r for each (r, s, b) in pairs: cross-attention
    (when `cross`) by attn[s] . A[b] + attn[r] * W[b] (W None: no own term), self-attention (when `self_` and at most
    self_max_tokens tokens) by attn[s]."""
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
        attn = (torch.einsum('bhid,bhjd->bhij', q, k) * d ** -0.5).softmax(dim=-1)
        ctl = attn.clone()
        for r, s, j in pairs:
            if context is None:
                ctl[r] = attn[s]
            else:
                ctl[r] = torch.einsum('hpw,wn->hpn', attn[s], A[j])
                if W is not None:
                    ctl[r] = ctl[r] + attn[r] * W[j]
        out = torch.einsum('bhij,bhjd->bhid', ctl, v).permute(0, 2, 1, 3).reshape(b, n, inner)
        return unet_openai._lin(sd, p + '.to_out.0', out)

    unet_openai._attention = attention
    try:
        yield
    finally:
        unet_openai._attention = plain


def p2p_refine_cycle(sd, cfg, x0, c_src, c_tgt, uc, S, eta, skip_steps, src_scale, tgt_scale, cross_steps, self_steps,
                     self_max_tokens=256, token_map=None, own_weight=None, prediction='eps', mask=None):
    """tests.p2p_oracle.p2p_cycle (same arguments, same loop and random draws) with refine's own term: own_weight [B, L], or None
    for the replace edit.  -> (target latent [B,C,h,w], z_list as latent_encode returns it)."""
    replace = p2p_oracle.controlled_attention
    p2p_oracle.controlled_attention = lambda pairs, cross, self_, tokens, A: refined_attention(pairs, cross, self_, tokens, A, own_weight)
    try:
        return p2p_oracle.p2p_cycle(sd, cfg, x0, c_src, c_tgt, uc, S, eta, skip_steps, src_scale, tgt_scale, cross_steps, self_steps,
                                    self_max_tokens, token_map, prediction, mask)
    finally:
        p2p_oracle.controlled_attention = replace
