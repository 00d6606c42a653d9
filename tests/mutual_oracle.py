"""CPU fp32 restatement of MasaCtrl's mutual self-attention control on the lock-step cycle (test infrastructure only).

The reference has no attention control, so this loop is pinned only by its definition, as p2p_oracle.py is.  It states
MutualSelfControl (Cao et al., 2023) on keys and values: for the duration of a U-Net call oracle.unet_openai's ``_attention`` is
substituted and counts the call's self-attention layers in forward order, and on a controlled (step, layer) -- step i >= start_step,
layer index >= start_layer -- each target row's K and V are replaced by its mapped source row's before the softmax:

    out_r = softmax(Q_r K_s^T * d^-1/2) . V_s        (r the target row, s its source row, per head)

The target's cond row maps to the source's cond row, its uncond row (when it has one) to the source's uncond row, or to the
source's cond row when the source runs without one.  Cross-attention and the source rows run unchanged.  The engine instead
redirects the fused kernel's K and V^T tiles, so the two routes share nothing but the definition.

The loop is p2p_oracle.p2p_cycle's with no Prompt-to-Prompt step (one U-Net call per step over [source | target] rows, random
draws in latent_encode's order, the mask blended as masked_oracle.blend does); unet_openai.unet_forward is wrapped to count its
steps.
"""
import contextlib

import torch

from oracle import unet_openai
from tests.p2p_oracle import _rows, p2p_cycle


@contextlib.contextmanager
def mutual_attention(pairs, start_step, start_layer):
    """Within the block, U-Net call i (counted from 0) is loop step i; in its self-attention layers >= start_layer, at steps
    >= start_step, row r takes its keys and values from row s for each (r, s) in pairs."""
    plain_attention, plain_forward = unet_openai._attention, unet_openai.unet_forward
    state = {'step': -1, 'layer': 0}

    def forward(*args, **kw):
        state['step'] += 1
        state['layer'] = 0
        return plain_forward(*args, **kw)

    def attention(sd, p, x, context, heads):
        if context is not None:
            return plain_attention(sd, p, x, context, heads)
        layer = state['layer']
        state['layer'] += 1
        if state['step'] < start_step or layer < start_layer:
            return plain_attention(sd, p, x, context, heads)
        q = unet_openai._lin(sd, p + '.to_q', x)
        k = unet_openai._lin(sd, p + '.to_k', x)
        v = unet_openai._lin(sd, p + '.to_v', x)
        b, n, inner = q.shape
        d = inner // heads
        src = torch.arange(b)
        for r, s in pairs:
            src[r] = s
        k, v = k[src], v[src]

        def split(t):
            return t.reshape(b, n, heads, d).permute(0, 2, 1, 3)

        q, k, v = split(q), split(k), split(v)
        attn = (torch.einsum('bhid,bhjd->bhij', q, k) * d ** -0.5).softmax(dim=-1)
        out = torch.einsum('bhij,bhjd->bhid', attn, v).permute(0, 2, 1, 3).reshape(b, n, inner)
        return unet_openai._lin(sd, p + '.to_out.0', out)

    unet_openai._attention, unet_openai.unet_forward = attention, forward
    try:
        yield
    finally:
        unet_openai._attention, unet_openai.unet_forward = plain_attention, plain_forward


def mutual_pairs(b, uc, src_scale, tgt_scale):
    """(target row, source row) of the lock-step call's rows [source (uncond, cond) | target (uncond, cond)], b samples per block."""
    ns, nt = _rows(uc, src_scale), _rows(uc, tgt_scale)
    src_cond, tgt_cond = (ns - 1) * b, (ns + nt - 1) * b
    pairs = [(tgt_cond + j, src_cond + j) for j in range(b)]
    if nt == 2:
        pairs += [(ns * b + j, j) for j in range(b)]             # uncond -> the source's first row: its uncond row, or its cond row
    return pairs


def mutual_cycle(sd, cfg, x0, c_src, c_tgt, uc, S, eta, skip_steps, src_scale, tgt_scale, start_step, start_layer, prediction='eps',
                 mask=None):
    """One source chain (c_src at src_scale) driving one target chain (c_tgt at tgt_scale) under mutual self-attention control from
    step start_step and self-attention layer start_layer on.  mask as in masked_cycle.  -> (target latent [B,C,h,w], z_list)."""
    pairs = mutual_pairs(x0.shape[0], uc, src_scale, tgt_scale)
    with mutual_attention(pairs, start_step, start_layer):
        return p2p_cycle(sd, cfg, x0, c_src, c_tgt, uc, S, eta, skip_steps, src_scale, tgt_scale, 0, 0, prediction=prediction, mask=mask)
