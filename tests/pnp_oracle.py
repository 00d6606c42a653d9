"""CPU fp32 restatement of Plug-and-Play feature and attention injection on the lock-step cycle (test infrastructure only).

The reference has no PnP, so this loop is pinned only by its definition, as mutual_oracle.py is.  It states PnP (Tumanyan et al.,
2023) on the network's own tensors: for the duration of a U-Net call oracle.unet_openai's ``_resblock`` and ``_attention`` are
substituted, the call's steps and self-attention layers are counted in forward order, and for each (target row r, source row s):

    ResBlock output_blocks.k.0, k in feature_blocks, step i < feature_steps:
        h = out_layers(in_layers(x) + emb) for all rows, then h[r] = h[s], then x_skip + h
    self-attention of layer index >= attention_start_layer, step i < attention_steps:
        out_r = softmax(Q_s K_s^T * d^-1/2) . V_r        (per head)

Cross-attention and the source rows run unchanged.  The engine instead writes row r of the out_layers GroupNorm from row s and
redirects the fused attention kernel's Q and K tiles, so the two routes share nothing but the definition.

The loop is p2p_oracle.p2p_cycle's with no Prompt-to-Prompt step.  p2p_cycle has no source scale 0, where the engine runs the
source chain as one row under uc; pnp_cycle runs that chain as its equal, a one-row chain under the context uc (scale 1), and maps
both target rows to it -- the source row that drives the chain.
"""
import contextlib

import torch

from oracle import unet_openai
from tests.mutual_oracle import mutual_pairs
from tests.p2p_oracle import p2p_cycle


@contextlib.contextmanager
def pnp_injection(pairs, feature_steps, feature_blocks, attention_steps, attention_start_layer):
    """Within the block, U-Net call i (counted from 0) is loop step i; row r takes row s's features and self-attention Q / K for
    each (r, s) in pairs, as the module docstring states."""
    plain_res, plain_attention, plain_forward = unet_openai._resblock, unet_openai._attention, unet_openai.unet_forward
    state = {'step': -1, 'layer': 0}
    controlled = {f'output_blocks.{k}.0' for k in feature_blocks}

    def source_of(b):
        src = torch.arange(b)
        for r, s in pairs:
            src[r] = s
        return src

    def forward(*args, **kw):
        state['step'] += 1
        state['layer'] = 0
        return plain_forward(*args, **kw)

    def resblock(sd, p, x, emb):
        if state['step'] >= feature_steps or p not in controlled:
            return plain_res(sd, p, x, emb)
        F = torch.nn.functional
        h = unet_openai._conv(sd, p + '.in_layers.2', F.silu(unet_openai._gn(sd, p + '.in_layers.0', x, 1e-5)))
        h = h + unet_openai._lin(sd, p + '.emb_layers.1', F.silu(emb))[..., None, None]
        h = unet_openai._conv(sd, p + '.out_layers.3', F.silu(unet_openai._gn(sd, p + '.out_layers.0', h, 1e-5)))
        h = h[source_of(h.shape[0])]
        if (p + '.skip_connection.weight') in sd:
            x = unet_openai._conv(sd, p + '.skip_connection', x, padding=0)
        return x + h

    def attention(sd, p, x, context, heads):
        if context is not None:
            return plain_attention(sd, p, x, context, heads)
        layer = state['layer']
        state['layer'] += 1
        if state['step'] >= attention_steps or layer < attention_start_layer:
            return plain_attention(sd, p, x, context, heads)
        q = unet_openai._lin(sd, p + '.to_q', x)
        k = unet_openai._lin(sd, p + '.to_k', x)
        v = unet_openai._lin(sd, p + '.to_v', x)
        b, n, inner = q.shape
        d = inner // heads
        src = source_of(b)
        q, k = q[src], k[src]

        def split(t):
            return t.reshape(b, n, heads, d).permute(0, 2, 1, 3)

        q, k, v = split(q), split(k), split(v)
        attn = (torch.einsum('bhid,bhjd->bhij', q, k) * d ** -0.5).softmax(dim=-1)
        out = torch.einsum('bhij,bhjd->bhid', attn, v).permute(0, 2, 1, 3).reshape(b, n, inner)
        return unet_openai._lin(sd, p + '.to_out.0', out)

    unet_openai._resblock, unet_openai._attention, unet_openai.unet_forward = resblock, attention, forward
    try:
        yield
    finally:
        unet_openai._resblock, unet_openai._attention, unet_openai.unet_forward = plain_res, plain_attention, plain_forward


def pnp_pairs(b, uc, src_scale, tgt_scale):
    """(target row, source row) of the oracle's lock-step call, b samples per block.  At source scale 0 the oracle runs the source
    chain as one row (pnp_cycle), so the pairs are those of a one-row source chain."""
    return mutual_pairs(b, uc, 1.0 if src_scale == 0 else src_scale, tgt_scale)


def pnp_cycle(sd, cfg, x0, c_src, c_tgt, uc, S, eta, skip_steps, src_scale, tgt_scale, feature_steps, attention_steps,
              feature_blocks=(4,), attention_start_layer=8, prediction='eps', mask=None):
    """One source chain (c_src at src_scale) driving one target chain (c_tgt at tgt_scale) under PnP injection; feature_steps /
    attention_steps are step counts of the refine_steps-step loop.  mask as in masked_cycle.  -> (target latent [B,C,h,w], z_list)."""
    pairs = pnp_pairs(x0.shape[0], uc, src_scale, tgt_scale)
    if src_scale == 0:                      # the source chain's only row: its uncond row, run as a one-row chain under uc
        c_src, src_scale = uc, 1.0
    with pnp_injection(pairs, feature_steps, feature_blocks, attention_steps, attention_start_layer):
        return p2p_cycle(sd, cfg, x0, c_src, c_tgt, uc, S, eta, skip_steps, src_scale, tgt_scale, 0, 0, prediction=prediction, mask=mask)
