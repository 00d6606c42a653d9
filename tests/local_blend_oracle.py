"""CPU restatement of Prompt-to-Prompt's LocalBlend on the lock-step cycle (test infrastructure only).

The reference has no LocalBlend, so this loop is pinned by P2P's own definition (LocalBlend, AttentionStore and get_mask in
prompt-to-prompt's released code) and by include/cdx.h, cdx_cycle_lockstep_blend.  It is tests/p2p_oracle.py's loop (one U-Net call
per step on [source (uncond, cond) | target (uncond, cond)], random draws in latent_encode's order) with three additions:

- During the call oracle.unet_openai's ``_attention`` is substituted.  Every controlled row's probabilities are replaced as
  p2p_refine_oracle states them (replace: attn_src . A_b; refine: plus attn_own * w_b), and then, as P2P's store holds the edited
  maps, every cross-attention of the input and output blocks over (h/4)(w/4) queries adds, in float64, the source and target cond
  rows' maps of that call contracted with the word weights: W_v(p) = sum_h sum_j attn[row, h, p, j] v_j.  The edited map is formed
  explicitly; the engine instead probes the source row with A_b v (the weight identity, test_local_blend_cpu.py).
- R_v += W_v at every step from the loop's first, in float64.
- At steps i >= start_step the target's x_{t-1} is blended with the source's under get_mask's mask (blend_mask), times the user mask
  when given.
"""
import contextlib

import numpy as np
import torch
import torch.nn.functional as F

from oracle import unet_openai
from oracle.dpm_encoder import _coeffs, latent_sample_xt_next
from oracle.schedules import DDIMTables
from tests.masked_oracle import blend
from tests.p2p_oracle import _rows
from tests.sd2_oracle import _eps_x0

F32 = torch.float32


def normalised(R, pool):
    """R [b, gh, gw] -> maxpool3x3(R) / max (pool) or R / max, per image; 0 / 0 stays NaN, as in get_mask."""
    M = F.max_pool2d(R.unsqueeze(1), 3, 1, 1).squeeze(1) if pool else R
    return M / R.flatten(1).amax(dim=1).view(-1, 1, 1)


def grid_mask(R_src, R_tgt, th_blend, S_src=None, S_tgt=None, th_sub=0.3):
    """get_mask on the grid: (blend words, pooled, source OR target) AND NOT (subtract words, unpooled, source OR target) -> bool
    [b, gh, gw].  The thresholds are compared in the maps' dtype (fp32 for the kernel's restatement)."""
    t = lambda th: torch.tensor(th, dtype=R_src.dtype)
    m = (normalised(R_src, True) > t(th_blend)) | (normalised(R_tgt, True) > t(th_blend))
    if S_src is not None:
        m = m & ~((normalised(S_src, False) > t(th_sub)) | (normalised(S_tgt, False) > t(th_sub)))
    return m


def upsample4(m):
    """[b, gh, gw] -> [b, 1, 4 gh, 4 gw], nearest."""
    return m.repeat_interleave(4, dim=-2).repeat_interleave(4, dim=-1).unsqueeze(1)


def mask_stage_fp32(maps, n_terms, n_vec, run, th_blend, th_sub, gh, gw, umask=None):
    """cdx_local_blend_mask in the kernel's order, fp32: run [B*n_vec, G] += (term 0 + term 1 + ...) in place -> mask [B,1,h,w]."""
    B = run.shape[0] // n_vec
    m = maps.view(B, n_vec, n_terms, gh * gw)
    w = m[:, :, 0]
    for t in range(1, n_terms):
        w = w + m[:, :, t]
    run.view(B, n_vec, -1).add_(w)
    R = run.view(B, n_vec, gh, gw)
    keep = grid_mask(R[:, 0], R[:, 1], th_blend, *((R[:, 2], R[:, 3], th_sub) if n_vec == 4 else ()))
    out = upsample4(keep).to(F32)
    return out if umask is None else torch.where(out == 1, umask, torch.zeros_like(umask))


@contextlib.contextmanager
def blend_attention(pairs, cross, self_, self_max_tokens, A, W, tokens, probes, store):
    """Within the block: the controlled rows' probabilities replaced as p2p_refine_oracle.refined_attention does (W None: replace),
    and for every (key, row, vec) in probes, store[key] += sum over heads and keys of the row's (edited) probabilities times vec,
    over the probed layers (float64)."""
    plain = unet_openai._attention

    def attention(sd, p, x, context, heads):
        probed = context is not None and x.shape[1] == tokens and (p.startswith('input_blocks.') or p.startswith('output_blocks.'))
        controlled = cross if context is not None else (self_ and x.shape[1] <= self_max_tokens)
        if not (controlled or probed):
            return plain(sd, p, x, context, heads)
        q = unet_openai._lin(sd, p + '.to_q', x)
        ctx = x if context is None else context
        k = unet_openai._lin(sd, p + '.to_k', ctx)
        v = unet_openai._lin(sd, p + '.to_v', ctx)
        b, n, inner = q.shape
        d = inner // heads

        def split(t):
            return t.reshape(b, t.shape[1], heads, d).permute(0, 2, 1, 3)

        qh, kh, vh = split(q), split(k), split(v)
        attn = (torch.einsum('bhid,bhjd->bhij', qh, kh) * d ** -0.5).softmax(dim=-1)
        ctl = attn.clone()
        if controlled:
            for r, s, j in pairs:
                if context is None:
                    ctl[r] = attn[s]
                else:
                    ctl[r] = torch.einsum('hpw,wn->hpn', attn[s], A[j])
                    if W is not None:
                        ctl[r] = ctl[r] + attn[r] * W[j]
        if probed:
            for key, r, vec in probes:
                m = torch.einsum('hpn,n->p', ctl[r].double(), vec.double())
                store[key] = store[key] + m if key in store else m
        if not controlled:
            return plain(sd, p, x, context, heads)
        out = torch.einsum('bhij,bhjd->bhid', ctl, vh).permute(0, 2, 1, 3).reshape(b, n, inner)
        return unet_openai._lin(sd, p + '.to_out.0', out)

    unet_openai._attention = attention
    try:
        yield
    finally:
        unet_openai._attention = plain


def blend_cycle(sd, cfg, x0, c_src, c_tgt, uc, S, eta, skip_steps, src_scale, tgt_scale, alpha_src, alpha_tgt, start_step, th_blend,
                th_sub=0.3, sub_src=None, sub_tgt=None, cross_steps=0, self_steps=0, self_max_tokens=256, token_map=None, own_weight=None,
                prediction='eps', mask=None, record=None):
    """p2p_cycle's loop (cross_steps / self_steps step counts; token_map [B, L, L] or None; own_weight [B, L] or None: replace)
    under LocalBlend: word vectors [B, L], start_step the first blended step, mask [B,1,h,w] the user mask or None.  record
    (optional list): per step, dict(R=[b, n_vec, gh, gw] float64 running sums, mask=[b,1,h,w] the step's blend mask (None before
    start_step)).  -> (target latent [B,C,h,w], z_list as latent_encode returns it)."""
    assert eta > 0 and src_scale != 0 and tgt_scale != 0
    tab = DDIMTables(S, eta)
    b, L = x0.shape[0], c_src.shape[1]
    h, w = x0.shape[2:]
    gh, gw = h // 4, w // 4
    A = token_map if token_map is not None else torch.eye(L).expand(b, L, L)
    ns, nt = _rows(uc, src_scale), _rows(uc, tgt_scale)
    src_cond, tgt_cond = (ns - 1) * b, (ns + nt - 1) * b
    pairs = [(tgt_cond + j, src_cond + j, j) for j in range(b)]
    vecs = [alpha_src, alpha_tgt] + ([sub_src, sub_tgt] if sub_src is not None else [])
    probes = [((j, v), (src_cond if v % 2 == 0 else tgt_cond) + j, vecs[v][j]) for j in range(b) for v in range(len(vecs))]
    R = torch.zeros(b, len(vecs), gh * gw, dtype=torch.float64)
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
        store = {}
        with blend_attention(pairs, i < cross_steps, i < self_steps, self_max_tokens, A, own_weight, gh * gw, probes, store):
            out = unet_openai.unet_forward(sd, cfg, x_in, t_in, c_in).chunk(ns + nt)
        for (j, v), m in store.items():
            R[j, v] += m
        Rg = R.view(b, len(vecs), gh, gw)
        m_i = None
        if i >= start_step:
            keep = grid_mask(Rg[:, 0], Rg[:, 1], th_blend, *((Rg[:, 2], Rg[:, 3], th_sub) if len(vecs) == 4 else ()))
            m_i = upsample4(keep).to(F32)
            if mask is not None:
                m_i = m_i * mask
        if record is not None:
            record.append(dict(R=Rg.clone(), mask=m_i))
        e_src = out[0] + src_scale * (out[1] - out[0]) if ns == 2 else out[0]
        e_tgt = out[ns] + tgt_scale * (out[ns + 1] - out[ns]) if nt == 2 else out[ns]
        a_t, a_prev, sigma_t, _ = _coeffs(tab, index, b)
        e_t, pred_x0 = _eps_x0(e_src, xt, int(step), index, tab, b, prediction)
        dir_xt = (1. - a_prev - sigma_t ** 2).sqrt() * e_t
        eps = (xt_next - a_prev.sqrt() * pred_x0 - dir_xt) / sigma_t / 1.0
        z_list.append(eps)
        e_t, pred_x0 = _eps_x0(e_tgt, y, int(step), index, tab, b, prediction)
        dir_xt = (1. - a_prev - sigma_t ** 2).sqrt() * e_t
        y_new = a_prev.sqrt() * pred_x0 + dir_xt + sigma_t * eps * 1.
        m_step = m_i if m_i is not None else mask
        y = y_new if m_step is None else blend(y_new, xt_next, m_step)
        xt = xt_next
    return y, z_list
