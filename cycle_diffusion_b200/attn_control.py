"""Prompt-to-Prompt attention control (Hertz et al., 2022; "Cross Attention Control") for the lock-step cycle.

The "replace" edit: in the first steps of the loop the target chain's conditional row attends with the source row's attention
probabilities (cross-attention remapped through a token map, self-attention copied), so the edit keeps the source image's layout.
The "refine" edit aligns the two prompts instead: a target token matched to a source token takes that token's cross-attention map,
a target token with no match keeps the row's own map (``own_weight``).  The engine does both inside the fused attention kernel
(include/cdx.h, cdx_cycle_lockstep_ctl and cdx_cycle_lockstep_refine); this module holds the value the Python surfaces take and
the host helpers that build token maps from two prompts' token ids.

MasaCtrl's mutual self-attention (Cao et al., 2023; ``MutualSelfControl``) is the complementary control for non-rigid edits: in
the decoder's self-attention layers the target rows keep their own queries and attend over the source row's keys and values
(cdx_cycle_lockstep_mutual), so the layout follows the target prompt and the content comes from the real image.

Plug-and-Play diffusion features (Tumanyan et al., 2023; ``PnPControl``) keep the real image's spatial layout for text-guided
translation: the target rows take the source row's decoder ResBlock features and its self-attention queries and keys
(cdx_cycle_lockstep_pnp), and the target prompt sets the appearance.
"""
from dataclasses import dataclass

import torch

from . import _cabi


def _fraction(name, f):
    if isinstance(f, bool) or not isinstance(f, (int, float)) or not 0.0 <= float(f) <= 1.0:
        raise ValueError(f'{name} must be a fraction in [0, 1], got {f!r}')
    return float(f)


@dataclass(frozen=True)
class AttentionControl:
    """cross_steps / self_steps: fractions of the loop's n steps; steps i < int(f * n) are controlled.  self_max_tokens: the
    self-attention layers of at most this many tokens are controlled (256: the 16x16 and 8x8 levels at 512^2).  token_map:
    optional float tensor [L, L] or [B, L, L], source token -> target token (P2P's mapper times its equalizer); None is the
    identity.  own_weight: optional float tensor [L] or [B, L], finite and >= 0 (P2P's refine): at a controlled cross-attention
    step target token j's probabilities become P_src . token_map[:, j] + own_weight[j] . P_own[j], P_own being the row's own; None
    is the replace edit.  The pipeline's refine passes token_map = A . diag(eq) and own_weight = (1 - colsum(A)) . eq."""
    cross_steps: float
    self_steps: float
    self_max_tokens: int = 256
    token_map: object = None
    own_weight: object = None

    def __post_init__(self):
        _fraction('cross_steps', self.cross_steps)
        _fraction('self_steps', self.self_steps)
        if isinstance(self.self_max_tokens, bool) or not isinstance(self.self_max_tokens, int) or self.self_max_tokens < 0:
            raise ValueError(f'self_max_tokens must be an integer >= 0, got {self.self_max_tokens!r}')
        if self.token_map is not None and not torch.is_tensor(self.token_map):
            raise ValueError(f'token_map must be a tensor [L, L] or [B, L, L], got {type(self.token_map)}')
        if self.own_weight is not None:
            if not torch.is_tensor(self.own_weight):
                raise ValueError(f'own_weight must be a tensor [L] or [B, L], got {type(self.own_weight)}')
            if not bool(torch.isfinite(self.own_weight).all()) or bool((self.own_weight < 0).any()):
                raise ValueError('own_weight must be finite and >= 0')

    def steps(self, n):
        """(cross_steps, self_steps) as step counts of an n-step loop."""
        return int(self.cross_steps * n), int(self.self_steps * n)

    def device_map(self, B, L, device):
        """The token map as a contiguous float32 [B, L, L] tensor on `device`, or None."""
        A = self.token_map
        if A is None:
            return None
        if A.dim() == 2:
            A = A.unsqueeze(0).expand(B, -1, -1)
        if A.dim() != 3 or tuple(A.shape) != (B, L, L):
            raise ValueError(f'token_map: expected [{L}, {L}] or [{B}, {L}, {L}], got {tuple(self.token_map.shape)}')
        A = A.to(device=device, dtype=torch.float32).contiguous()
        if not bool(torch.isfinite(A).all()):
            raise ValueError('token_map must be finite')
        return A

    def device_weight(self, B, L, device):
        """own_weight as a contiguous float32 [B, L] tensor on `device`, or None."""
        w = self.own_weight
        if w is None:
            return None
        if w.dim() == 1:
            w = w.unsqueeze(0).expand(B, -1)
        if w.dim() != 2 or tuple(w.shape) != (B, L):
            raise ValueError(f'own_weight: expected [{L}] or [{B}, {L}], got {tuple(self.own_weight.shape)}')
        return w.to(device=device, dtype=torch.float32).contiguous()

    def c_struct(self, n, B, L, device):
        """-> (cdx_attn_control for an n-step loop, the device token map it points to, the device own weight or None; keep both
        alive over the call)."""
        A = self.device_map(B, L, device)
        w = self.device_weight(B, L, device)
        cross, self_ = self.steps(n)
        return _cabi.AttnControl(cross, self_, self.self_max_tokens, A.data_ptr() if A is not None else None), A, w


@dataclass(frozen=True)
class MutualSelfControl:
    """MasaCtrl's mutual self-attention control: at loop steps i >= start_step (0-based, of the steps that run after strength's
    skip), in every SpatialTransformer whose index in forward order (input blocks, middle block, output blocks; 16 in SD v1 / 2.x)
    is >= start_layer, the target chain's rows attend with their own queries over the source chain's keys and values -- the cond
    row over the source's cond row, the uncond row over the source's uncond row (its cond row when the source has none).  The
    defaults are MasaCtrl's: the last six layers (the decoder's two finest levels) from step 4 on."""
    start_step: int = 4
    start_layer: int = 10

    def __post_init__(self):
        for name in ('start_step', 'start_layer'):
            v = getattr(self, name)
            if isinstance(v, bool) or not isinstance(v, int) or v < 0:
                raise ValueError(f'{name} must be an integer >= 0, got {v!r}')


@dataclass(frozen=True)
class PnPControl:
    """Plug-and-Play's feature and attention injection: at loop steps i < int(feature_steps * n) (0-based, of the n steps that run
    after strength's skip), the ResBlock output_blocks.k.0 of every k in feature_blocks gives each target row its own skip plus
    out_layers of the source row's in_layers output; at steps i < int(attention_steps * n), in every SpatialTransformer whose index
    in forward order (input blocks, middle block, output blocks; 16 in SD v1 / 2.x) is >= attention_start_layer, the target rows
    attend with the source row's queries and keys over their own values.  The target's cond row reads the source's cond row, its
    uncond row the source's uncond row (the source's only row when it has none).  The defaults are PnP's: pnp_f_t = 0.8 and
    pnp_attn_t = 0.5, block 4 (up_blocks[1].resnets[1]), layers from 8 (up_blocks[1].attentions[1]) on."""
    feature_steps: float = 0.8
    attention_steps: float = 0.5
    feature_blocks: tuple = (4,)
    attention_start_layer: int = 8

    def __post_init__(self):
        _fraction('feature_steps', self.feature_steps)
        _fraction('attention_steps', self.attention_steps)
        blocks = self.feature_blocks
        if not isinstance(blocks, (tuple, list)):
            raise ValueError(f'feature_blocks must be a tuple of output-block indices, got {blocks!r}')
        for k in blocks:
            if isinstance(k, bool) or not isinstance(k, int) or k < 0:
                raise ValueError(f'feature_blocks: indices must be integers >= 0, got {k!r}')
        if len(set(blocks)) != len(blocks):
            raise ValueError(f'feature_blocks: duplicate index in {tuple(blocks)}')
        object.__setattr__(self, 'feature_blocks', tuple(blocks))
        v = self.attention_start_layer
        if isinstance(v, bool) or not isinstance(v, int) or v < 0:
            raise ValueError(f'attention_start_layer must be an integer >= 0, got {v!r}')

    def steps(self, n):
        """(feature_steps, attention_steps) as step counts of an n-step loop."""
        return int(self.feature_steps * n), int(self.attention_steps * n)


def replace_token_map(src_ids, tgt_ids, L):
    """P2P's "replace" mapper for two prompts' token ids (BOS and EOS included, before padding) that differ in one contiguous
    run: -> float32 [L, L], source position -> target position.  Identity on the common prefix; the differing run one-to-one when both runs have the same length, else every
    source token of the run to every target token of it with weight 1 / len(target run); the rest shifted by the length
    difference, positions pushed past L dropped.  Identical sequences give the identity."""
    src, tgt = [int(t) for t in src_ids], [int(t) for t in tgt_ids]
    A = torch.zeros(L, L, dtype=torch.float32)
    p = 0
    while p < min(len(src), len(tgt)) and src[p] == tgt[p]:
        p += 1
    s = 0                                              # common suffix, not reaching into the prefix
    while s < min(len(src), len(tgt)) - p and src[len(src) - 1 - s] == tgt[len(tgt) - 1 - s]:
        s += 1
    ns, nt = len(src) - p - s, len(tgt) - p - s       # the differing runs [p, p + ns) and [p, p + nt)
    for i in range(min(p, L)):
        A[i, i] = 1.0
    if ns == nt:
        for k in range(ns):
            if p + k < L:
                A[p + k, p + k] = 1.0
    elif nt > 0:
        for i in range(p, min(p + ns, L)):
            for j in range(p, min(p + nt, L)):
                A[i, j] = 1.0 / nt
    shift = nt - ns
    for i in range(p + ns, L):                          # the suffix, and the padding past the prompts, shifted
        if i + shift < L:
            A[i, i + shift] = 1.0
    return A


def refine_token_map(src_ids, tgt_ids, L):
    """P2P's "refine" mapper for two prompts' token ids (BOS and EOS included, before padding): -> float32 [L, L], A[m(j), j] = 1
    for every target position j aligned to source position m(j), a zero column for a target token with no source.

    The alignment is global (Needleman-Wunsch): match +1, mismatch -1, gap 0, boundary row and column 0.  The traceback prefers, on
    ties, a target token with no source, then a dropped source token, then the diagonal; a mismatch is never taken, so a
    substituted word is a drop plus an insertion and attends on its own.  Target positions j >= len(tgt_ids) (padding) map to
    source position j; anything past L is dropped.  Identical sequences give the identity."""
    src, tgt = [int(t) for t in src_ids], [int(t) for t in tgt_ids]
    n, m = len(src), len(tgt)
    score = [[0] * (m + 1) for _ in range(n + 1)]
    for i in range(1, n + 1):
        for j in range(1, m + 1):
            score[i][j] = max(score[i - 1][j - 1] + (1 if src[i - 1] == tgt[j - 1] else -1), score[i][j - 1], score[i - 1][j])
    src_of = [-1] * m                                   # m(j) per target position of the prompt
    i, j = n, m
    while i > 0 or j > 0:
        if j > 0 and score[i][j] == score[i][j - 1]:
            j -= 1                                       # left: target token j - 1 has no source
        elif i > 0 and score[i][j] == score[i - 1][j]:
            i -= 1                                       # up: source token i - 1 is dropped
        else:
            src_of[j - 1] = i - 1                        # diagonal: a match (a mismatch never ties the better gap)
            i, j = i - 1, j - 1
    A = torch.zeros(L, L, dtype=torch.float32)
    for j in range(L):
        s_ = src_of[j] if j < m else j
        if 0 <= s_ < L:
            A[s_, j] = 1.0
    return A
