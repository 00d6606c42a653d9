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

Prompt-to-Prompt's LocalBlend (``LocalBlend``) keeps a real-image edit local: at every step the target chain is blended with the
source chain outside the region the blend words' accumulated cross-attention points to (cdx_cycle_lockstep_blend).

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


def _weights(name, v):
    if not torch.is_tensor(v) or v.dim() not in (1, 2):
        raise ValueError(f'{name} must be a tensor [L] or [B, L], got {tuple(v.shape) if torch.is_tensor(v) else type(v)}')
    v = v.detach().to(torch.float64)
    if not bool(torch.isfinite(v).all()) or bool((v < 0).any()):
        raise ValueError(f'{name} must be finite and >= 0')
    if bool((v.reshape(-1, v.shape[-1]).sum(dim=-1) == 0).any()):
        raise ValueError(f'{name}: a weight vector is all zero (no blend word in the prompt)')


@dataclass(frozen=True)
class LocalBlend:
    """Prompt-to-Prompt's LocalBlend.  alpha_src / alpha_tgt: per-token weights [L] or [B, L] of the blend words in the source and
    the target prompt (P2P's alpha_layers; word_token_weights builds them), finite, >= 0 and not all zero.  sub_src / sub_tgt:
    optional, both or neither: the subtract words (P2P's substruct_words).  From loop step int(start_blend * n) on, the target
    chain keeps its own x_{t-1} only where maxpool3x3(R) / max(R) > threshold[0] for the source or the target blend map R (the
    words' cross-attention summed over the probed layers, heads and every step so far), and not where R_sub / max(R_sub) >
    threshold[1] for either subtract map; elsewhere it takes the source chain's.  threshold values in [0, 1)."""
    alpha_src: object
    alpha_tgt: object
    sub_src: object = None
    sub_tgt: object = None
    start_blend: float = 0.2
    threshold: tuple = (0.3, 0.3)

    def __post_init__(self):
        _weights('alpha_src', self.alpha_src)
        _weights('alpha_tgt', self.alpha_tgt)
        if (self.sub_src is None) != (self.sub_tgt is None):
            raise ValueError('sub_src and sub_tgt: give both or neither')
        if self.sub_src is not None:
            _weights('sub_src', self.sub_src)
            _weights('sub_tgt', self.sub_tgt)
        _fraction('start_blend', self.start_blend)
        th = self.threshold
        if not isinstance(th, (tuple, list)) or len(th) != 2 or any(isinstance(t, bool) or not isinstance(t, (int, float)) or
                                                                      not 0.0 <= float(t) < 1.0 for t in th):
            raise ValueError(f'threshold must be a pair (th_blend, th_sub) in [0, 1), got {th!r}')
        object.__setattr__(self, 'threshold', (float(th[0]), float(th[1])))

    def start_step(self, n):
        """The first blended step of an n-step loop."""
        return int(self.start_blend * n)

    def vectors(self, B, L, device):
        """(alpha_src, alpha_tgt, sub_src, sub_tgt) as contiguous float32 [B, L] tensors on `device` (the subtract pair None when
        not given)."""
        def one(name, v):
            if v is None:
                return None
            if v.dim() == 1:
                v = v.unsqueeze(0).expand(B, -1)
            if tuple(v.shape) != (B, L):
                raise ValueError(f'{name}: expected [{L}] or [{B}, {L}], got {tuple(v.shape)}')
            return v.to(device=device, dtype=torch.float32).contiguous()
        return tuple(one(k, getattr(self, k)) for k in ('alpha_src', 'alpha_tgt', 'sub_src', 'sub_tgt'))

    def c_struct(self, n, B, L, device):
        """-> (cdx_local_blend for an n-step loop, the device vectors it points to; keep them alive over the call)."""
        vs = self.vectors(B, L, device)
        ptr = lambda t: t.data_ptr() if t is not None else None
        return _cabi.LocalBlendC(*[ptr(t) for t in vs], self.start_step(n), self.threshold[0], self.threshold[1]), vs


def word_token_weights(prompt_ids, word_ids, L):
    """P2P's get_word_inds as weights: -> float32 [L] with 1 at every position of every occurrence of the run word_ids in
    prompt_ids (the prompt's tokens, start token included, so positions are context rows), 0 elsewhere; positions >= L are
    dropped.  ValueError when the run does not occur below L."""
    p, w = list(prompt_ids), list(word_ids)
    if not w:
        raise ValueError('word_token_weights: an empty word')
    out = torch.zeros(L, dtype=torch.float32)
    for i in range(len(p) - len(w) + 1):
        if p[i: i + len(w)] == w:
            out[i: min(i + len(w), L)] = 1.0
    if not bool(out.any()):
        raise ValueError(f'word_token_weights: the word {w} is not among the first {L} tokens of the prompt')
    return out


def words_weights(token_rows, word_rows, L):
    """[B, L] float32 from per-prompt token rows and per-prompt word lists (each word a token run): 1 at every occurrence of every
    word, as P2P sets alpha_layers."""
    rows = []
    for ids, words in zip(token_rows, word_rows):
        r = torch.zeros(L, dtype=torch.float32)
        for w in words:
            r = torch.maximum(r, word_token_weights(ids, w, L))
        rows.append(r)
    return torch.stack(rows)


def word_lists(texts, words):
    """words: a word (str), a tuple / list of words for every text, or a list with one such entry per text -> one tuple of words
    per text."""
    if isinstance(words, str):
        return [(words,)] * len(texts)
    words = list(words)
    if len(words) == len(texts) and all(not isinstance(w, str) for w in words):
        return [tuple(w) for w in words]
    if all(isinstance(w, str) for w in words):
        return [tuple(words)] * len(texts)
    raise ValueError(f'words: a word, a tuple of words, or one tuple per text ({len(texts)}), got {words!r}')


BLEND_KEYS = {'words', 'subtract_words', 'start_blend', 'threshold'}


def resolve_local_blend(spec, cond_stage, sources, targets):
    """A LocalBlend as it is, or {'words': (source_words, target_words), ['subtract_words': (source_words, target_words)],
    ['start_blend': 0.2], ['threshold': (0.3, 0.3)]} -> LocalBlend, the words turned into per-token weights of the source and target
    prompts by the conditioning model's word_token_weights(texts, words).  ValueError for anything else."""
    if isinstance(spec, LocalBlend):
        return spec
    if not isinstance(spec, dict):
        raise ValueError(f'local_blend: a LocalBlend or a dict with words, got {type(spec)}')
    extra = set(spec) - BLEND_KEYS
    if extra or 'words' not in spec:
        raise ValueError(f"local_blend: a dict with 'words' and optionally {sorted(BLEND_KEYS - {'words'})}, got keys {sorted(spec)}")
    weights = getattr(cond_stage, 'word_token_weights', None)
    if weights is None:
        raise ValueError('local_blend: the conditioning model has no word_token_weights(texts, words); pass a LocalBlend')

    def pair(key):
        p = spec[key]
        if not isinstance(p, (tuple, list)) or len(p) != 2:
            raise ValueError(f'local_blend: {key} must be a pair (source words, target words), got {p!r}')
        return weights(list(sources), p[0]), weights(list(targets), p[1])

    a_src, a_tgt = pair('words')
    s_src, s_tgt = pair('subtract_words') if spec.get('subtract_words') is not None else (None, None)
    return LocalBlend(a_src, a_tgt, s_src, s_tgt, spec.get('start_blend', 0.2), spec.get('threshold', (0.3, 0.3)))


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
