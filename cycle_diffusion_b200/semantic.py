"""Semantic guidance (SEGA, Brack et al., 2023; the editing term of LEDITS++) for the lock-step cycle.

Each concept ("glasses", "a hat", "snow") adds or removes itself from the target chain's image with its own strength and direction,
without a rewritten prompt.  Its term is its prompt's U-Net output minus the unconditional one, scaled, and kept only where it is
strongest: at or above the threshold-th percentile of its magnitude over each image's latent plane, per channel.  A momentum over
the steps accumulates the terms before the warmup ends.  The engine runs the concept rows in the step's one U-Net call and the
whole term in its fused step kernel, after one launch that selects each plane's percentile exactly (include/cdx.h,
cdx_cycle_lockstep_semantic); this module holds the value the Python surfaces take.

LEDITS++ (Brack et al., 2024) makes each edit local with an implicit mask per concept: the concept's own cross-attention map (its
words' probabilities, summed over the U-Net's 1/4-resolution cross-attention layers and heads, then smoothed) says where it lands,
and its term is kept only where that map is in its top percentile, optionally intersected with the term's channel-summed magnitude
(use_cross_attn_mask, use_intersect_mask; cdx_cycle_lockstep_semantic_attn).
"""
import ctypes
import math
from dataclasses import dataclass

from . import _cabi

MAX_CONCEPTS = _cabi.CDX_SEMANTIC_MAX


def _number(name, v):
    if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(float(v)):
        raise ValueError(f'{name} must be a finite number, got {v!r}')
    return float(v)


def _per_concept(name, v, m, check):
    """A scalar broadcast to m concepts, or a list / tuple of exactly m values; each passed through check(name, value)."""
    vals = list(v) if isinstance(v, (list, tuple)) else [v] * m
    if len(vals) != m:
        raise ValueError(f'{name}: {len(vals)} values for {m} editing prompts')
    return tuple(check(name, x) for x in vals)


def _threshold(name, v):
    v = _number(name, v)
    if not 0.0 <= v < 1.0:
        raise ValueError(f'{name} must lie in [0, 1), got {v!r}')
    return v


def _flag(name, v):
    if not isinstance(v, bool):
        raise ValueError(f'{name} must be a bool, got {v!r}')
    return v


def _tokens(name, v):
    if isinstance(v, bool) or not isinstance(v, int) or v < 1:
        raise ValueError(f'{name} must be an integer >= 1, got {v!r}')
    return v


def _steps(name, v):
    if v is None:
        return None
    if isinstance(v, bool) or not isinstance(v, int) or v < 0:
        raise ValueError(f'{name} must be an integer >= 0 or None, got {v!r}')
    return v


@dataclass(frozen=True)
class SemanticGuidance:
    """SEGA's parameters for m concepts (1 <= m <= 8), named as diffusers' SemanticStableDiffusionPipeline names them; a scalar
    applies to every concept, a list gives one value per concept.  At loop step i (0-based, of the steps that run after strength's
    skip) concept k's term is sigma_k (o_k - o_uc), sigma_k = -edit_guidance_scale[k] when reverse_editing_direction[k] else
    +edit_guidance_scale[k], kept where its magnitude reaches the edit_threshold[k]-th percentile of its h x w plane (per image and
    channel) and while i < edit_cooldown_steps[k] (None: every step).  G = sum of the terms + edit_momentum_scale * nu, nu <-
    edit_mom_beta * nu + (1 - edit_mom_beta) * G; the target chain's guided output takes G from step edit_warmup_steps on.
    use_cross_attn_mask (LEDITS++): concept k's term is kept where the smoothed cross-attention map of its tokens 1..edit_token_counts[k]
    reaches its edit_threshold[k]-th percentile instead (the per-channel rule is not applied); use_intersect_mask also requires the
    channel sum of |term| to reach its percentile over the plane, and implies the attention mask.  edit_token_counts (one per concept,
    each >= 1; at most the context length - 2, checked by the engine) is needed with either flag."""
    edit_guidance_scale: tuple = (5.0,)
    reverse_editing_direction: tuple = (False,)
    edit_threshold: tuple = (0.9,)
    edit_cooldown_steps: tuple = (None,)
    edit_warmup_steps: int = 10
    edit_momentum_scale: float = 0.1
    edit_mom_beta: float = 0.4
    use_cross_attn_mask: bool = False
    use_intersect_mask: bool = False
    edit_token_counts: tuple = None

    @classmethod
    def for_concepts(cls, m, edit_guidance_scale=5, reverse_editing_direction=False, edit_threshold=0.9, edit_cooldown_steps=None,
                     edit_warmup_steps=10, edit_momentum_scale=0.1, edit_mom_beta=0.4, use_cross_attn_mask=False, use_intersect_mask=False,
                     edit_token_counts=None):
        """m concepts; scalars broadcast to all of them, lists must have m entries.  ValueError otherwise."""
        if isinstance(m, bool) or not isinstance(m, int) or not 1 <= m <= MAX_CONCEPTS:
            raise ValueError(f'semantic guidance takes 1 to {MAX_CONCEPTS} editing prompts, got {m!r}')
        return cls(_per_concept('edit_guidance_scale', edit_guidance_scale, m, _number),
                   _per_concept('reverse_editing_direction', reverse_editing_direction, m, _flag),
                   _per_concept('edit_threshold', edit_threshold, m, _threshold),
                   _per_concept('edit_cooldown_steps', edit_cooldown_steps, m, _steps),
                   edit_warmup_steps, edit_momentum_scale, edit_mom_beta, use_cross_attn_mask, use_intersect_mask,
                   None if edit_token_counts is None else _per_concept('edit_token_counts', edit_token_counts, m, _tokens))

    def __post_init__(self):
        m = len(self.edit_guidance_scale) if isinstance(self.edit_guidance_scale, (list, tuple)) else 0
        if not 1 <= m <= MAX_CONCEPTS:
            raise ValueError(f'semantic guidance takes 1 to {MAX_CONCEPTS} concepts, got {m}')
        for name, check in (('edit_guidance_scale', _number), ('reverse_editing_direction', _flag), ('edit_threshold', _threshold),
                            ('edit_cooldown_steps', _steps)):
            v = getattr(self, name)
            if not isinstance(v, (list, tuple)):
                raise ValueError(f'{name}: one value per concept (a tuple of {m}), got {v!r}')
            object.__setattr__(self, name, _per_concept(name, v, m, check))
        w = self.edit_warmup_steps
        if isinstance(w, (list, tuple)):
            raise ValueError('edit_warmup_steps: one warmup is shared by all concepts (the momentum is), got a list')
        if isinstance(w, bool) or not isinstance(w, int) or w < 0:
            raise ValueError(f'edit_warmup_steps must be an integer >= 0, got {w!r}')
        _number('edit_momentum_scale', self.edit_momentum_scale)
        if not 0.0 <= _number('edit_mom_beta', self.edit_mom_beta) <= 1.0:
            raise ValueError(f'edit_mom_beta must lie in [0, 1], got {self.edit_mom_beta!r}')
        _flag('use_cross_attn_mask', self.use_cross_attn_mask)
        _flag('use_intersect_mask', self.use_intersect_mask)
        if self.edit_token_counts is not None:
            if not isinstance(self.edit_token_counts, (list, tuple)):
                raise ValueError(f'edit_token_counts: one count per concept (a tuple of {m}), got {self.edit_token_counts!r}')
            object.__setattr__(self, 'edit_token_counts', _per_concept('edit_token_counts', self.edit_token_counts, m, _tokens))
        if self.mask_mode and self.edit_token_counts is None:
            raise ValueError('use_cross_attn_mask / use_intersect_mask need edit_token_counts: the tokens of each concept prompt')

    @property
    def m(self):
        return len(self.edit_guidance_scale)

    @property
    def mask_mode(self):
        """0 SEGA's per-channel thresholds, 1 LEDITS++'s attention mask, 2 the attention mask intersected with the magnitude mask."""
        return 2 if self.use_intersect_mask else 1 if self.use_cross_attn_mask else 0

    def attn_mask_struct(self, L):
        """-> cdx_semantic_attn_mask for contexts of L tokens; a count outside 1..L-2 raises ValueError."""
        for k, n in enumerate(self.edit_token_counts):
            if not 1 <= n <= L - 2:
                raise ValueError(f'edit_token_counts[{k}] = {n}: a concept of a {L}-token context has 1 to {L - 2} own tokens')
        counts = list(self.edit_token_counts) + [0] * (MAX_CONCEPTS - self.m)
        return _cabi.SemanticAttnMaskC(int(self.mask_mode == 2), (ctypes.c_int * MAX_CONCEPTS)(*counts))

    def signed_scales(self):
        return tuple(-s if r else s for s, r in zip(self.edit_guidance_scale, self.reverse_editing_direction))

    def c_struct(self, n):
        """-> cdx_semantic_guidance for an n-step loop (a cooldown of None: n, every step guides).  beta1 = fp32(1 - beta), the
        subtraction in double."""
        m = self.m
        pad = lambda vals, fill: list(vals) + [fill] * (MAX_CONCEPTS - m)
        cool = [n if c is None else c for c in self.edit_cooldown_steps]
        beta = float(self.edit_mom_beta)
        return _cabi.SemanticGuidanceC(m, (ctypes.c_float * MAX_CONCEPTS)(*pad(self.signed_scales(), 0.0)),
                                       (ctypes.c_float * MAX_CONCEPTS)(*pad(self.edit_threshold, 0.0)), (ctypes.c_int * MAX_CONCEPTS)(*pad(cool, 0)),
                                       self.edit_warmup_steps, float(self.edit_momentum_scale), beta, 1.0 - beta)

