"""Diffusers-style surface: ``CycleDiffusionPipeline.__call__`` delegating to the same C-ABI loop drivers.

The Diffusers pipeline is NOT part of /root/reference and diffusers is not installed here, so parity at this surface is
*unpinned* (SURVEY.md 8b); the argument list follows diffusers <= 0.2x from the survey.  Semantics are mapped onto the
reference's sampler: ``strength`` -> ``skip_steps = S - int(S * strength)`` (ddim.py:470), DDIMScheduler ``steps_offset=1``
== the ``+1`` of util.py:58, ``posterior_sample`` == sample_xt_next (ddim.py:582-601), ``compute_noise`` == compute_eps
(ddim.py:575-579).  The loop is the engine's lock-step driver (``cdx_cycle_lockstep``): the source chain (source prompt,
source_guidance_scale) and the target chain (prompt, guidance_scale) advance together, one U-Net call per step on the batch
[source segments | target segments] and one fused elementwise kernel that recovers the step's noise and consumes it at once --
no ``z`` buffer exists.  ``two_phase=True`` runs the reference wrapper's encode -> z -> decode instead (same result per sample
up to split-K summation order; tests/test_cycle_gpu.py compares the two).
"""
from dataclasses import dataclass

import torch

from .attn_control import AttentionControl, LocalBlend, MutualSelfControl, PnPControl, resolve_local_blend
from .engine import check_mask
from .schedule import DDIMSchedule, EditFriendlySchedule
from .semantic import SemanticGuidance


@dataclass
class CycleDiffusionPipelineOutput:
    images: object
    nsfw_content_detected: object = None


class CycleDiffusionPipeline:
    def __init__(self, generator, precision='full'):
        """generator: wrappers._LatentGenerator (engine + U-Net + VAE + text encoder callable).  precision: 'full' or 'autocast'
        (txt2img.py --precision): conditioning, first stage and sampling loop run inside ``engine.precision(precision)``."""
        if precision not in generator.engine.PRECISIONS:
            raise ValueError(f'precision must be one of {sorted(generator.engine.PRECISIONS)}, got {precision!r}')
        self.g = generator
        self.engine = generator.engine
        self.precision = precision
        # the U-Net's output parameterisation is the generator's (SD 2.x "-v": 'v'); the loop drivers convert v inside the step
        pred = getattr(generator, 'parameterization', 'eps')
        if generator.unet.prediction != pred:
            generator.unet.set_prediction(pred)

    @classmethod
    def from_wrapper(cls, wrapper):
        return cls(wrapper.generator, precision=wrapper.precision)

    def _check_image(self, image):
        g = self.g
        assert torch.is_tensor(image) and image.dim() == 4, 'image: float tensor [B,3,H,W] in [0,1] (PIL preprocessing is host glue)'
        # any H x W the first stage and the U-Net can both halve all the way down: no silent resize
        side = g.vae.down * 2 ** (len(g.unet.cfg['channel_mult']) - 1)
        if image.shape[2] % side or image.shape[3] % side:
            raise ValueError(f'image height and width must both be multiples of {side} (the first stage\'s factor {g.vae.down} x '
                             f'2^(len(channel_mult) - 1)), got {image.shape[2]}x{image.shape[3]}')

    @torch.no_grad()
    def generate_mask(self, image, source_prompt, target_prompt, num_maps_per_mask=10, mask_encode_strength=0.5,
                      mask_thresholding_ratio=3.0, num_inference_steps=50, generator=None, output_type='pt', rows_per_call=None):
        """DiffEdit's mask (Couairon et al., 2022): where the U-Net's predictions under the source and the target prompt disagree
        on the noised image is where the edit goes.  image [B,3,H,W] in [0,1] -> float32 [B,1,H,W] in {0, 1} on the device, one mask
        per image, ready for ``mask_image=`` (output_type='latent': [B,1,H/f,W/f] at latent resolution).
        The latent is made as ``__call__`` makes it (same generator draw), then noised num_maps_per_mask times (one further draw,
        [B, n, C, h, w]) to the first timestep of the S-step schedule at mask_encode_strength; the map is the mean over maps and
        channels of |e_tgt - e_src| (UNet.edit_map), the mask is map > mask_thresholding_ratio * mean(map) / 2 per image
        (Engine.edit_mask).  Unlike diffusers' generate_mask: the mean is per image, not over the batch; two U-Net rows per map,
        not four (the guidance scale cancels in the normalisation, so there is none); an all-zero map gives an empty mask.
        rows_per_call: U-Net rows per call (UNet.edit_map's default); the result does not depend on it."""
        g, e = self.g, self.engine
        self._check_image(image)
        S = num_inference_steps
        if not (0 < mask_encode_strength <= 1) or int(S * mask_encode_strength) < 1:
            raise ValueError(f'mask_encode_strength must be in (0, 1] with int(num_inference_steps * strength) >= 1, got '
                             f'{mask_encode_strength} at {S} steps')
        if not (isinstance(num_maps_per_mask, int) and num_maps_per_mask >= 1):
            raise ValueError(f'num_maps_per_mask must be an integer >= 1, got {num_maps_per_mask!r}')
        if not mask_thresholding_ratio > 0:
            raise ValueError(f'mask_thresholding_ratio must be > 0, got {mask_thresholding_ratio}')
        if output_type not in ('pt', 'latent'):
            raise ValueError(f"output_type must be 'pt' or 'latent', got {output_type!r}")
        B = image.shape[0]
        per_image = lambda p: [p] * B if isinstance(p, str) else (list(p) * B if len(p) == 1 else list(p))
        sources, targets = per_image(source_prompt), per_image(target_prompt)
        with e.precision(self.precision):
            rnd = lambda shape: torch.randn(shape, generator=generator)
            c_src = g.get_learned_conditioning(sources)
            c_tgt = g.get_learned_conditioning(targets)
            # t and its noise level from the tables the cycle uses; eta does not enter them
            sched = DDIMSchedule(S, 0.0, S - int(S * mask_encode_strength), g.alphas_cumprod)
            moments = g.encode_first_stage(e.shift_scale(image, -0.5, 2.0))
            lat_shape = (B, moments.shape[1] // 2, moments.shape[2], moments.shape[3])
            x0 = e.vae_posterior(moments, rnd(lat_shape) if g.sample_posterior else None, g.scale_factor)
            noise = rnd((B, num_maps_per_mask) + lat_shape[1:])
            acc = g.unet.edit_map(x0, c_src, c_tgt, sched, noise, rows_per_call)
            _, mask, mask_img = e.edit_mask(acc, num_maps_per_mask, mask_thresholding_ratio,
                                            f=None if output_type == 'latent' else g.vae.down, channels=lat_shape[1])
        return mask if output_type == 'latent' else mask_img

    P2P_KEYS = {'edit_type', 'cross_replace_steps', 'self_replace_steps', 'self_replace_max_tokens', 'token_map', 'equalizer'}
    MUTUAL_KEYS = {'edit_type', 'start_step', 'start_layer'}
    PNP_KEYS = {'edit_type', 'feature_steps', 'attention_steps', 'feature_blocks', 'attention_start_layer'}

    @classmethod
    def _attn_control(cls, kw, source_guidance_scale, two_phase):
        """cross_attention_kwargs -> AttentionControl, MutualSelfControl, PnPControl or None (no 'edit_type'); ValueError for what
        the engine cannot do."""
        if not kw or 'edit_type' not in kw:
            return None
        kind = kw['edit_type']
        if kind in ('replace', 'reweight', 'refine') and 'local_blend' in kw:       # CycleDiffusionPipeline._local_blend's key
            if not isinstance(kw['local_blend'], (LocalBlend, dict)):
                raise ValueError(f"cross_attention_kwargs: local_blend must be an attn_control.LocalBlend or a dict of words, got "
                                 f"{type(kw['local_blend'])}")
            kw = {k: v for k, v in kw.items() if k != 'local_blend'}
        if kind == 'mutual_self':
            extra = set(kw) - cls.MUTUAL_KEYS
            if extra:
                raise ValueError(f"cross_attention_kwargs: keys {sorted(extra)} do not apply to edit_type='mutual_self' (it takes "
                                 f"start_step and start_layer; Prompt-to-Prompt edits are a separate edit_type)")
            if two_phase:
                raise ValueError('mutual self-attention needs the lock-step loop: the source chain does not run during the decode '
                                 '(two_phase=False)')
            try:
                return MutualSelfControl(kw.get('start_step', 4), kw.get('start_layer', 10))
            except ValueError as err:
                raise ValueError(f'cross_attention_kwargs: {err}') from None
        if kind == 'pnp':
            extra = set(kw) - cls.PNP_KEYS
            if extra:
                raise ValueError(f"cross_attention_kwargs: keys {sorted(extra)} do not apply to edit_type='pnp' (it takes feature_steps, "
                                 f"attention_steps, feature_blocks and attention_start_layer)")
            if two_phase:
                raise ValueError('Plug-and-Play needs the lock-step loop: the source chain does not run during the decode (two_phase=False)')
            try:
                return PnPControl(**{k: v for k, v in kw.items() if k != 'edit_type'})
            except ValueError as err:
                raise ValueError(f'cross_attention_kwargs: {err}') from None
        if kind not in ('replace', 'reweight', 'refine'):
            raise ValueError(f"edit_type must be 'replace', 'reweight', 'refine', 'mutual_self' or 'pnp', got {kind!r}")
        extra = set(kw) - cls.P2P_KEYS
        if extra:
            raise ValueError(f'cross_attention_kwargs: unsupported keys {sorted(extra)}')
        for key in ('cross_replace_steps', 'self_replace_steps'):
            if key not in kw:
                raise ValueError(f'cross_attention_kwargs: {key} is required with edit_type')
        if two_phase:
            raise ValueError('attention control needs the lock-step loop: the source chain does not run during the decode (two_phase=False)')
        if source_guidance_scale == 0:
            raise ValueError('attention control needs the source prompt: source_guidance_scale 0 runs no source-prompt row')
        A, eq = kw.get('token_map'), kw.get('equalizer')
        if kind == 'refine' and A is None:
            raise ValueError("edit_type='refine' needs a token_map (the prompts' alignment: attn_control.refine_token_map)")
        if A is not None:
            if not torch.is_tensor(A) or A.dim() not in (2, 3) or A.shape[-1] != A.shape[-2]:
                raise ValueError(f'token_map: expected a tensor [L,L] or [B,L,L], got {tuple(A.shape) if torch.is_tensor(A) else type(A)}')
            A = A.to(torch.float32)
        own = None
        if kind == 'refine':
            colsum = A.sum(dim=-2)                        # per target token: how much of it the source supplies
            if not bool(torch.isfinite(colsum).all()) or bool((colsum < -1e-6).any()) or bool((colsum > 1 + 1e-6).any()):
                raise ValueError('token_map: with refine every column sum must lie in [0, 1]')
            own = (1.0 - colsum).clamp_min(0.0)           # the rest of each target token is its own attention
        if eq is not None:
            if not torch.is_tensor(eq) or eq.dim() not in (1, 2) or (A is not None and eq.shape[-1] != A.shape[-1]):
                raise ValueError(f'equalizer: expected a tensor [L] or [B,L] matching token_map, got '
                                 f'{tuple(eq.shape) if torch.is_tensor(eq) else type(eq)}')
            eq = eq.to(torch.float32)
            L = eq.shape[-1]
            base = A if A is not None else torch.eye(L)
            A = base * eq.unsqueeze(-2)                   # token_map . diag(equalizer)
            if own is not None:
                own = own * eq                            # (1 - colsum) . equalizer
        try:
            return AttentionControl(kw['cross_replace_steps'], kw['self_replace_steps'], kw.get('self_replace_max_tokens', 256), A, own)
        except ValueError as err:
            raise ValueError(f'cross_attention_kwargs: {err}') from None

    @staticmethod
    def _local_blend(kw, source_guidance_scale, guidance_scale, two_phase, editing_prompt):
        """cross_attention_kwargs['local_blend'] as given (a LocalBlend or a dict of words, resolved once the prompts are known), or
        None; ValueError where LocalBlend cannot run.  Without an edit_type the dict may hold nothing else."""
        if not kw or 'local_blend' not in kw:
            return None
        if 'edit_type' not in kw and set(kw) != {'local_blend'}:
            raise ValueError(f"cross_attention_kwargs: keys {sorted(set(kw) - {'local_blend'})} need an edit_type")
        if two_phase:
            raise ValueError('LocalBlend needs the lock-step loop: it blends the target chain with the source chain (two_phase=False)')
        if editing_prompt is not None:
            raise ValueError('LocalBlend does not combine with semantic guidance (editing_prompt) in one loop')
        if source_guidance_scale == 0:
            raise ValueError('LocalBlend needs the source prompt: source_guidance_scale 0 runs no source-prompt row')
        if guidance_scale == 0:
            raise ValueError('LocalBlend needs the target prompt: guidance_scale 0 runs no target-prompt row')
        return kw['local_blend']

    def _token_counts(self, concepts, given):
        """LEDITS++'s token span per concept: the caller's edit_token_counts, or the conditioning model's count capped at L - 2."""
        if given is not None:
            return given
        counts = getattr(self.g.cond_stage, 'token_counts', None)
        if counts is None:
            raise ValueError('use_cross_attn_mask / use_intersect_mask: the conditioning model has no token_counts(texts); pass '
                             'edit_token_counts')
        L = int(self.g.get_learned_conditioning(concepts[:1]).shape[1])
        return [max(1, min(int(n), L - 2)) for n in counts(concepts)]

    @torch.no_grad()
    def __call__(self, prompt, source_prompt, image=None, strength=0.8, num_inference_steps=50, guidance_scale=7.5,
                 source_guidance_scale=1, num_images_per_prompt=1, eta=None, generator=None, prompt_embeds=None, output_type='pt',
                 return_dict=True, callback=None, callback_steps=1, cross_attention_kwargs=None, clip_skip=None, two_phase=False,
                 mask_image=None, paste_back=False, editing_prompt=None, reverse_editing_direction=False, edit_guidance_scale=5,
                 edit_threshold=0.9, edit_cooldown_steps=None, edit_warmup_steps=10, edit_momentum_scale=0.1, edit_mom_beta=0.4,
                 use_cross_attn_mask=False, use_intersect_mask=False, edit_token_counts=None, inversion='cycle'):
        """mask_image: optional float tensor [B,1,H,W] or [1,1,H,W] in [0,1] at the image's size, 1 = "may change" (diffusers'
        convention).  Outside the mask the latent stays on the source image's own chain (cdx_cycle_lockstep_masked), so the
        unmasked region decodes to the image's VAE reconstruction.  paste_back: additionally composite the output with the input
        image at image resolution, so pixels where the mask is 0 are the input image exactly.  A mask needs the lock-step loop:
        ``two_phase=True`` with a mask raises ValueError.  mask_image='auto': the mask is generated from the prompts first, exactly
        ``self.generate_mask(image, source_prompt, prompt, generator=generator, num_inference_steps=num_inference_steps)`` with its
        defaults, on the same generator.

        cross_attention_kwargs: Prompt-to-Prompt attention control (Hertz et al., 2022) when it has an ``edit_type``:
        {'edit_type': 'replace' | 'reweight' | 'refine', 'cross_replace_steps': f, 'self_replace_steps': f,
        ['self_replace_max_tokens': n], ['token_map': [L,L] | [B,L,L]], ['equalizer': [L] | [B,L]]}, fractions f in [0, 1] of the
        loop's steps.  The target's cond row takes the source row's attention maps, cross-attention through A = token_map .
        diag(equalizer) (attn_control.replace_token_map builds token_map from two prompts' token ids).  'refine' needs a
        token_map (attn_control.refine_token_map aligns two prompts' token ids) whose column sums lie in [0, 1]: target token j
        takes P_src . A[:, j] and keeps (1 - colsum_j) . eq_j of its own map, so a word the source prompt lacks attends on its own.
        two_phase=True and a source_guidance_scale of 0 raise ValueError.
        'local_blend' (with these edit types, or alone): Prompt-to-Prompt's LocalBlend, an attn_control.LocalBlend or
        {'words': (source_words, target_words), ['subtract_words': (source_words, target_words)], ['start_blend': 0.2],
        ['threshold': (0.3, 0.3)]}, the words (a word or a tuple of words, for every image) turned into per-token weights by the
        conditioning model's word_token_weights.  From step int(start_blend * n) of the loop's n steps on, the target chain keeps
        its own latent only where the blend words' cross-attention, summed over the 1/4-resolution layers and every step so far,
        is above threshold[0] of its maximum (after a 3x3 max-pool) in the source or the target prompt, and not above threshold[1]
        for a subtract word; elsewhere it takes the source chain's.  Unlike mask_image, which is fixed for the loop, the mask is
        recomputed at every step and follows the object; with mask_image the two multiply, and paste_back still pastes outside
        mask_image.  It composes with every inversion and precision='autocast'; with edit_type 'mutual_self' or 'pnp',
        editing_prompt, two_phase=True, a source_guidance_scale or guidance_scale of 0, or latent sides that are not multiples of 4
        it raises ValueError.  Any other dict without 'edit_type' is ignored.
        {'edit_type': 'mutual_self', ['start_step': 4], ['start_layer': 10]}: MasaCtrl's mutual self-attention (Cao et al., 2023)
        instead, for non-rigid edits (a pose or a layout change): from loop step start_step on, in the SpatialTransformers from
        index start_layer on (16 in SD v1 / 2.x; the defaults control the decoder's two finest levels), the target rows keep their
        own queries and attend over the source rows' keys and values (attn_control.MutualSelfControl).  Prompt-to-Prompt keys,
        other keys and two_phase=True raise ValueError; it composes with mask_image.
        {'edit_type': 'pnp', ['feature_steps': 0.8], ['attention_steps': 0.5], ['feature_blocks': (4,)], ['attention_start_layer': 8]}:
        Plug-and-Play diffusion features (Tumanyan et al., 2023) instead, for structure-preserving text-guided translation: in the
        first feature_steps of the loop's steps the ResBlocks of the output blocks feature_blocks give the target rows the source
        row's features (out_layers of its in_layers output, on the target's own skip), and in the first attention_steps the
        SpatialTransformers from index attention_start_layer on give them the source row's self-attention queries and keys
        (attn_control.PnPControl).  source_prompt="" with source_guidance_scale=0 reproduces PnP's unconditional source branch.
        Other keys, values out of range and two_phase=True raise ValueError; it composes with mask_image.

        editing_prompt: semantic guidance (SEGA, Brack et al., 2023), named as diffusers' semantic pipelines name it: a str or a list
        of m <= 8 concept prompts added to (reverse_editing_direction False) or removed from (True) the target image, each with its
        own edit_guidance_scale, edit_threshold (the percentile in [0, 1) of its term's magnitude per latent plane above which it
        applies) and edit_cooldown_steps (None: every step); a scalar applies to every concept, a list gives one per concept.
        edit_warmup_steps, edit_momentum_scale and edit_mom_beta are shared (semantic.SemanticGuidance).  Steps are counted over the
        loop's int(num_inference_steps * strength) steps.  The concept prompts are broadcast to every image.  It composes with
        mask_image and precision='autocast'; two_phase=True, an edit_type in cross_attention_kwargs, list lengths other than m and
        a per-concept warmup list raise ValueError.  Without editing_prompt the edit_* arguments are unused.

        use_cross_attn_mask / use_intersect_mask: LEDITS++'s implicit masks (Brack et al., 2024; its argument names), both off by
        default.  Each concept's term is kept where its own cross-attention map (its prompt's tokens, at the U-Net's 1/4-resolution
        cross-attention layers, smoothed) is in its edit_threshold-th percentile, instead of SEGA's per-channel rule; intersect also
        requires the term's channel-summed magnitude to be in its percentile (and implies the attention mask).  The tokens of each
        concept come from the conditioning model's token_counts(concepts) (capped at the context length - 2), or from
        edit_token_counts (an int or one per concept), which a conditioning callable without token_counts needs.  The latent's sides
        must be multiples of 4.  A mask flag without editing_prompt raises ValueError.

        inversion: how the source chain is made.  'cycle' (default): CycleDiffusion's DPM-Encoder, a DDIM posterior chain at eta
        (None: 0.1).  'ddpm' and 'dpmsolver++': LEDITS++'s edit-friendly inversion (Brack et al., 2024), the source's x at every
        step drawn from q(x_t | x0) on its own and each step's noise recovered from consecutive draws (Huberman-Spiegelglas et al.,
        2024), stepped by the eta = 1 DDIM step ('ddpm') or the second-order SDE-DPM-Solver++ step ('dpmsolver++',
        schedule.EditFriendlySchedule).  Both are stochastic by construction: an eta other than 1 raises ValueError.  The generator
        is drawn from identically under every inversion, and every control above composes with each.  two_phase=True with an
        edit-friendly inversion raises ValueError."""
        if inversion not in ('cycle',) + tuple(EditFriendlySchedule.SOLVERS):
            raise ValueError(f"inversion must be 'cycle', 'ddpm' or 'dpmsolver++', got {inversion!r}")
        if inversion == 'cycle':
            eta = 0.1 if eta is None else eta
        else:
            if eta is not None and eta != 1:
                raise ValueError(f'inversion={inversion!r} samples at eta = 1 by construction, got eta={eta}')
            if two_phase:
                raise ValueError(f'inversion={inversion!r} runs in the lock-step loop only (two_phase=False)')
        attn_control = self._attn_control(cross_attention_kwargs, source_guidance_scale, two_phase)
        blend_spec = self._local_blend(cross_attention_kwargs, source_guidance_scale, guidance_scale, two_phase, editing_prompt)
        semantic, concepts = None, None
        if editing_prompt is not None:
            concepts = [editing_prompt] if isinstance(editing_prompt, str) else list(editing_prompt)
            if two_phase:
                raise ValueError('semantic guidance needs the lock-step loop: its terms are formed at every step of the target chain '
                                 '(two_phase=False)')
            if attn_control is not None:
                raise ValueError('semantic guidance does not combine with a cross_attention_kwargs edit_type in one loop')
            semantic = SemanticGuidance.for_concepts(len(concepts), edit_guidance_scale, reverse_editing_direction, edit_threshold,
                                                     edit_cooldown_steps, edit_warmup_steps, edit_momentum_scale, edit_mom_beta,
                                                     use_cross_attn_mask, use_intersect_mask, self._token_counts(concepts, edit_token_counts)
                                                     if use_cross_attn_mask or use_intersect_mask else edit_token_counts)
        elif use_cross_attn_mask or use_intersect_mask:
            raise ValueError('use_cross_attn_mask / use_intersect_mask mask the semantic guidance terms: pass editing_prompt')
        if strength < 0 or strength > 1:
            raise ValueError(f'The value of strength should in [0.0, 1.0] but is {strength}')
        if not isinstance(callback_steps, int) or callback_steps <= 0:
            raise ValueError('`callback_steps` has to be a positive integer')
        if mask_image is not None and two_phase:
            raise ValueError('mask_image needs the lock-step loop: the two-phase z holds noises, not the source chain (two_phase=False)')
        if paste_back and mask_image is None:
            raise ValueError('paste_back needs a mask_image')
        if isinstance(mask_image, str):
            if mask_image != 'auto':
                raise ValueError(f"mask_image: a tensor or 'auto', got {mask_image!r}")
            if prompt is None:
                raise ValueError("mask_image='auto' generates the mask from the prompt text: pass prompt")
            mask_image = self.generate_mask(image, source_prompt, prompt, generator=generator, num_inference_steps=num_inference_steps)
        assert inversion != 'cycle' or eta > 0, 'CycleDiffusion needs a stochastic sampler (eta > 0), ddim.py:268'
        g, e = self.g, self.engine
        prompts = [prompt] if isinstance(prompt, str) else list(prompt)
        sources = [source_prompt] if isinstance(source_prompt, str) else list(source_prompt)
        self._check_image(image)
        B = image.shape[0] * num_images_per_prompt
        if mask_image is not None:
            if not (torch.is_tensor(mask_image) and mask_image.dim() == 4 and mask_image.shape[0] in (1, image.shape[0])
                    and tuple(mask_image.shape[1:]) == (1,) + tuple(image.shape[2:])):
                raise ValueError(f'mask_image: expected [{image.shape[0]} or 1, 1, {image.shape[2]}, {image.shape[3]}], got '
                                 f'{tuple(mask_image.shape) if torch.is_tensor(mask_image) else type(mask_image)}')
            mask_image = check_mask(mask_image, mask_image.shape, e.device, 'mask_image')
            if mask_image.shape[0] == 1:
                mask_image = mask_image.expand(image.shape[0], -1, -1, -1)
            mask_image = mask_image.repeat_interleave(num_images_per_prompt, dim=0).contiguous()
        if num_images_per_prompt > 1:
            image = image.repeat_interleave(num_images_per_prompt, dim=0)
            prompts = [p for p in prompts for _ in range(num_images_per_prompt)]
            sources = [p for p in sources for _ in range(num_images_per_prompt)]
        if len(prompts) == 1 and B > 1:
            prompts, sources = prompts * B, sources * B
        local_blend = resolve_local_blend(blend_spec, g.cond_stage, sources, prompts) if blend_spec is not None else None
        with e.precision(self.precision):
            rnd = lambda shape: torch.randn(shape, generator=generator)
            c_tgt = prompt_embeds if prompt_embeds is not None else g.get_learned_conditioning(prompts)
            c_src = g.get_learned_conditioning(sources)
            uc = g.get_learned_conditioning(B * [''])
            c_edit = g.get_learned_conditioning(concepts).unsqueeze(0).expand(B, -1, -1, -1).contiguous() if concepts else None
            S = num_inference_steps
            skip = S - min(int(S * strength), S)
            sched = DDIMSchedule(S, eta, skip, g.alphas_cumprod) if inversion == 'cycle' else \
                EditFriendlySchedule(S, skip, g.alphas_cumprod, solver=inversion)
            x = e.shift_scale(image, -0.5, 2.0)
            moments = g.encode_first_stage(x)
            lat_shape = (B, moments.shape[1] // 2, moments.shape[2], moments.shape[3])
            x0 = e.vae_posterior(moments, rnd(lat_shape) if g.sample_posterior else None, g.scale_factor)
            n_rec = sched.refine_steps
            noise = torch.zeros((n_rec + 1,) + lat_shape)
            noise[0] = rnd(lat_shape)
            for i in range(n_rec):
                if sched.refine_steps - 1 - i != 0:
                    noise[1 + i] = rnd(lat_shape)
            if two_phase:
                z = g.unet.latent_encode(x0, c_src, uc, source_guidance_scale, sched, n_rec, noise)
                latents = g.unet.latent_decode(z, c_tgt, uc, guidance_scale, sched)
            else:
                mask = e.mask_pool(mask_image, g.vae.down) if mask_image is not None else None
                latents = g.unet.cycle_lockstep(x0, c_src, c_tgt, uc, source_guidance_scale, guidance_scale, sched, noise, mask=mask,
                                                attn_control=attn_control, semantic=semantic, c_edit=c_edit, local_blend=local_blend)
            if callback is not None:
                callback(n_rec - 1, sched.t_loop[-1], latents)
            if paste_back:
                img = e.mask_composite(g.decode_first_stage(latents), image, mask_image)
            else:
                img = e.shift_scale(g.decode_first_stage(latents), 1.0, 0.5).clamp(0, 1)
        if output_type == 'np':
            img = img.permute(0, 2, 3, 1).float().cpu().numpy()
        elif output_type == 'pil':
            from PIL import Image
            arr = (img.permute(0, 2, 3, 1).float().cpu().numpy() * 255).round().astype('uint8')
            img = [Image.fromarray(a) for a in arr]
        if not return_dict:
            return (img, None)
        return CycleDiffusionPipelineOutput(images=img)
