"""Drop-in `gan_wrapper` classes: the reference's plugin surface for the hot path, backed by libcdx.

Mirrors (same constructor kwargs, method names, argument meaning, return layouts and precondition checks):
  SDStochasticTextWrapper            ref model/gan_wrapper/stable_diffusion_stochastic_text_wrapper.py:100-253
  SD2StochasticTextWrapper           the same wrapper for the SD 2.x checkpoints (v2-1_512 eps, v2-1_768 v-prediction)
  LatentDiffStochasticTextWrapper    ref model/gan_wrapper/latentdiff_stochastic_text_wrapper.py:102-252
  DDPMDDIMWrapper                    ref model/gan_wrapper/ddpm_ddim_wrapper.py:317-538
  get_gan_wrapper                    ref model/gan_wrapper/get_gan_wrapper.py:3-31

Differences that are deliberate and documented in INTEGRATION.md:
  * weights come from a reference-format ``state_dict`` / checkpoint path given by keyword (or ``'synthetic'``);
    the packed blob can be shared between wrappers and broadcast across ranks;
  * the text encoder is ``cond_stage(list[str]) -> [B,77,D]``: either an injected callable or the in-engine towers
    (``ClipTextCondStage`` / ``BertTextCondStage``, SURVEY.md 8f-1), which are built automatically from the checkpoint's
    ``cond_stage_model.*`` keys when a host ``tokenizer`` is given.  The deterministic ``SyntheticTextEncoder`` stand-in is
    used ONLY together with ``state_dict='synthetic'``; a real checkpoint without a conditioning model raises;
  * random draws are taken from the torch CPU generator in the reference's order and uploaded, so a run is
    reproducible against the reference CPU path under the same ``torch.manual_seed``;
  * Directional-CLIP ranking of the ensemble is an injected callable (SURVEY.md 8f-3); with a single ensemble
    member no ranking is needed.
"""
import hashlib
import os

import numpy as np
import torch

from . import specs
from .attn_control import resolve_local_blend
from .engine import Engine, UNet, VAE, check_mask
from .ensemble import EnsemblePlan, MemberNoise
from .schedule import DDIMSchedule, PixelSchedule, same_schedule

# Recovery steps per chunk of the lock-step pixel loop (DDPMDDIMWrapper.cycle): device memory holds one chunk of noise, not
# es_steps of it.  At 256^2 and batch 8 a chunk is 32 x 8 x 3 x 256^2 x 4 B = 0.2 GB (the two-phase path: 1.3 GB per image at 850 steps).
LOCKSTEP_CHUNK = 32

# U-Net rows per call of the lock-step ensemble search (the text wrappers' ensemble_rows default).  The row-budget sweep of
# tools/bench_ensemble.py (DESIGN.md section 8; SD v1-4, H100) found the time per sample-forward falling only slightly from 12 to
# 48 rows (11.70 -> 11.28 ms), and a 96-row SD call exceeds the engine's GroupNorm statistics pool, so 48 it is.
ENSEMBLE_ROWS = 48


class ClipTextCondStage:
    """In-engine conditioning model: drop-in for ``model.get_learned_conditioning`` with FrozenCLIPEmbedder behind it
    (ddpm.py:545-556 -> encoders/modules.py:148-158): ``list[str] -> [B, 77, 768]`` on the engine's device.

    ``tokenizer``: callable ``list[str] -> LongTensor [B, L]`` -- e.g. ``lambda t: hf_tok(t, truncation=True, max_length=77,
    padding='max_length', return_tensors='pt')['input_ids']`` with HF ``CLIPTokenizer`` (the BPE vocabulary is host data and
    not part of the engine).  ``state_dict``: HF CLIPTextModel keys, optionally under ``prefix`` (the SD checkpoint keeps them
    under ``cond_stage_model.transformer.``)."""

    def __init__(self, engine, state_dict, tokenizer, cfg=None, prefix=''):
        from .engine import TextEncoder
        self.cfg = cfg or specs.clip_text_config()
        self.tokenizer = tokenizer
        self.encoder = TextEncoder(engine, self.cfg)
        self.encoder.load_state_dict({k: v for k, v in state_dict.items() if k.startswith(prefix)}, prefix=prefix)

    END_ID = 49407      # CLIP's <|endoftext|> (the OpenCLIP tokenizer's too)

    def __call__(self, texts):
        ids = self.tokenizer(list(texts))
        assert ids.dim() == 2 and ids.shape[0] == len(texts), 'tokenizer must return [B, L] ids'
        return self.encoder(ids)

    def token_counts(self, texts):
        """The prompt's own tokens per text (LEDITS++'s attention masks read tokens 1..n): the position of the first end token after
        the start token, minus 1 (the whole row when it has none)."""
        ids = self.tokenizer(list(texts))
        out = []
        for row in ids.tolist():
            end = next((j for j in range(1, len(row)) if row[j] == self.END_ID), len(row))
            out.append(end - 1)
        return out

    def word_token_weights(self, texts, words):
        """LocalBlend's per-token weights of `words` in each text (attn_control.word_token_weights over the tokenizer's ids):
        words is a word, a tuple of words for every text, or one tuple per text; a word is the token run the tokenizer gives it
        alone (between its start and end tokens).  -> float32 [B, L]; ValueError when a word is not in its text."""
        from .attn_control import word_lists, words_weights
        per_text = word_lists(texts, words)
        ids = self.tokenizer(list(texts))
        runs = {w: self._word_run(w) for ws in per_text for w in ws}
        return words_weights(ids.tolist(), [[runs[w] for w in ws] for ws in per_text], ids.shape[1])

    def _word_run(self, word):
        row = self.tokenizer([word])[0].tolist()
        end = next((j for j in range(1, len(row)) if row[j] == self.END_ID), len(row))
        return row[1:end]


class BertTextCondStage(ClipTextCondStage):
    """Same for the LDM text2img-large conditioning model: BERTEmbedder (encoders/modules.py:79-102; 32 x 1280 x_transformer
    encoder over BERT word pieces).  ``tokenizer``: e.g. HF ``BertTokenizerFast`` with ``padding='max_length', max_length=77``
    (modules.py:66-72); the LDM checkpoint keeps the weights under ``cond_stage_model.``."""

    END_ID = 102        # BERT's [SEP]

    def __init__(self, engine, state_dict, tokenizer, cfg=None, prefix=''):
        super().__init__(engine, state_dict, tokenizer, cfg or specs.bert_text_config(), prefix)


class OpenClipTextCondStage(ClipTextCondStage):
    """SD 2.x conditioning model: FrozenOpenCLIPEmbedder(arch="ViT-H-14", layer="penultimate").encode_with_transformer after
    tokenisation -- token + positional embedding, the first 23 of the 24 pre-LN blocks (causal attention, exact-erf GELU MLP),
    ln_final -> [B, 77, 1024].  ``state_dict``: the checkpoint's OpenCLIP keys under ``prefix`` (``cond_stage_model.model.``),
    mapped to the engine's HF-named CDX_TEXT_OPENCLIP tower by specs.openclip_to_hf.  ``tokenizer``: a host callable
    ``list[str] -> LongTensor [B, 77]`` (open_clip.tokenize: start / end tokens, zero padding)."""

    def __init__(self, engine, state_dict, tokenizer, cfg=None, prefix='cond_stage_model.model.'):
        from .engine import TextEncoder
        self.cfg = cfg or specs.openclip_h14_text_config()
        self.tokenizer = tokenizer
        self.encoder = TextEncoder(engine, self.cfg)
        self.encoder.load_state_dict(specs.openclip_to_hf(state_dict, self.cfg['layers'], prefix))


class SyntheticTextEncoder:
    """Deterministic stand-in for FrozenCLIPEmbedder / BERTEmbedder: prompt string -> N(0,1) tokens [77, dim].

    Same interface as ``model.get_learned_conditioning`` (ddpm.py:545-556).  Not a language model: it only gives
    distinct, reproducible conditioning tensors so the sampling path can be exercised without checkpoints.
    """

    def __init__(self, dim, n_tokens=77, device='cpu'):
        self.dim, self.n_tokens, self.device = dim, n_tokens, device

    def __call__(self, texts):
        assert isinstance(texts, list) and isinstance(texts[0], str)       # SDW:29-30
        out = []
        for t in texts:
            seed = int.from_bytes(hashlib.sha256(t.encode('utf-8')).digest()[:4], 'little')
            g = torch.Generator().manual_seed(seed)
            out.append(torch.randn(self.n_tokens, self.dim, generator=g))
        return torch.stack(out).to(self.device)

    def token_counts(self, texts):
        """The whitespace word count of each text (the stand-in has no tokenizer)."""
        return [len(t.split()) for t in texts]

    def word_token_weights(self, texts, words):
        """LocalBlend's per-token weights of `words` in each text, whitespace word k being token k + 1 (after the start token), as
        token_counts counts them; a word of several whitespace words is their run.  -> float32 [B, n_tokens]."""
        from .attn_control import word_lists, words_weights
        per_text = word_lists(texts, words)
        return words_weights([['<start>'] + t.split() for t in texts], [[w.split() for w in ws] for ws in per_text], self.n_tokens)


def _load_sd(state_dict, ckpt_default, synth_params, seed):
    if isinstance(state_dict, dict):
        return state_dict
    if state_dict == 'synthetic':
        return specs.synth_state_dict(synth_params, seed)
    path = state_dict if isinstance(state_dict, str) else ckpt_default
    if not os.path.exists(path):
        raise FileNotFoundError(f'checkpoint {path} not found; pass state_dict=<dict>, a path, or "synthetic"')
    sd = torch.load(path, map_location='cpu')
    return sd['state_dict'] if 'state_dict' in sd else sd       # txt2img.py:27-32 / DW:378-379


def encode_noise(sched, n_rec, shape):
    """Draws of _ddpm_ddim_encoding in order: x_T (ddim.py:479), then one per step except index==0 (ddim.py:583-584, 599: the last
    step returns x0 without a draw)."""
    noise = torch.zeros((n_rec + 1,) + tuple(shape))
    noise[0] = torch.randn(shape)
    for i in range(n_rec):
        if sched.refine_steps - 1 - i != 0:
            noise[1 + i] = torch.randn(shape)
    return noise


class _LatentGenerator:
    """What the text wrappers call ``self.generator`` (LatentDiffusion): U-Net + first stage + cond stage."""

    def __init__(self, engine, unet, vae, cond_stage, channels, image_size, scale_factor, sample_posterior):
        self.engine, self.unet, self.vae, self.cond_stage = engine, unet, vae, cond_stage
        self.channels, self.image_size, self.scale_factor = channels, image_size, scale_factor
        self.sample_posterior = sample_posterior
        self.alphas_cumprod = None      # default LDM linear schedule (v1-inference.yaml:5-9)
        self.parameterization = unet.prediction     # what the U-Net predicts: 'eps', or 'v' for the SD 2.x "-v" models

    def get_learned_conditioning(self, c):
        return self.cond_stage(c)

    def encode_first_stage(self, image):
        return self.vae.encode_moments(image)                              # moments of the DiagonalGaussianDistribution

    def get_first_stage_encoding(self, moments):
        if self.vae.cfg.get('vq'):                                         # VQModelInterface: the encoder output itself (ddpm.py:536-543, tensor branch)
            return self.engine.affine(moments, self.scale_factor, 0.0)
        noise = None
        if self.sample_posterior:                                          # ddpm.py:536-543; distributions.py:36 draws on the CPU
            B, C2, h, w = moments.shape
            noise = torch.randn(B, C2 // 2, h, w)
        return self.engine.vae_posterior(moments, noise, self.scale_factor)

    def encode_image(self, image, resolution):
        """image [B,3,R,R] in [0,1] -> x0: (image - 0.5) * 2.0, then the first stage and its encoding (whose posterior draw comes
        before any noise of the sampling loop)."""
        image = self.engine.shift_scale(image, -0.5, 2.0)
        assert image.shape[2] == image.shape[3] == resolution
        return self.get_first_stage_encoding(self.encode_first_stage(image))

    def decode_first_stage(self, z):
        return self.vae.decode(self.engine.affine(z, 1. / self.scale_factor, 0.0))     # ddpm.py:705


class _StochasticTextWrapperBase(torch.nn.Module):
    RESOLUTION = 512
    LATENT = 64
    CONTEXT_DIM = 768
    SAMPLE_POSTERIOR = True
    CKPT_DIR = 'ckpts/stable_diffusion'
    COND_PREFIX = 'cond_stage_model.transformer.'     # FrozenCLIPEmbedder.transformer (encoders/modules.py:140-146)
    COND_CLASS = ClipTextCondStage

    @classmethod
    def default_checkpoint(cls, source_model_type):
        """SDW:21-23: ``ckpts/stable_diffusion/<source_model_type>``."""
        return os.path.join(cls.CKPT_DIR, str(source_model_type))

    def __init__(self, source_model_type, custom_steps, eta, white_box_steps, skip_steps,
                 encoder_unconditional_guidance_scales=None, decoder_unconditional_guidance_scales=None, n_trials=None, *,
                 engine=None, device=0, state_dict=None, cond_stage=None, ranker=None, unet_config=None, vae_config=None,
                 latent_size=None, resolution=None, generator=None, seed=1234, tokenizer=None, ensemble_batch=16, ensemble_rows=ENSEMBLE_ROWS):
        super().__init__()
        # ensemble members that share a schedule are batched along the batch dimension, up to this many samples per sampling loop
        # (cdx_latent_loop_ens); None / 0 = one member at a time, the reference's loop shape
        self.ensemble_batch = ensemble_batch
        # lock-step ensemble search (cycle_ensemble): U-Net rows per call a chunk of source chains may fill (at least one chain)
        self.ensemble_rows = ensemble_rows
        self.encoder_unconditional_guidance_scales = encoder_unconditional_guidance_scales
        self.decoder_unconditional_guidance_scales = decoder_unconditional_guidance_scales
        self.n_trials = n_trials
        self.eta, self.custom_steps, self.white_box_steps, self.skip_steps = eta, custom_steps, white_box_steps, skip_steps
        self.resolution = resolution or self.RESOLUTION
        # SDW:117: "full" or "autocast" (txt2img.py --precision).  encode / generate / cycle run inside _precision_scope; a value
        # other than these two raises ValueError when the wrapper is called (the reference treats a typo as "full")
        self.precision = "full"
        self.directional_clip = ranker
        if generator is not None:
            self.generator = generator
            self.engine = generator.engine
        else:
            self.engine = engine or Engine(device)
            ucfg = unet_config or specs.sd_unet_config(self.CONTEXT_DIM)
            vcfg = vae_config or specs.kl_f8_config()
            unet, vae = self._build_unet(ucfg), VAE(self.engine, vcfg)
            ckpt = self.default_checkpoint(source_model_type)
            cond = cond_stage
            if state_dict == 'synthetic':
                unet.load_state_dict(specs.synth_state_dict(specs.openai_unet_params(ucfg), seed))
                vae.load_state_dict(specs.synth_state_dict(specs.kl_vae_params(vcfg), seed + 1))
                if cond is None:
                    cond = SyntheticTextEncoder(ucfg['context_dim'])        # random-init weights: random (but reproducible) conditioning
            else:
                sd = _load_sd(state_dict, ckpt, None, seed)
                unet.load_state_dict(sd, prefix='model.diffusion_model.', strict=False)
                vae.load_state_dict(sd, prefix='first_stage_model.', strict=False)
                if cond is None:
                    # the reference builds the conditioning model from the same checkpoint (txt2img.py:27-45); do the same, and never
                    # fall back silently to noise tokens when real weights were loaded
                    has_tower = any(k.startswith(self.COND_PREFIX) for k in sd)
                    if tokenizer is not None and has_tower:
                        cond = self.COND_CLASS(self.engine, sd, tokenizer, prefix=self.COND_PREFIX)
                    else:
                        raise ValueError(
                            f'{type(self).__name__}: a checkpoint was loaded but no conditioning model is available '
                            f'({"no " + self.COND_PREFIX + "* keys in the checkpoint" if not has_tower else "no tokenizer= given"}). '
                            'Pass cond_stage=<callable list[str] -> [B,77,D]> or tokenizer=<callable list[str] -> ids [B,L]> '
                            '(the in-engine text tower is then built from the checkpoint).')
            self.generator = _LatentGenerator(self.engine, unet, vae, cond, ucfg['in_channels'], latent_size or self.LATENT, 0.18215,
                                              self.SAMPLE_POSTERIOR)
        self._dummy = torch.nn.Parameter(torch.zeros(1, device=self.engine.device), requires_grad=False)

    def _build_unet(self, ucfg):
        return UNet(self.engine, ucfg, 'openai')

    def _precision_scope(self):
        """SDW:143-144, 173: ``autocast("cuda")`` when precision == "autocast", else a null context -- here the engine's mma
        mode 5 (single-term fp16 tensor-core products, fp32 activations), the previous mode restored on exit."""
        return self.engine.precision(self.precision)

    # -- helpers mirroring the module-level functions of the reference wrapper
    def _get_condition(self, text, bs):
        assert isinstance(text, list)
        assert isinstance(text[0], str)
        uc = self.generator.get_learned_conditioning(bs * [""])
        c = self.generator.get_learned_conditioning(text)
        return c, uc

    def _encode_noise(self, sched, n_rec, shape):
        return encode_noise(sched, n_rec, shape)

    def _chunks(self, members, bsz):
        per = max(1, (self.ensemble_batch or 1) // max(1, bsz))
        return [members[i:i + per] for i in range(0, len(members), per)]

    def _generate_batched(self, z_ensemble, decode_text):
        """generate() with the members of one schedule batched along B: the conditioning is computed once, the context K / V
        projections once per loop, and (member, scale) pairs share U-Net calls.  Random draws (ddim.py:640) keep the reference order."""
        g = self.generator
        bsz = z_ensemble[0].shape[0]
        c, uc = self._get_condition(decode_text, bsz)
        nsc = len(self.decoder_unconditional_guidance_scales)
        imgs = [None] * (len(z_ensemble) * nsc)
        jobs = {}                                         # skip -> [(output slot, eps_list, scale, extra)]
        for i, z in enumerate(z_ensemble):
            skip_steps = self.skip_steps[i % len(self.skip_steps)]
            if self.white_box_steps != -1:
                eps_list = z.view(bsz, (self.white_box_steps - skip_steps), g.channels, g.image_size, g.image_size)
            else:
                eps_list = z.view(bsz, 1, g.channels, g.image_size, g.image_size)
            sched = DDIMSchedule(self.custom_steps, self.eta, skip_steps, g.alphas_cumprod)
            n_extra = sched.refine_steps - (eps_list.shape[1] - 1)
            for k, scale in enumerate(self.decoder_unconditional_guidance_scales):
                extra = torch.stack([torch.randn(eps_list[:, 0].shape) for _ in range(n_extra)]) if n_extra > 0 else None
                jobs.setdefault(skip_steps, []).append((i * nsc + k, eps_list, float(scale), extra))
        for skip_steps, members in jobs.items():
            sched = DDIMSchedule(self.custom_steps, self.eta, skip_steps, g.alphas_cumprod)
            for chunk in self._chunks(members, bsz):
                zc = torch.cat([m[1].to(self.engine.device) for m in chunk], dim=0)
                sc = torch.tensor([m[2] for m in chunk for _ in range(bsz)])
                ex = torch.cat([m[3] for m in chunk], dim=1) if chunk[0][3] is not None else None
                rep = len(chunk)
                sample = g.unet.latent_decode_ens(zc, c.repeat(rep, 1, 1), uc.repeat(rep, 1, 1), sc, sched, ex)
                dec = g.decode_first_stage(sample)
                for j, m in enumerate(chunk):
                    imgs[m[0]] = dec[j * bsz:(j + 1) * bsz]
        return imgs

    def _encode_batched(self, x0, encode_text):
        g = self.generator
        bsz = x0.shape[0]
        c, uc = self._get_condition(encode_text, bsz)
        assert self.eta > 0                                                       # ddim.py:268
        jobs, order = {}, 0
        for _trial in range(self.n_trials):
            for enc_scale in self.encoder_unconditional_guidance_scales:
                for skip_steps in self.skip_steps:
                    sched = DDIMSchedule(self.custom_steps, self.eta, skip_steps, g.alphas_cumprod)
                    n_rec = max(0, min(sched.refine_steps, self.white_box_steps - skip_steps - 1))
                    noise = self._encode_noise(sched, n_rec, x0.shape)            # drawn in the reference's member order
                    jobs.setdefault((skip_steps, n_rec), []).append((order, float(enc_scale), noise))
                    order += 1
        z_ensemble = [None] * order
        for (skip_steps, n_rec), members in jobs.items():
            sched = DDIMSchedule(self.custom_steps, self.eta, skip_steps, g.alphas_cumprod)
            for chunk in self._chunks(members, bsz):
                rep = len(chunk)
                sc = torch.tensor([m[1] for m in chunk for _ in range(bsz)])
                nz = torch.cat([m[2] for m in chunk], dim=1)
                z = g.unet.latent_encode_ens(x0.repeat(rep, 1, 1, 1), c.repeat(rep, 1, 1), uc.repeat(rep, 1, 1), sc, sched, n_rec, nz)
                for j, m in enumerate(chunk):
                    z_ensemble[m[0]] = z[j * bsz:(j + 1) * bsz].reshape(bsz, -1)
        return z_ensemble

    def generate(self, z_ensemble, decode_text):
        with self._precision_scope():
            return self._generate(z_ensemble, decode_text)

    def _generate(self, z_ensemble, decode_text):
        g = self.generator
        if self.ensemble_batch and len(z_ensemble) * len(self.decoder_unconditional_guidance_scales) > 1:
            return self._generate_batched(z_ensemble, decode_text)
        img_ensemble = []
        for i, z in enumerate(z_ensemble):
            skip_steps = self.skip_steps[i % len(self.skip_steps)]
            bsz = z.shape[0]
            if self.white_box_steps != -1:
                eps_list = z.view(bsz, (self.white_box_steps - skip_steps), g.channels, g.image_size, g.image_size)
            else:
                eps_list = z.view(bsz, 1, g.channels, g.image_size, g.image_size)
            for scale in self.decoder_unconditional_guidance_scales:
                c, uc = self._get_condition(decode_text, bsz)
                sched = DDIMSchedule(self.custom_steps, self.eta, skip_steps, g.alphas_cumprod)
                n_extra = sched.refine_steps - (eps_list.shape[1] - 1)
                extra = None
                if n_extra > 0:                                                   # ddim.py:640: fresh noise where none was recovered
                    extra = torch.stack([torch.randn(eps_list[:, 0].shape) for _ in range(n_extra)])
                sample = g.unet.latent_decode(eps_list, c, uc, scale, sched, extra)
                img_ensemble.append(g.decode_first_stage(sample))
        return img_ensemble

    def encode(self, image, encode_text):
        with self._precision_scope():                  # SDW:173-186: the first stage and the ensemble loops
            return self._encode(image, encode_text)

    def _encode(self, image, encode_text):
        g = self.generator
        x0 = g.encode_image(image, self.resolution)
        bsz = image.shape[0]
        if self.ensemble_batch and self.n_trials * len(self.encoder_unconditional_guidance_scales) * len(self.skip_steps) > 1:
            return self._encode_batched(x0, encode_text)
        z_ensemble = []
        for _trial in range(self.n_trials):
            for enc_scale in self.encoder_unconditional_guidance_scales:
                for skip_steps in self.skip_steps:
                    c, uc = self._get_condition(encode_text, bsz)
                    assert self.eta > 0                                           # ddim.py:268
                    sched = DDIMSchedule(self.custom_steps, self.eta, skip_steps, g.alphas_cumprod)
                    n_rec = max(0, min(sched.refine_steps, self.white_box_steps - skip_steps - 1))
                    noise = self._encode_noise(sched, n_rec, x0.shape)
                    z = g.unet.latent_encode(x0, c, uc, enc_scale, sched, n_rec, noise)
                    z_ensemble.append(z.view(bsz, -1))
        return z_ensemble

    def single_member(self):
        """True when the ensemble has exactly one member whose every step is recovered (the plain CycleDiffusion cycle)."""
        if not (self.n_trials == 1 and len(self.skip_steps) == 1 and len(self.encoder_unconditional_guidance_scales) == 1
                and len(self.decoder_unconditional_guidance_scales) == 1):
            return False
        sched = DDIMSchedule(self.custom_steps, self.eta, self.skip_steps[0], self.generator.alphas_cumprod)
        return self.white_box_steps != -1 and self.white_box_steps - self.skip_steps[0] - 1 >= sched.refine_steps

    def cycle(self, image, encode_text, decode_text, mask=None, attn_control=None, local_blend=None):
        """encode(image, encode_text) followed by forward(z, image, encode_text, decode_text) for a single-member ensemble, on the
        engine's lock-step driver (cdx_cycle_lockstep): both chains advance together, one U-Net call per step on the batch
        [source | target uncond | target cond], and the noise recovered at a step is consumed by the target chain at once -- the
        ``z`` tensor of SDW:169-206 is never materialised.  Same random draws in the same order as encode(); same result per sample
        as the two calls (tests/test_cycle_gpu.py).  Called by TextUnsupervisedTranslation.forward when single_member().  The whole
        cycle runs in the wrapper's precision scope, as encode() and generate() do.

        mask: optional [B,1,R,R] in [0,1] at image resolution, 1 = may change (masked editing): pooled to the latent grid, and
        outside it the translated latent stays on the source image's chain (cdx_cycle_lockstep_masked).
        attn_control: optional attn_control.AttentionControl, Prompt-to-Prompt's "replace" edit, or its "refine" edit when the
        control has an own_weight; attn_control.MutualSelfControl, MasaCtrl's mutual self-attention; or attn_control.PnPControl,
        Plug-and-Play's feature and self-attention injection (UNet.cycle_lockstep).
        local_blend: optional attn_control.LocalBlend, or a dict {'words': (source_words, target_words), ...}
        (attn_control.resolve_local_blend, through the conditioning model): Prompt-to-Prompt's LocalBlend on the target chain."""
        assert self.single_member(), 'cycle(): single-member ensembles only (use encode() + forward())'
        if local_blend is not None:
            local_blend = resolve_local_blend(local_blend, self.generator.cond_stage, encode_text, decode_text)
        with self._precision_scope():
            return self._cycle(image, encode_text, decode_text, mask, attn_control, local_blend)

    def _latent_mask(self, mask, bsz):
        """Image-resolution mask [B,1,R,R] -> the latent grid (mean over the first stage's f x f blocks), or None."""
        if mask is None:
            return None
        R = self.resolution
        mask = check_mask(mask, (bsz, 1, R, R), self.engine.device)
        return self.engine.mask_pool(mask, self.generator.vae.down)

    def _cycle(self, image, encode_text, decode_text, mask=None, attn_control=None, local_blend=None):
        g, e = self.generator, self.engine
        bsz = image.shape[0]
        m = self._latent_mask(mask, bsz)                  # checked before the first random draw
        x0 = g.encode_image(image, self.resolution)
        c_src, uc = self._get_condition(encode_text, bsz)
        c_tgt, _ = self._get_condition(decode_text, bsz)
        assert self.eta > 0
        sched = DDIMSchedule(self.custom_steps, self.eta, self.skip_steps[0], g.alphas_cumprod)
        noise = self._encode_noise(sched, sched.refine_steps, x0.shape)
        sample = g.unet.cycle_lockstep(x0, c_src, c_tgt, uc, self.encoder_unconditional_guidance_scales[0],
                                       self.decoder_unconditional_guidance_scales[0], sched, noise, mask=m, attn_control=attn_control,
                                       local_blend=local_blend)
        return e.shift_scale(g.decode_first_stage(sample), 1.0, 0.5)

    def forward(self, z_ensemble, original_img, encode_text, decode_text):
        img_ensemble = self.generate(z_ensemble, decode_text)
        assert len(img_ensemble) == len(self.decoder_unconditional_guidance_scales) * len(
            self.encoder_unconditional_guidance_scales) * len(self.skip_steps) * self.n_trials
        img_ensemble = [self.engine.shift_scale(img, 1.0, 0.5) for img in img_ensemble]     # Normalize(mean=-1, std=2)
        if len(img_ensemble) == 1:
            return img_ensemble[0]
        self.require_ranker()
        if hasattr(self.directional_clip, 'rank'):        # in-engine DirectionalCLIP (clip_rank.py): scores, argmax and gather stay on the device
            return self.directional_clip.rank(img_ensemble, original_img, encode_text, decode_text)[0]
        scores = []
        for img in img_ensemble:
            _, s = self.directional_clip(img, original_img, encode_text, decode_text)
            assert s.shape == (img.shape[0],)
            scores.append(s)
        best_idx = torch.argmax(torch.stack(scores, dim=1), dim=1)
        return torch.stack([img_ensemble[best_idx[b].item()][b] for b in range(best_idx.shape[0])], dim=0)

    def n_candidates(self):
        return (self.n_trials * len(self.encoder_unconditional_guidance_scales) * len(self.skip_steps)
                * len(self.decoder_unconditional_guidance_scales))

    def require_ranker(self):
        """An ensemble of more than one candidate is ranked by ``ranker``: raise when there is none."""
        if self.n_candidates() > 1 and self.directional_clip is None:
            raise NotImplementedError('ranking an ensemble needs ranker=<callable(img, original_img, encode_text, decode_text) -> (_, score[B])>, '
                                      'e.g. cycle_diffusion_b200.clip_rank.DirectionalCLIP(engine, clip_state_dict, tokenizer) (SURVEY.md 8f-3)')

    def _schedules(self):
        return {skip: DDIMSchedule(self.custom_steps, self.eta, skip, self.generator.alphas_cumprod) for skip in dict.fromkeys(self.skip_steps)}

    def lockstep_ensemble(self):
        """True when cycle_ensemble can run the ensemble search: more than one candidate, eta > 0, every step of every skip
        recovered (white_box_steps - skip - 1 >= refine_steps, as in all published configurations) and a ranker."""
        if self.n_candidates() <= 1 or not self.eta > 0 or self.white_box_steps == -1 or self.directional_clip is None:
            return False
        return all(self.white_box_steps - skip - 1 >= s.refine_steps for skip, s in self._schedules().items())

    def ensemble_plan(self, bsz):
        scheds = self._schedules()
        return EnsemblePlan(self.n_trials, self.encoder_unconditional_guidance_scales, self.skip_steps, self.decoder_unconditional_guidance_scales,
                            bsz, {k: s.refine_steps for k, s in scheds.items()}, self.ensemble_rows), scheds

    def cycle_ensemble(self, image, encode_text, decode_text, mask=None):
        """encode(image, encode_text) followed by forward(z, image, encode_text, decode_text) for an ensemble (lockstep_ensemble()),
        in lock-step and streamed: each (member, sample) pair's DPM-Encoder chain drives its decoder-scale chains with the noise it
        recovers (cdx_latent_cycle_fan), a chain runs a CFG row only when its scale needs one, and each chunk's candidates are
        decoded, scored and folded into a per-sample best (cdx_ensemble_select) as soon as the chunk finishes.  No z and no list of
        candidate images is kept.  Same random draws in the same order as encode().

        -> (img [B,3,R,R] in [0,1], unclamped; best_idx [B] int64 in the reference's candidate order, member * n_dec + k;
        scores [B, candidates]).  Loops and VAE run in the wrapper's precision scope, ranking outside it, as in encode + forward.

        mask: optional [B,1,R,R] in [0,1] at image resolution (masked editing, as in cycle()): every candidate of sample b is
        edited under mask[b] only; the masks are gathered on the device in each chunk's chain order."""
        assert self.lockstep_ensemble(), 'cycle_ensemble(): needs an ensemble with every step recovered, eta > 0 and a ranker'
        g, e, rank = self.generator, self.engine, self.directional_clip
        bsz = image.shape[0]
        m_lat = self._latent_mask(mask, bsz)
        with self._precision_scope():
            x0 = g.encode_image(image, self.resolution)
            c_src, uc = self._get_condition(encode_text, bsz)
            c_tgt, _ = self._get_condition(decode_text, bsz)
        plan, scheds = self.ensemble_plan(bsz)
        noise = MemberNoise(plan, lambda skip: self._encode_noise(scheds[skip], scheds[skip].refine_steps, x0.shape))
        R = self.resolution
        sel = e.ensemble_select(bsz, plan.n_candidates, R, R)
        ref = rank.reference(image, encode_text, decode_text) if hasattr(rank, 'reference') else None
        eb = max(1, self.ensemble_batch or 1)
        K = plan.n_dec
        for chunk in plan.chunks:
            samples = torch.tensor([b for _, b in chunk.chains], device=e.device)
            pick = lambda t: t[samples.to(t.device)]
            with self._precision_scope():
                lat = g.unet.cycle_fan(pick(x0), pick(c_src), pick(c_tgt), pick(uc), [plan.members[m][1] for m, _ in chunk.chains],
                                       [plan.dec_scales] * len(chunk.chains), scheds[chunk.skip], noise.chunk(chunk),
                                       mask=pick(m_lat) if m_lat is not None else None)
                imgs = torch.cat([g.decode_first_stage(lat[i:i + eb]) for i in range(0, lat.shape[0], eb)])
            imgs = e.shift_scale(imgs, 1.0, 0.5)                                            # Normalize(mean=-1, std=2)
            cand = [plan.candidate(m, k) for m, _ in chunk.chains for k in range(K)]
            samp = samples.repeat_interleave(K)
            if ref is not None:
                s = rank.scores(imgs, ref, samp)
            else:                                                                           # a plain callable: per-sample slices
                rows = samp.tolist()
                _, s = rank(imgs, image[samp.to(image.device)], [encode_text[b] for b in rows], [decode_text[b] for b in rows])
                assert s.shape == (imgs.shape[0],)
            sel.add(s, cand, samp, imgs)
        return sel.best_img, sel.best_idx, sel.scores

    @property
    def device(self):
        return self.engine.device


class SDStochasticTextWrapper(_StochasticTextWrapperBase):
    """Stable Diffusion v1 (512 px, latent 64, CLIP context 768, posterior *sample*)."""


class SD2StochasticTextWrapper(_StochasticTextWrapperBase):
    """Stable Diffusion 2.x: ``parameterization='eps'`` is v2-1_512 ("base", 512 px, latent 64), ``'v'`` is v2-1_768 ("-v",
    768 px, latent 96, v-prediction), the ldm yaml key of the same name.  OpenCLIP-H context 1024 (OpenClipTextCondStage from the
    checkpoint's ``cond_stage_model.model.*`` keys), 64-channel heads, Linear transformer projections, posterior *sample*.
    Everything else -- precision, encode / forward, cycle, cycle_ensemble -- is SDStochasticTextWrapper's."""
    CONTEXT_DIM = 1024
    COND_PREFIX = 'cond_stage_model.model.'           # FrozenOpenCLIPEmbedder.model (open_clip CLIP without `visual`)
    COND_CLASS = OpenClipTextCondStage
    RESOLUTIONS = {'eps': 512, 'v': 768}

    def __init__(self, *args, parameterization='eps', resolution=None, latent_size=None, unet_config=None, **kwargs):
        if parameterization not in self.RESOLUTIONS:
            raise ValueError(f"parameterization must be 'eps' or 'v', got {parameterization!r}")
        self.parameterization = parameterization
        resolution = resolution or self.RESOLUTIONS[parameterization]
        super().__init__(*args, resolution=resolution, latent_size=latent_size or resolution // 8,
                         unet_config=unet_config or specs.sd2_unet_config(), **kwargs)
        if self.generator.unet.prediction != parameterization:      # a generator passed in is switched to this wrapper's yaml key
            self.generator.unet.set_prediction(parameterization)
        self.generator.parameterization = parameterization

    def _build_unet(self, ucfg):
        return UNet(self.engine, ucfg, 'openai').set_prediction(self.parameterization)


class LatentDiffStochasticTextWrapper(_StochasticTextWrapperBase):
    """LDM text2img-large (256 px, latent 32, BERT context 1280, posterior *mean*: latentdiff/.../ddpm.py:537-538)."""
    RESOLUTION = 256
    LATENT = 32
    CONTEXT_DIM = 1280
    SAMPLE_POSTERIOR = False
    CKPT_DIR = 'ckpts/ldm_models'
    COND_PREFIX = 'cond_stage_model.'                 # BERTEmbedder (encoders/modules.py:79-98)
    COND_CLASS = BertTextCondStage

    @classmethod
    def default_checkpoint(cls, source_model_type):
        """LDW:21-23: ``ckpts/ldm_models/<source_model_type>/model.ckpt``."""
        return os.path.join(cls.CKPT_DIR, str(source_model_type), 'model.ckpt')


class LatentDiffStochasticWrapper(torch.nn.Module):
    """Unconditional latent-diffusion models (ffhq256 -> celeba256; VQ-f4 first stage, U-Net without context), SURVEY 8f-4.

    ref model/gan_wrapper/latentdiff_stochastic_wrapper.py:185-316: ``encode(image, class_label=None) -> z [B, white_box_steps*C*h*w]``,
    ``forward(z, class_label=None) -> img in [0,1]``, optional eta = 1 refinement pass after the decode (convsample_ddim :57-79 ->
    DDIMSampler.refine, ddim.py:114-168, 339-393).  The class-conditional branch (enforce_class_input: ClassEmbedder cross-attention
    conditioning, cin256) is not built."""

    @staticmethod
    def default_checkpoint(source_model_type):
        """latentdiff_stochastic_wrapper.py:16: ``ckpts/ldm_models/ldm/<source_model_type>/model.ckpt``."""
        return os.path.join('ckpts', 'ldm_models', 'ldm', str(source_model_type), 'model.ckpt')

    def __init__(self, source_model_type, custom_steps, eta, white_box_steps, refine_steps=0, enforce_class_input=None,
                 unconditional_guidance_scale=None, *, engine=None, device=0, state_dict=None, unet_config=None, vae_config=None,
                 latent_size=64, resolution=256, generator=None, seed=1234, alphas_cumprod=None, scale_factor=1.0):
        super().__init__()
        if enforce_class_input:
            raise NotImplementedError('class-conditional latent diffusion (ClassEmbedder conditioning) is not built; unconditional models only')
        self.enforce_class_input = enforce_class_input
        self.unconditional_guidance_scale = unconditional_guidance_scale
        self.refine_steps = refine_steps
        self.eta, self.custom_steps, self.white_box_steps = eta, custom_steps, white_box_steps
        self.vanilla = False
        if generator is not None:
            self.generator, self.engine = generator, generator.engine
        else:
            self.engine = engine or Engine(device)
            ucfg, vcfg = unet_config or specs.ldm_uncond_unet_config(), vae_config or specs.vq_f4_config()
            unet, vae = UNet(self.engine, ucfg, 'openai'), VAE(self.engine, vcfg)
            if state_dict == 'synthetic':
                unet.load_state_dict(specs.synth_state_dict(specs.openai_unet_params(ucfg), seed))
                vae.load_state_dict(specs.synth_state_dict(specs.kl_vae_params(vcfg), seed + 1))
            else:
                sd = _load_sd(state_dict, self.default_checkpoint(source_model_type), None, seed)
                unet.load_state_dict(sd, prefix='model.diffusion_model.', strict=False)
                vae.load_state_dict(sd, prefix='first_stage_model.', strict=False)
            self.generator = _LatentGenerator(self.engine, unet, vae, None, ucfg['in_channels'], latent_size, scale_factor, False)
            # ffhq256 / celeba256 LDMs: linear_start 0.0015, linear_end 0.0195 (upstream config.yaml; pass alphas_cumprod to override)
            from .schedule import ldm_alphas_cumprod
            self.generator.alphas_cumprod = alphas_cumprod if alphas_cumprod is not None else ldm_alphas_cumprod(1000, 0.0015, 0.0195)
        self.resolution = resolution
        g = self.generator
        self.latent_dim = g.image_size ** 2 * g.channels * self.white_box_steps
        self._dummy = torch.nn.Parameter(torch.zeros(1, device=self.engine.device), requires_grad=False)

    def _sched(self):
        return DDIMSchedule(self.custom_steps, self.eta, 0, self.generator.alphas_cumprod)

    def generate(self, z, class_label):
        g = self.generator
        bsz = z.shape[0]
        eps_list = z.view(bsz, self.white_box_steps, g.channels, g.image_size, g.image_size)
        sched = self._sched()
        n_extra = sched.refine_steps - (eps_list.shape[1] - 1)
        extra = torch.stack([torch.randn(eps_list[:, 0].shape) for _ in range(n_extra)]) if n_extra > 0 else None      # ddim.py:640
        sample = g.unet.latent_decode(eps_list, None, None, 1.0, sched, extra)
        return self._refine_and_decode(sample)

    def _refine_and_decode(self, sample):
        g = self.generator
        if self.refine_steps > 0:                                     # refine_eta = 1 (latentdiff_stochastic_wrapper.py:68-77)
            noise = torch.stack([torch.randn(sample.shape) for _ in range(self.refine_steps + 1)])
            sample = g.unet.latent_refine(sample, None, None, 1.0, self.custom_steps, self.refine_steps, noise, g.alphas_cumprod)
        return g.decode_first_stage(sample)

    def encode(self, image, class_label=None):
        g = self.generator
        bsz = image.shape[0]
        x0 = g.encode_image(image, self.resolution)
        assert self.eta > 0
        sched = self._sched()
        n_rec = max(0, min(sched.refine_steps, self.white_box_steps - 1))
        noise = encode_noise(sched, n_rec, x0.shape)
        z = g.unet.latent_encode(x0, None, None, 1.0, sched, n_rec, noise).view(bsz, -1)
        assert z.shape[1] == self.latent_dim
        return z

    def cycle(self, image, target):
        """``target(self.encode(image))`` for a target wrapper with the same schedule (see lockstep_compatible), as one lock-step
        loop (cdx_latent_cycle_pair): the source chain runs under this wrapper's U-Net, the target chain under the target's, and
        the noise recovered at a step is consumed by the target chain at once, so ``z`` is never written.  Same random draws in
        the same order, same result bit for bit.  Then the target's own refine pass and first-stage decode."""
        g = self.generator
        x0 = g.encode_image(image, self.resolution)
        assert self.eta > 0
        sched = self._sched()
        n_rec = max(0, min(sched.refine_steps, self.white_box_steps - 1))
        assert n_rec + 1 == self.white_box_steps, 'white_box_steps - 1 > custom_steps (encode() would fail the latent_dim check)'
        noise = encode_noise(sched, n_rec, x0.shape)
        n_extra = sched.refine_steps - n_rec
        extra = torch.stack([torch.randn(x0.shape) for _ in range(n_extra)]) if n_extra > 0 else None      # ddim.py:640
        sample = g.unet.latent_cycle_pair(target.generator.unet, x0, sched, n_rec, noise, extra)
        return target.engine.shift_scale(target._refine_and_decode(sample), 1.0, 0.5)

    def forward(self, z, class_label=None):
        return self.engine.shift_scale(self.generate(z, class_label), 1.0, 0.5)

    @property
    def device(self):
        return self.engine.device


class DDPMDDIMWrapper(torch.nn.Module):
    """Pixel-space DPM-Encoder / decoder (improved-DDPM U-Net for AFHQ / FFHQ)."""

    def __init__(self, source_model_type, sample_type, custom_steps, es_steps, source_model_path=None, refine_steps=0,
                 refine_iterations=1, eta=None, t_0=None, enforce_class_input=None, *, engine=None, device=0, state_dict=None,
                 image_size=None, unet=None, seed=4321, dataset=None, var_type='fixedsmall', rng='cpu'):
        super().__init__()
        # DW:360-369: the model family follows config.data.dataset -- CelebA_HQ / LSUN checkpoints are Ho et al. DDPM U-Nets
        # (models/ddpm/diffusion.py), AFHQ / FFHQ ones improved-DDPM U-Nets.  `dataset` (or a source_model_type that names one) selects it.
        # rng='cpu': every draw comes from the torch CPU generator in the reference's order (reproduces the reference CPU path under a
        # seed); rng='cuda': drawn on the engine's device (the reference's own GPU runs do this; avoids es_steps x image of host randn +
        # H2D per batch -- 1.5 GB at 250 steps, batch 8, 256^2)
        assert rng in ('cpu', 'cuda')
        self.rng = rng
        name = (dataset or str(source_model_type)).lower()
        self.model_family = 'ddpm' if any(k in name for k in ('celeba', 'lsun', 'bedroom', 'church')) else 'iddpm'
        self.enforce_class_input = enforce_class_input
        self.custom_steps, self.refine_steps, self.refine_iterations = custom_steps, refine_steps, refine_iterations
        self.sample_type, self.eta = sample_type, eta
        self.t_0 = t_0 if t_0 is not None else 999
        self.es_steps = es_steps
        if self.sample_type == 'ddim':
            assert self.eta > 0
        elif self.sample_type == 'ddpm':
            assert self.eta is None
        else:
            raise ValueError()
        if image_size is None:
            digits = ''.join(ch for ch in str(source_model_type) if ch.isdigit())
            image_size = int(digits) if digits else 256
        self.learn_sigma = False
        if unet is not None:
            self.generator, self.engine = unet, unet.engine
        else:
            self.engine = engine or Engine(device)
            if self.model_family == 'ddpm':
                cfg = specs.ddpm_config(image_size)
                params = specs.ddpm_unet_params(cfg)
            else:
                cfg = specs.iddpm_config(image_size)
                params = specs.iddpm_unet_params(cfg)
            self.generator = UNet(self.engine, cfg, self.model_family)
            sd = _load_sd(state_dict if state_dict is not None else source_model_path, source_model_path or '', params, seed)
            self.generator.load_state_dict(sd)
        self.resolution = image_size
        self.channels = 3
        self.latent_dim = self.resolution ** 2 * self.channels * self.es_steps
        self.sched = PixelSchedule(sample_type, custom_steps, es_steps, eta, self.t_0, var_type=var_type)     # config.model.var_type, DW:362-367
        self._dummy = torch.nn.Parameter(torch.zeros(1, device=self.engine.device), requires_grad=False)

    def _randn(self, shape):
        return torch.randn(shape, device=self.engine.device) if self.rng == 'cuda' else torch.randn(shape)

    def generate(self, z, class_label):
        bsz = z.shape[0]
        eps_list = z.view(bsz, self.es_steps, self.channels, self.resolution, self.resolution)
        if self.enforce_class_input:
            assert class_label is not None
            raise NotImplementedError()
        shape = eps_list[:, 0].shape
        last = self._randn(shape).unsqueeze(0)       # denoising_step draws once more; the draw is multiplied by 0 (DU:115,131)
        x = self.generator.pixel_decode(eps_list, self.sched, last_noise=last)
        return self._refine(x, shape)

    def _refine(self, x, shape):
        bsz = shape[0]
        if self.refine_steps != 0:
            assert self.refine_steps < self.custom_steps
            ref = PixelSchedule(self.sample_type, self.custom_steps, self.es_steps, 1 if self.sample_type == 'ddim' else None, self.t_0)
            pairs = self.sched.pairs[-self.refine_steps:] if self.refine_steps <= len(self.sched.pairs) else self.sched.pairs
            coefs = [ref.step_coef(i, j, 1 if self.sample_type == 'ddim' else None) for i, j in pairs]
            t_loop = [float(i) for i, _ in pairs]
            at = PixelSchedule._extract(self.sched.cumprod, self.refine_steps - 1)               # DW:436-437
            for _ in range(self.refine_iterations):
                xt = self.engine.q_sample(x, self._randn(shape), at.sqrt().item(), (1 - at).sqrt().item())
                noises = torch.stack([self._randn(shape) for _ in pairs])
                x = self.generator.pixel_decode(xt.view(bsz, 1, *shape[1:]), ref, coefs=coefs, t_loop=t_loop, last_noise=noises)
        return x

    def encode(self, image, class_label=None):
        e = self.engine
        image = e.shift_scale(image, -0.5, 2.0)
        assert image.shape[2] == image.shape[3] == self.resolution
        if self.enforce_class_input:
            assert class_label is not None
            raise NotImplementedError()
        bsz = image.shape[0]
        n_rec = self.es_steps - 1
        if self.rng == 'cuda':
            noise = torch.randn((n_rec + 1,) + tuple(image.shape), device=e.device)
        else:
            noise = torch.stack([torch.randn(image.shape) for _ in range(n_rec + 1)])     # sample_xt, then one per sample_xt_next
        z = self.generator.pixel_encode(image, self.sched, noise).view(bsz, -1)
        assert z.shape[1] == self.latent_dim
        return z

    def forward(self, z, class_label=None):
        img = self.generate(z, class_label)
        return self.engine.shift_scale(img, 1.0, 0.5)

    def cycle(self, image, target):
        """``target(self.encode(image))`` for a target wrapper with the same schedule (see lockstep_compatible), as one lock-step
        loop (cdx_pixel_cycle_lockstep): per step the source U-Net call on the source chain and the target U-Net call on the target
        chain, then one fused kernel that recovers the step's noise and advances the target chain with it, so ``z`` is never
        written.  The loop walks the es_steps - 1 recovery steps in chunks of LOCKSTEP_CHUNK, so device memory holds one chunk of
        noise.  Then the target's own last step and refine pass, as target.generate does.

        rng='cpu': the same draws in the same order as the two calls (x_T, one per recovery step, then the target's ``last`` and
        refine draws), so the result is bit-identical.  They are drawn chunk by chunk into two pinned buffers used in turn, so the
        host draws chunk k+1 while the device runs chunk k.  rng='cuda': drawn on the device per chunk, which matches the two-phase
        path in distribution only (bit for bit when one chunk covers every step)."""
        e = self.engine
        x = e.shift_scale(image, -0.5, 2.0)
        assert x.shape[2] == x.shape[3] == self.resolution
        shape = tuple(x.shape)
        n_rec = self.es_steps - 1
        chunk = max(1, int(LOCKSTEP_CHUNK))
        state = e.empty(2, *shape)
        if self.rng == 'cuda':
            for i0, i1 in _chunk_ranges(n_rec, chunk):
                noise = torch.randn((i1 - i0 + (i0 == 0),) + shape, device=e.device)
                self.generator.pixel_cycle_lockstep(target.generator, x, self.sched, state, noise, i0, i1)
        else:
            bufs = [torch.empty((min(chunk, n_rec) + 1,) + shape, pin_memory=True) for _ in range(2 if n_rec > chunk else 1)]
            copied = [None] * len(bufs)
            for j, (i0, i1, host) in enumerate(lockstep_noise_chunks(shape, n_rec, chunk, bufs)):
                noise = torch.empty(host.shape, device=e.device)
                noise.copy_(host, non_blocking=True)
                copied[j % len(bufs)] = torch.cuda.Event()
                copied[j % len(bufs)].record()
                self.generator.pixel_cycle_lockstep(target.generator, x, self.sched, state, noise, i0, i1)
                nxt = copied[(j + 1) % len(bufs)]
                if nxt is not None:
                    nxt.synchronize()          # the next chunk is drawn into the buffer this upload read
        last = target._randn(shape).unsqueeze(0)      # target.generate's last step: t = 0 with the `last` draw (DU:115,131)
        y = target.generator.pixel_decode(state[1].unsqueeze(1), target.sched, coefs=target.sched.coef[n_rec:],
                                          t_loop=target.sched.t_loop[n_rec:], last_noise=last)
        return target.engine.shift_scale(target._refine(y, shape), 1.0, 0.5)

    @property
    def device(self):
        return self.engine.device


def _chunk_ranges(n_rec, chunk):
    """[i0, i1) ranges of the lock-step pixel loop: [0, n_rec) in pieces of `chunk` steps; one empty range when n_rec == 0
    (the call that only draws x_T)."""
    return [(i0, min(n_rec, i0 + chunk)) for i0 in range(0, max(n_rec, 1), chunk)]


def lockstep_noise_chunks(shape, n_rec, chunk, buffers=None):
    """The CPU draws of DDPMDDIMWrapper.encode (x_T, then one per recovery step; torch.randn(shape) each, in that order) in the
    chunks the lock-step loop consumes them: yields (i0, i1, noise) with noise [i1 - i0, *shape], preceded by the x_T draw when
    i0 == 0.  ``buffers``: host tensors of at least min(chunk, n_rec) + 1 draws, filled in turn (pinned buffers for asynchronous
    uploads); without them each chunk is a new tensor."""
    for j, (i0, i1) in enumerate(_chunk_ranges(n_rec, chunk)):
        k = i1 - i0 + (i0 == 0)
        noise = buffers[j % len(buffers)][:k] if buffers else torch.empty((k,) + tuple(shape))
        for d in range(k):
            noise[d].normal_()                 # what torch.randn(shape) draws
        yield i0, i1, noise


def lockstep_compatible(source, target):
    """Can UnsupervisedTranslation run source.cycle(image, target) instead of target(source.encode(image))?  Both wrappers of
    the same kind with a lock-step loop, no class input, and identical schedules (coefficient tables, timesteps, x_T scalars,
    number of recovered steps)."""
    if type(source) is not type(target) or not isinstance(source, (DDPMDDIMWrapper, LatentDiffStochasticWrapper)):
        return False
    if source.enforce_class_input or target.enforce_class_input:
        return False
    if isinstance(source, DDPMDDIMWrapper):
        return source.es_steps == target.es_steps and same_schedule(source.sched, target.sched)
    g, h = source.generator, target.generator
    return (source.white_box_steps == target.white_box_steps and (g.channels, g.image_size) == (h.channels, h.image_size)
            and same_schedule(source._sched(), target._sched()))


def get_gan_wrapper(args, target=False, **extra):
    """Same kwarg plumbing as the reference factory: every ``[gan]`` key but ``gan_type`` becomes a kwarg;
    ``target_*`` keys are renamed ``source_*`` for the target model.  ``extra`` carries engine/state_dict/... ."""
    items = list(args.items()) if isinstance(args, dict) else list(args)
    gan_type = args['gan_type'] if isinstance(args, dict) else args.gan_type
    kwargs = {}
    for kw, arg in items:
        if kw != 'gan_type':
            if (not kw.startswith('source_')) and (not kw.startswith('target_')):
                kwargs[kw] = arg
            else:
                if target and kw.startswith('target_'):
                    kwargs['source_' + kw[len('target_'):]] = arg
                elif (not target) and kw.startswith('source_'):
                    kwargs[kw] = arg
    kwargs.update(extra)
    if gan_type == "LatentDiffStochastic":
        return LatentDiffStochasticWrapper(**kwargs)
    elif gan_type == "DDPM_DDIM":
        return DDPMDDIMWrapper(**kwargs)
    elif gan_type == "LatentDiffStochasticText":
        return LatentDiffStochasticTextWrapper(**kwargs)
    elif gan_type == "SDStochasticText":
        return SDStochasticTextWrapper(**kwargs)
    elif gan_type == "SD2StochasticText":
        return SD2StochasticTextWrapper(**kwargs)
    else:
        raise ValueError()
