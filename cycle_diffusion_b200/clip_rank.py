"""Directional-CLIP ranking and the text-task metrics on the device (SURVEY.md 8f-3).

  DirectionalCLIP   ref model/energy/clean_clip.py:7-41   __call__(img, original_img, encode_text, decode_text) -> (clip_score, dclip_score)
  CLIP              ref model/energy/clean_clip.py:44-70  __call__(img, text) -> clip_score
  translate_text_metrics   ref evaluation/translate_text.py:65-89 (calculate_psnr / calculate_ssim, evaluation/utils.py:13-66)

The reference runs OpenAI CLIP ViT-B/32 (``clip.load``).  Both towers, the bicubic preprocessing, the score arithmetic and the metric
reductions run in libcdx; the BPE tokeniser stays on the host (``tokenizer``: list[str] -> LongTensor [B, 77], e.g. ``clip.tokenize``).
Weights: an OpenAI-clip ``state_dict`` (``visual.*``, ``transformer.*``, ``token_embedding`` ...) or the equivalent HF ``CLIPModel`` one.
An instance is a drop-in for the wrappers' ``ranker=``: candidates never leave the GPU.
"""
import torch

from . import specs
from .engine import ClipVision, TextEncoder


def openai_to_hf(sd):
    """OpenAI clip state_dict (clip/model.py) -> HF CLIPModel key names (fused in_proj split into q / k / v)."""
    out = {}

    def block(src, dst):
        w, b = sd[src + '.attn.in_proj_weight'], sd[src + '.attn.in_proj_bias']
        W = w.shape[1]
        for i, nm in enumerate(('q_proj', 'k_proj', 'v_proj')):
            out[f'{dst}.self_attn.{nm}.weight'] = w[i * W:(i + 1) * W]
            out[f'{dst}.self_attn.{nm}.bias'] = b[i * W:(i + 1) * W]
        out[f'{dst}.self_attn.out_proj.weight'] = sd[src + '.attn.out_proj.weight']
        out[f'{dst}.self_attn.out_proj.bias'] = sd[src + '.attn.out_proj.bias']
        for a, b_ in (('ln_1', 'layer_norm1'), ('ln_2', 'layer_norm2'), ('mlp.c_fc', 'mlp.fc1'), ('mlp.c_proj', 'mlp.fc2')):
            out[f'{dst}.{b_}.weight'] = sd[f'{src}.{a}.weight']
            out[f'{dst}.{b_}.bias'] = sd[f'{src}.{a}.bias']

    nv = len({k.split('.')[3] for k in sd if k.startswith('visual.transformer.resblocks.')})
    nt = len({k.split('.')[2] for k in sd if k.startswith('transformer.resblocks.')})
    for l in range(nv):
        block(f'visual.transformer.resblocks.{l}', f'vision_model.encoder.layers.{l}')
    for l in range(nt):
        block(f'transformer.resblocks.{l}', f'text_model.encoder.layers.{l}')
    out['vision_model.embeddings.class_embedding'] = sd['visual.class_embedding']
    out['vision_model.embeddings.patch_embedding.weight'] = sd['visual.conv1.weight']
    out['vision_model.embeddings.position_embedding.weight'] = sd['visual.positional_embedding']
    for a, b_ in (('visual.ln_pre', 'vision_model.pre_layrnorm'), ('visual.ln_post', 'vision_model.post_layernorm'),
                  ('ln_final', 'text_model.final_layer_norm')):
        out[b_ + '.weight'], out[b_ + '.bias'] = sd[a + '.weight'], sd[a + '.bias']
    out['visual_projection.weight'] = sd['visual.proj'].t().contiguous()           # x @ proj  ==  Linear(weight = proj^T)
    out['text_projection.weight'] = sd['text_projection'].t().contiguous()
    out['text_model.embeddings.token_embedding.weight'] = sd['token_embedding.weight']
    out['text_model.embeddings.position_embedding.weight'] = sd['positional_embedding']
    return out


class DirectionalCLIP:
    def __init__(self, engine, state_dict, tokenizer, vision_cfg=None, text_cfg=None):
        sd = openai_to_hf(state_dict) if 'visual.conv1.weight' in state_dict else state_dict
        self.engine, self.tokenizer = engine, tokenizer
        self.vcfg, self.tcfg = vision_cfg or specs.clip_b32_vision_config(), text_cfg or specs.clip_b32_text_config()
        self.vision = ClipVision(engine, self.vcfg)
        self.vision.load_state_dict({k: v for k, v in sd.items() if k.startswith('vision_model.') or k.startswith('visual_projection.')})
        self.text = TextEncoder(engine, self.tcfg)
        self.text.load_state_dict({k: v for k, v in sd.items() if k.startswith('text_model.') or k.startswith('text_projection.')})

    def encode_image(self, img):
        return self.vision(self.engine.clip_preprocess(img, self.vcfg['image_size']))

    def encode_text(self, texts):
        ids = self.tokenizer(list(texts))
        assert ids.dim() == 2 and ids.shape[0] == len(texts)
        return self.text.features(ids)

    @torch.no_grad()
    def __call__(self, img, original_img, encode_text, decode_text):
        assert len(decode_text) == img.shape[0]
        assert len(encode_text) == original_img.shape[0]
        return self.engine.dclip_scores(self.encode_image(img), self.encode_image(original_img), self.encode_text(encode_text),
                                        self.encode_text(decode_text))

    @torch.no_grad()
    def reference(self, original_img, encode_text, decode_text):
        """What every candidate of one forward is scored against, computed once: (original-image features, source-text features,
        target-text features), each [B, D]."""
        assert len(encode_text) == original_img.shape[0] == len(decode_text)
        return self.encode_image(original_img), self.encode_text(encode_text), self.encode_text(decode_text)

    @torch.no_grad()
    def scores(self, img, ref, sel=None):
        """D-CLIP scores [n] of a candidate batch img [n,3,R,R] against ``ref`` (from reference()); candidate c belongs to sample
        sel[c] (None: candidate b is sample b)."""
        orig_f, enc_f, dec_f = ref if sel is None else (f[sel] for f in ref)
        assert orig_f.shape[0] == img.shape[0]
        return self.engine.dclip_scores(self.encode_image(img), orig_f, enc_f, dec_f)[1]

    def rank(self, img_ensemble, original_img, encode_text, decode_text):
        """SDW:233-249: D-CLIP score of every candidate, per-sample argmax, gather -- all on the device."""
        ref = self.reference(original_img, encode_text, decode_text)
        scores = torch.stack([self.scores(img, ref) for img in img_ensemble], dim=1)                                    # [B, members]
        best = scores.argmax(dim=1)
        stack = torch.stack(list(img_ensemble), dim=1)                                                                  # [B, members, 3, R, R]
        return stack[torch.arange(stack.shape[0], device=stack.device), best], best, scores


class CLIP(DirectionalCLIP):
    @torch.no_grad()
    def __call__(self, img, text):
        assert len(text) == img.shape[0]
        f_img, f_txt = self.encode_image(img), self.encode_text(text)
        return self.engine.dclip_scores(f_img, f_img, f_txt, f_txt)[0]


def translate_text_metrics(engine, img, original_img):
    """Per pair: dict of tensors psnr / ssim / l2 [B] (evaluation/translate_text.py:76-89; inputs in [0,1], clamped inside)."""
    m = engine.image_metrics(img, original_img)
    return {'psnr': m[:, 0], 'ssim': m[:, 1], 'l2': m[:, 2]}
