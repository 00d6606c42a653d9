"""Parameter inventories (reference state_dict key -> shape) and synthetic ("random-init") weights.

The key names are the reference checkpoint's own (SURVEY.md Appendix C):
  * SD / LDM U-Net      ``model.diffusion_model.*``   built by UNetModel.__init__, ref ldm/modules/diffusionmodules/openaimodel.py:506-686
  * KL-f8 VAE           ``first_stage_model.*``       ref ldm/modules/diffusionmodules/model.py:368-533, ldm/models/autoencoder.py:302-303
  * i-DDPM U-Net        bare keys                     ref model/lib/ddpm_ddim/models/improved_ddpm/unet.py:476-626
The C++ graph executors (csrc/nets.cu) enumerate the same names through ``cdx_net_param_*``;
``tests/test_cabi.py`` cross-checks the two lists on the CPU (inventory-only nets need no GPU), and
``tests/golden/make_golden.py`` checks them against the reference modules with ``load_state_dict(strict=True)``.

There are no checkpoints in this environment, so benchmarks and tests use ``synth_state_dict``:
fan-in-scaled uniform weights for *every* tensor, including the ones the reference zero-initialises
(``zero_module``: openaimodel.py:229-231, 312, 685; attention.py:244) -- an all-zero tensor would make
every parity check vacuous (SURVEY.md section 4).
"""
import math
import torch


# ------------------------------------------------------------------ config defaults

def sd_unet_config(context_dim=768):
    """v1-inference.yaml:29-44 (SD v1-4); LDM text2img-large uses context_dim=1280 (txt2img-1p4B-eval.yaml:20-42)."""
    return dict(in_channels=4, out_channels=4, model_channels=320, attention_resolutions=(4, 2, 1),
                num_res_blocks=2, channel_mult=(1, 2, 4, 4), num_heads=8, context_dim=context_dim)


def sd2_unet_config():
    """v2-inference.yaml / v2-inference-v.yaml unet_config (SD 2.x base and -v): SD v1's topology with a fixed head WIDTH of 64
    (5 / 10 / 20 heads), the OpenCLIP-H context width 1024 and Linear proj_in / proj_out (use_linear_in_transformer)."""
    return dict(in_channels=4, out_channels=4, model_channels=320, attention_resolutions=(4, 2, 1),
                num_res_blocks=2, channel_mult=(1, 2, 4, 4), num_head_channels=64, context_dim=1024, use_linear_in_transformer=True)


def kl_f8_config():
    """v1-inference.yaml:51-65."""
    return dict(ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2, in_channels=3, out_ch=3, z_channels=4, embed_dim=4)


def iddpm_config(image_size=256):
    """AFHQ_DICT + create_model channel_mult table, script_util.py:5-73."""
    mult = {256: (1, 1, 2, 2, 4, 4), 128: (1, 1, 2, 3, 4), 64: (1, 2, 3, 4)}[image_size]
    return dict(image_size=image_size, in_channels=3, out_channels=6, model_channels=128, num_res_blocks=1,
                channel_mult=mult, attention_resolutions=(image_size // 16,), num_head_channels=64)


# ------------------------------------------------------------------ inventories

def _conv(out, name, cin, cout, k):
    out.append((name + '.weight', (cout, cin, k, k), 'w'))
    out.append((name + '.bias', (cout,), 'b'))


def _lin(out, name, cin, cout, bias=True):
    out.append((name + '.weight', (cout, cin), 'w'))
    if bias:
        out.append((name + '.bias', (cout,), 'b'))


def _norm(out, name, c):
    out.append((name + '.weight', (c,), 'nw'))
    out.append((name + '.bias', (c,), 'nb'))


def openai_unet_params(cfg, prefix=''):
    """Ordered (name, shape, kind) list of the SD/LDM UNetModel (spatial-transformer variant)."""
    mc, mult, nrb, ar = cfg['model_channels'], cfg['channel_mult'], cfg['num_res_blocks'], cfg['attention_resolutions']
    ctx, ted = cfg.get('context_dim', 0), 4 * cfg['model_channels']
    out = []

    def res(p, cin, cout):
        _norm(out, p + '.in_layers.0', cin)
        _conv(out, p + '.in_layers.2', cin, cout, 3)
        _lin(out, p + '.emb_layers.1', ted, cout)
        _norm(out, p + '.out_layers.0', cout)
        _conv(out, p + '.out_layers.3', cout, cout, 3)
        if cin != cout:
            _conv(out, p + '.skip_connection', cin, cout, 1)

    def st(p, c):
        if not ctx:                      # use_spatial_transformer=False: AttentionBlock (openaimodel.py:278-315), conv1d weights
            _norm(out, p + '.norm', c)
            out.append((p + '.qkv.weight', (3 * c, c, 1), 'w'))
            out.append((p + '.qkv.bias', (3 * c,), 'b'))
            out.append((p + '.proj_out.weight', (c, c, 1), 'w'))
            out.append((p + '.proj_out.bias', (c,), 'b'))
            return
        lin = cfg.get('use_linear_in_transformer', False)     # SD 2.x: Linear [C, C] projections instead of 1x1 convolutions
        _norm(out, p + '.norm', c)
        _lin(out, p + '.proj_in', c, c) if lin else _conv(out, p + '.proj_in', c, c, 1)
        t = p + '.transformer_blocks.0'
        for a, kd in (('attn1', c), ('attn2', ctx)):
            _lin(out, f'{t}.{a}.to_q', c, c, bias=False)
            _lin(out, f'{t}.{a}.to_k', kd, c, bias=False)
            _lin(out, f'{t}.{a}.to_v', kd, c, bias=False)
            _lin(out, f'{t}.{a}.to_out.0', c, c)
        _lin(out, t + '.ff.net.0.proj', c, 8 * c)
        _lin(out, t + '.ff.net.2', 4 * c, c)
        for n in ('norm1', 'norm2', 'norm3'):
            _norm(out, f'{t}.{n}', c)
        _lin(out, p + '.proj_out', c, c) if lin else _conv(out, p + '.proj_out', c, c, 1)

    P = prefix
    _lin(out, P + 'time_embed.0', mc, ted)
    _lin(out, P + 'time_embed.2', ted, ted)
    _conv(out, P + 'input_blocks.0.0', cfg['in_channels'], mc, 3)
    chans = [mc]
    ch, ds, bi = mc, 1, 1
    for level, m in enumerate(mult):
        for _ in range(nrb):
            res(f'{P}input_blocks.{bi}.0', ch, m * mc)
            ch = m * mc
            if ds in ar:
                st(f'{P}input_blocks.{bi}.1', ch)
            chans.append(ch)
            bi += 1
        if level != len(mult) - 1:
            _conv(out, f'{P}input_blocks.{bi}.0.op', ch, ch, 3)
            chans.append(ch)
            bi += 1
            ds *= 2
    res(P + 'middle_block.0', ch, ch)
    st(P + 'middle_block.1', ch)
    res(P + 'middle_block.2', ch, ch)
    bo = 0
    for level, m in list(enumerate(mult))[::-1]:
        for i in range(nrb + 1):
            ich = chans.pop()
            res(f'{P}output_blocks.{bo}.0', ch + ich, mc * m)
            ch = mc * m
            li = 1
            if ds in ar:
                st(f'{P}output_blocks.{bo}.{li}', ch)
                li += 1
            if level and i == nrb:
                _conv(out, f'{P}output_blocks.{bo}.{li}.conv', ch, ch, 3)
                ds //= 2
            bo += 1
    _norm(out, P + 'out.0', ch)
    _conv(out, P + 'out.2', mc, cfg['out_channels'], 3)
    return out


def iddpm_unet_params(cfg, prefix=''):
    """Ordered (name, shape, kind) list of the improved-DDPM UNetModel (scale-shift norm, res-block up/down)."""
    mc, mult, nrb, ar = cfg['model_channels'], cfg['channel_mult'], cfg['num_res_blocks'], cfg['attention_resolutions']
    ted = 4 * mc
    out = []

    def res(p, cin, cout):
        _norm(out, p + '.in_layers.0', cin)
        _conv(out, p + '.in_layers.2', cin, cout, 3)
        _lin(out, p + '.emb_layers.1', ted, 2 * cout)
        _norm(out, p + '.out_layers.0', cout)
        _conv(out, p + '.out_layers.3', cout, cout, 3)
        if cin != cout:
            _conv(out, p + '.skip_connection', cin, cout, 1)

    def attn(p, c):
        _norm(out, p + '.norm', c)
        out.append((p + '.qkv.weight', (3 * c, c, 1), 'w'))
        out.append((p + '.qkv.bias', (3 * c,), 'b'))
        out.append((p + '.proj_out.weight', (c, c, 1), 'w'))
        out.append((p + '.proj_out.bias', (c,), 'b'))

    P = prefix
    _lin(out, P + 'time_embed.0', mc, ted)
    _lin(out, P + 'time_embed.2', ted, ted)
    ch = int(mult[0] * mc)
    _conv(out, P + 'input_blocks.0.0', cfg['in_channels'], ch, 3)
    chans = [ch]
    ds, bi = 1, 1
    for level, m in enumerate(mult):
        for _ in range(nrb):
            res(f'{P}input_blocks.{bi}.0', ch, int(m * mc))
            ch = int(m * mc)
            if ds in ar:
                attn(f'{P}input_blocks.{bi}.1', ch)
            chans.append(ch)
            bi += 1
        if level != len(mult) - 1:
            res(f'{P}input_blocks.{bi}.0', ch, ch)
            chans.append(ch)
            bi += 1
            ds *= 2
    res(P + 'middle_block.0', ch, ch)
    attn(P + 'middle_block.1', ch)
    res(P + 'middle_block.2', ch, ch)
    bo = 0
    for level, m in list(enumerate(mult))[::-1]:
        for i in range(nrb + 1):
            ich = chans.pop()
            res(f'{P}output_blocks.{bo}.0', ch + ich, int(mc * m))
            ch = int(mc * m)
            li = 1
            if ds in ar:
                attn(f'{P}output_blocks.{bo}.{li}', ch)
                li += 1
            if level and i == nrb:
                res(f'{P}output_blocks.{bo}.{li}', ch, ch)
                ds //= 2
            bo += 1
    _norm(out, P + 'out.0', ch)
    _conv(out, P + 'out.2', int(mult[0] * mc), cfg['out_channels'], 3)
    return out


def kl_vae_params(cfg, prefix=''):
    """Ordered (name, shape, kind) list of AutoencoderKL's encoder, decoder, quant_conv, post_quant_conv."""
    ch, mult, nrb = cfg['ch'], cfg['ch_mult'], cfg['num_res_blocks']
    zc, ed = cfg['z_channels'], cfg['embed_dim']
    out = []

    def res(p, cin, cout):
        _norm(out, p + '.norm1', cin)
        _conv(out, p + '.conv1', cin, cout, 3)
        _norm(out, p + '.norm2', cout)
        _conv(out, p + '.conv2', cout, cout, 3)
        if cin != cout:
            _conv(out, p + '.nin_shortcut', cin, cout, 1)

    def attn(p, c):
        _norm(out, p + '.norm', c)
        for n in ('q', 'k', 'v', 'proj_out'):
            _conv(out, f'{p}.{n}', c, c, 1)

    E = prefix + 'encoder.'
    _conv(out, E + 'conv_in', cfg['in_channels'], ch, 3)
    in_mult = (1,) + tuple(mult)
    block_in = ch
    for lvl in range(len(mult)):
        block_in, block_out = ch * in_mult[lvl], ch * mult[lvl]
        for b in range(nrb):
            res(f'{E}down.{lvl}.block.{b}', block_in, block_out)
            block_in = block_out
        if lvl != len(mult) - 1:
            _conv(out, f'{E}down.{lvl}.downsample.conv', block_in, block_in, 3)
    res(E + 'mid.block_1', block_in, block_in)
    attn(E + 'mid.attn_1', block_in)
    res(E + 'mid.block_2', block_in, block_in)
    _norm(out, E + 'norm_out', block_in)
    vq = bool(cfg.get('vq'))
    _conv(out, E + 'conv_out', block_in, (1 if vq else 2) * zc, 3)

    D = prefix + 'decoder.'
    block_in = ch * mult[-1]
    _conv(out, D + 'conv_in', zc, block_in, 3)
    res(D + 'mid.block_1', block_in, block_in)
    attn(D + 'mid.attn_1', block_in)
    res(D + 'mid.block_2', block_in, block_in)
    for lvl in reversed(range(len(mult))):
        block_out = ch * mult[lvl]
        for b in range(nrb + 1):
            res(f'{D}up.{lvl}.block.{b}', block_in, block_out)
            block_in = block_out
        if lvl != 0:
            _conv(out, f'{D}up.{lvl}.upsample.conv', block_in, block_in, 3)
    _norm(out, D + 'norm_out', block_in)
    _conv(out, D + 'conv_out', block_in, cfg['out_ch'], 3)
    if vq:                                                   # VQModel: quantize.embedding (taming VectorQuantizer2), single-width quant_conv
        out.append((prefix + 'quantize.embedding.weight', (cfg['n_embed'], ed), 'w'))
    _conv(out, prefix + 'quant_conv', (1 if vq else 2) * zc, (1 if vq else 2) * ed, 1)
    _conv(out, prefix + 'post_quant_conv', ed, zc, 1)
    return out


# ------------------------------------------------------------------ synthetic weights

def clip_text_config(vocab_size=49408, width=768, layers=12, heads=12, max_len=77, mlp_width=3072):
    """CLIP ViT-L/14 text tower ("openai/clip-vit-large-patch14", the SD v1 conditioning model; encoders/modules.py:140-146)."""
    return dict(vocab_size=vocab_size, width=width, layers=layers, heads=heads, max_len=max_len, mlp_width=mlp_width)


def clip_text_params(cfg, prefix=''):
    """Ordered (name, shape, kind) list in HF CLIPTextModel.state_dict() order (without the position_ids buffer)."""
    W, M = cfg['width'], cfg['mlp_width']
    T = prefix + 'text_model.'
    out = [(T + 'embeddings.token_embedding.weight', (cfg['vocab_size'], W), 'w'),
           (T + 'embeddings.position_embedding.weight', (cfg['max_len'], W), 'w')]
    for l in range(cfg['layers']):
        p = f'{T}encoder.layers.{l}'
        for nm in ('k_proj', 'v_proj', 'q_proj', 'out_proj'):
            out += [(f'{p}.self_attn.{nm}.weight', (W, W), 'w'), (f'{p}.self_attn.{nm}.bias', (W,), 'b')]
        out += [(f'{p}.layer_norm1.weight', (W,), 'nw'), (f'{p}.layer_norm1.bias', (W,), 'nb')]
        out += [(f'{p}.mlp.fc1.weight', (M, W), 'w'), (f'{p}.mlp.fc1.bias', (M,), 'b')]
        out += [(f'{p}.mlp.fc2.weight', (W, M), 'w'), (f'{p}.mlp.fc2.bias', (W,), 'b')]
        out += [(f'{p}.layer_norm2.weight', (W,), 'nw'), (f'{p}.layer_norm2.bias', (W,), 'nb')]
    out += [(T + 'final_layer_norm.weight', (W,), 'nw'), (T + 'final_layer_norm.bias', (W,), 'nb')]
    return out


def openclip_h14_text_config(layers=23, total_layers=24, vocab_size=49408, width=1024, heads=16, max_len=77, mlp_width=4096):
    """SD 2.x conditioning model: FrozenOpenCLIPEmbedder(arch="ViT-H-14", layer="penultimate") -- 24 pre-LN blocks of width 1024,
    16 heads, exact-erf GELU; `layers` = 23 blocks run (the penultimate output), then ln_final.  `total_layers` is what the
    checkpoint holds (block 23 is loaded by nobody)."""
    return dict(kind='openclip', vocab_size=vocab_size, width=width, layers=layers, total_layers=total_layers, heads=heads,
                max_len=max_len, mlp_width=mlp_width)


def openclip_text_params(cfg, prefix=''):
    """Ordered (name, shape, kind) list of the OpenCLIP text transformer as the SD 2 checkpoint stores it under
    ``cond_stage_model.model.`` (open_clip CLIP without `visual`): all `total_layers` blocks, text_projection and logit_scale."""
    W, M, V = cfg['width'], cfg['mlp_width'], cfg['vocab_size']
    P = prefix
    out = [(P + 'positional_embedding', (cfg['max_len'], W), 'w'), (P + 'text_projection', (W, W), 'w'),
           (P + 'logit_scale', (), 'b'), (P + 'token_embedding.weight', (V, W), 'w')]
    for l in range(cfg.get('total_layers', cfg['layers'])):
        p = f'{P}transformer.resblocks.{l}'
        out += [(p + '.ln_1.weight', (W,), 'nw'), (p + '.ln_1.bias', (W,), 'nb'),
                (p + '.attn.in_proj_weight', (3 * W, W), 'w'), (p + '.attn.in_proj_bias', (3 * W,), 'b'),
                (p + '.attn.out_proj.weight', (W, W), 'w'), (p + '.attn.out_proj.bias', (W,), 'b'),
                (p + '.ln_2.weight', (W,), 'nw'), (p + '.ln_2.bias', (W,), 'nb'),
                (p + '.mlp.c_fc.weight', (M, W), 'w'), (p + '.mlp.c_fc.bias', (M,), 'b'),
                (p + '.mlp.c_proj.weight', (W, M), 'w'), (p + '.mlp.c_proj.bias', (W,), 'b')]
    out += [(P + 'ln_final.weight', (W,), 'nw'), (P + 'ln_final.bias', (W,), 'nb')]
    return out


def openclip_to_hf(sd, layers, prefix=''):
    """OpenCLIP text-transformer keys (under `prefix`) -> the HF CLIPTextModel keys of the engine's OpenCLIP tower, blocks
    0 .. layers-1 only: in_proj split into q / k / v (stacked [q; k; v] along dim 0), positional_embedding ->
    position_embedding.weight, ln_1 / ln_2 / mlp.c_fc / mlp.c_proj / ln_final -> layer_norm1 / layer_norm2 / mlp.fc1 / mlp.fc2 /
    final_layer_norm.  text_projection, logit_scale and the blocks past `layers` are not used for conditioning."""
    T = 'text_model.'
    out = {T + 'embeddings.token_embedding.weight': sd[prefix + 'token_embedding.weight'],
           T + 'embeddings.position_embedding.weight': sd[prefix + 'positional_embedding']}
    for l in range(layers):
        o, h = f'{prefix}transformer.resblocks.{l}.', f'{T}encoder.layers.{l}.'
        q, k, v = sd[o + 'attn.in_proj_weight'].chunk(3, dim=0)
        qb, kb, vb = sd[o + 'attn.in_proj_bias'].chunk(3, dim=0)
        for nm, w, b in (('q_proj', q, qb), ('k_proj', k, kb), ('v_proj', v, vb)):
            out[h + f'self_attn.{nm}.weight'], out[h + f'self_attn.{nm}.bias'] = w, b
        for src, dst in (('attn.out_proj', 'self_attn.out_proj'), ('ln_1', 'layer_norm1'), ('ln_2', 'layer_norm2'),
                         ('mlp.c_fc', 'mlp.fc1'), ('mlp.c_proj', 'mlp.fc2')):
            out[h + dst + '.weight'], out[h + dst + '.bias'] = sd[o + src + '.weight'], sd[o + src + '.bias']
    out[T + 'final_layer_norm.weight'], out[T + 'final_layer_norm.bias'] = sd[prefix + 'ln_final.weight'], sd[prefix + 'ln_final.bias']
    return out


def hf_to_openclip(sd, layers, prefix=''):
    """The inverse of openclip_to_hf for blocks 0 .. layers-1 (no text_projection / logit_scale)."""
    T = 'text_model.'
    out = {prefix + 'token_embedding.weight': sd[T + 'embeddings.token_embedding.weight'],
           prefix + 'positional_embedding': sd[T + 'embeddings.position_embedding.weight']}
    for l in range(layers):
        o, h = f'{prefix}transformer.resblocks.{l}.', f'{T}encoder.layers.{l}.'
        out[o + 'attn.in_proj_weight'] = torch.cat([sd[h + f'self_attn.{n}.weight'] for n in ('q_proj', 'k_proj', 'v_proj')])
        out[o + 'attn.in_proj_bias'] = torch.cat([sd[h + f'self_attn.{n}.bias'] for n in ('q_proj', 'k_proj', 'v_proj')])
        for src, dst in (('attn.out_proj', 'self_attn.out_proj'), ('ln_1', 'layer_norm1'), ('ln_2', 'layer_norm2'),
                         ('mlp.c_fc', 'mlp.fc1'), ('mlp.c_proj', 'mlp.fc2')):
            out[o + src + '.weight'], out[o + src + '.bias'] = sd[h + dst + '.weight'], sd[h + dst + '.bias']
    out[prefix + 'ln_final.weight'], out[prefix + 'ln_final.bias'] = sd[T + 'final_layer_norm.weight'], sd[T + 'final_layer_norm.bias']
    return out


def bert_text_config(vocab_size=30522, width=1280, layers=32, heads=8, dim_head=64, max_len=77, mlp_width=None):
    """LDM text2img-large conditioning model: BERTEmbedder(n_embed=1280, n_layer=32) (txt2img-1p4B-eval.yaml:66-71;
    encoders/modules.py:79-98): x_transformer Encoder defaults heads=8, dim_head=64, ff mult 4."""
    return dict(kind='xtransformer', vocab_size=vocab_size, width=width, layers=layers, heads=heads, dim_head=dim_head, max_len=max_len,
                mlp_width=mlp_width or 4 * width)


def bert_text_params(cfg, prefix=''):
    """Ordered (name, shape, kind) list of TransformerWrapper(Encoder(dim, depth)).state_dict() without the unused to_logits."""
    W, M, inner = cfg['width'], cfg['mlp_width'], cfg['heads'] * cfg['dim_head']
    T = prefix + 'transformer.'
    out = [(T + 'token_emb.weight', (cfg['vocab_size'], W), 'w'), (T + 'pos_emb.emb.weight', (cfg['max_len'], W), 'w')]
    for l in range(cfg['layers']):
        pa, pf = f'{T}attn_layers.layers.{2 * l}', f'{T}attn_layers.layers.{2 * l + 1}'
        out += [(pa + '.0.weight', (W,), 'nw'), (pa + '.0.bias', (W,), 'nb')]
        out += [(pa + '.1.to_q.weight', (inner, W), 'w'), (pa + '.1.to_k.weight', (inner, W), 'w'), (pa + '.1.to_v.weight', (inner, W), 'w')]
        out += [(pa + '.1.to_out.weight', (W, inner), 'w'), (pa + '.1.to_out.bias', (W,), 'b')]
        out += [(pf + '.0.weight', (W,), 'nw'), (pf + '.0.bias', (W,), 'nb')]
        out += [(pf + '.1.net.0.0.weight', (M, W), 'w'), (pf + '.1.net.0.0.bias', (M,), 'b')]
        out += [(pf + '.1.net.2.weight', (W, M), 'w'), (pf + '.1.net.2.bias', (W,), 'b')]
    out += [(T + 'norm.weight', (W,), 'nw'), (T + 'norm.bias', (W,), 'nb')]
    return out


def synth_state_dict(params, seed, gain=1.0):
    """Deterministic CPU fp32 weights for an inventory; identical on every machine with the same torch build.

    conv/linear weights and all biases ~ U(-b, b) with b = gain / sqrt(fan_in); norm weights 1 + 0.1 N(0,1);
    norm biases 0.1 N(0,1).  One generator, tensors drawn in inventory order.
    """
    g = torch.Generator(device='cpu')
    g.manual_seed(seed)
    sd = {}
    fan_in = 1
    for name, shape, kind in params:
        if kind == 'nw':
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif kind == 'nb':
            t = 0.1 * torch.randn(shape, generator=g)
        else:
            if kind == 'w':
                fan_in = int(math.prod(shape[1:]))
            b = gain / math.sqrt(fan_in)
            t = (torch.rand(shape, generator=g) * 2.0 - 1.0) * b
        sd[name] = t.contiguous()
    return sd


def clip_b32_vision_config():
    """OpenAI CLIP ViT-B/32 image tower (clip/model.py build_model; what clean_clip.py:10 loads)."""
    return dict(kind='clip_vision', width=768, layers=12, heads=12, mlp_width=3072, patch=32, image_size=224, proj_dim=512)


def clip_b32_text_config():
    return dict(kind='clip', vocab_size=49408, width=512, layers=12, heads=8, max_len=77, mlp_width=2048, proj_dim=512)


def clip_vision_params(cfg):
    """(name, shape, kind) in the engine's inventory order for the CLIP image tower (csrc/nets.cu make_text, CDX_CLIP_VISION)."""
    W, P, n = cfg['width'], cfg['patch'], (cfg['image_size'] // cfg['patch']) ** 2
    V = 'vision_model.'
    out = [(V + 'embeddings.class_embedding', (W,), 'b'), (V + 'embeddings.patch_embedding.weight', (W, 3, P, P), 'w'),
           (V + 'embeddings.position_embedding.weight', (n + 1, W), 'w'), (V + 'pre_layrnorm.weight', (W,), 'nw'), (V + 'pre_layrnorm.bias', (W,), 'nb')]
    for l in range(cfg['layers']):
        p = f'{V}encoder.layers.{l}'
        for nm in ('k_proj', 'v_proj', 'q_proj', 'out_proj'):
            out += [(f'{p}.self_attn.{nm}.weight', (W, W), 'w'), (f'{p}.self_attn.{nm}.bias', (W,), 'b')]
        out += [(f'{p}.layer_norm1.weight', (W,), 'nw'), (f'{p}.layer_norm1.bias', (W,), 'nb'),
                (f'{p}.mlp.fc1.weight', (cfg['mlp_width'], W), 'w'), (f'{p}.mlp.fc1.bias', (cfg['mlp_width'],), 'b'),
                (f'{p}.mlp.fc2.weight', (W, cfg['mlp_width']), 'w'), (f'{p}.mlp.fc2.bias', (W,), 'b'),
                (f'{p}.layer_norm2.weight', (W,), 'nw'), (f'{p}.layer_norm2.bias', (W,), 'nb')]
    out += [(V + 'post_layernorm.weight', (W,), 'nw'), (V + 'post_layernorm.bias', (W,), 'nb'), ('visual_projection.weight', (cfg['proj_dim'], W), 'w')]
    return out


def ldm_uncond_unet_config():
    """Unconditional LDM U-Net of the ffhq256 / celeba256 zoo entries the reference's LatentDiffStochastic configs load
    (models/ldm/ffhq256/config.yaml upstream; the yaml is not in the tree -- values from the CompVis release): no context,
    AttentionBlock with 32 channels per head."""
    return dict(in_channels=3, out_channels=3, model_channels=224, attention_resolutions=(8, 4, 2), num_res_blocks=2,
                channel_mult=(1, 2, 3, 4), num_head_channels=32, context_dim=0)


def vq_f4_config():
    """VQModelInterface first stage of the same models: embed_dim 3, 8192 codes, ch 128, ch_mult (1,2,4)."""
    return dict(ch=128, ch_mult=(1, 2, 4), num_res_blocks=2, in_channels=3, out_ch=3, z_channels=3, embed_dim=3, vq=True, n_embed=8192)


def ddpm_config(image_size=256, ch=128, ch_mult=(1, 1, 2, 2, 4, 4), attn_resolutions=(16,), num_res_blocks=2):
    """Ho et al. DDPM U-Net as the CelebA-HQ / LSUN checkpoints are built (ddpm/diffusion.py:192-297; the DDIM repo's celeba_hq.yml /
    bedroom.yml: ch 128, ch_mult (1,1,2,2,4,4), 2 res blocks, attention at 16x16, resamp_with_conv).  ``attention_resolutions`` holds
    the downsample FACTORS at which attention runs (image_size / resolution), like the other U-Net configs here."""
    return dict(image_size=image_size, in_channels=3, out_channels=3, model_channels=ch, num_res_blocks=num_res_blocks, channel_mult=tuple(ch_mult),
                attention_resolutions=tuple(image_size // r for r in attn_resolutions))


def ddpm_unet_params(cfg):
    """(name, shape, kind) of ddpm/diffusion.py DDPM in the engine's inventory order (csrc/nets.cu build_ddpm_inventory)."""
    ch, mult, nrb, ar = cfg['model_channels'], cfg['channel_mult'], cfg['num_res_blocks'], cfg['attention_resolutions']
    ted = 4 * ch
    out = []

    def res(p, cin, cout):
        _norm(out, p + '.norm1', cin)
        _conv(out, p + '.conv1', cin, cout, 3)
        _lin(out, p + '.temb_proj', ted, cout)
        _norm(out, p + '.norm2', cout)
        _conv(out, p + '.conv2', cout, cout, 3)
        if cin != cout:
            _conv(out, p + '.nin_shortcut', cin, cout, 1)

    def attn(p, c):
        _norm(out, p + '.norm', c)
        for nm in ('q', 'k', 'v', 'proj_out'):
            _conv(out, f'{p}.{nm}', c, c, 1)

    _lin(out, 'temb.dense.0', ch, ted)
    _lin(out, 'temb.dense.1', ted, ted)
    _conv(out, 'conv_in', cfg['in_channels'], ch, 3)
    in_mult = (1,) + tuple(mult)
    ds, block_in = 1, ch
    for lvl in range(len(mult)):
        block_in, block_out = ch * in_mult[lvl], ch * mult[lvl]
        for b in range(nrb):
            res(f'down.{lvl}.block.{b}', block_in, block_out)
            block_in = block_out
        if ds in ar:
            for b in range(nrb):
                attn(f'down.{lvl}.attn.{b}', block_out)
        if lvl != len(mult) - 1:
            _conv(out, f'down.{lvl}.downsample.conv', block_in, block_in, 3)
            ds *= 2
    res('mid.block_1', block_in, block_in)
    attn('mid.attn_1', block_in)
    res('mid.block_2', block_in, block_in)
    for lvl in reversed(range(len(mult))):
        block_out, skip_in = ch * mult[lvl], ch * mult[lvl]
        for b in range(nrb + 1):
            if b == nrb:
                skip_in = ch * in_mult[lvl]
            res(f'up.{lvl}.block.{b}', block_in + skip_in, block_out)
            block_in = block_out
        if ds in ar:
            for b in range(nrb + 1):
                attn(f'up.{lvl}.attn.{b}', block_out)
        if lvl != 0:
            _conv(out, f'up.{lvl}.upsample.conv', block_in, block_in, 3)
            ds //= 2
    _norm(out, 'norm_out', block_in)
    _conv(out, 'conv_out', block_in, cfg['out_channels'], 3)
    return out
