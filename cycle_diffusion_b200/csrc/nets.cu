// nets.cu -- graph executors for the three network families on the path.
//
//   SD v1 / LDM text2img U-Net   UNetModel.forward      ref ldm/modules/diffusionmodules/openaimodel.py:710-742 (built :506-686)
//                                ResBlock._forward      ref openaimodel.py:255-275
//                                SpatialTransformer     ref ldm/modules/attention.py:196-261
//   improved-DDPM pixel U-Net    UNetModel.forward      ref model/lib/ddpm_ddim/models/improved_ddpm/unet.py:639-668 (built :476-626)
//                                ResBlock / AttentionBlock / QKVAttentionLegacy   ref unet.py:241-261, 304-310, 342-363
//   KL-f8 VAE                    Encoder / Decoder      ref ldm/modules/diffusionmodules/model.py:434-459, 535-568
//                                ResnetBlock / AttnBlock / Downsample / Upsample   ref model.py:42-202
//
// Design decisions (DESIGN.md has the full rationale):
//   * activations are NHWC, so a [B,H,W,C] feature map *is* the [B*HW, C] token matrix: the reference's
//     'b c h w -> b (h w) c' rearranges disappear and every conv / Linear is one implicit-GEMM family;
//   * skip-connection concatenation (th.cat, OAI:736) is never materialised: GroupNorm and the 1x1 skip conv read
//     two sources;
//   * nearest-2x upsampling is folded into the following conv's gather; bias, timestep-embedding add and the
//     residual add are GEMM epilogues; all 22 ResBlock emb projections run as ONE GEMM per U-Net call;
//   * q/k/v (self) and k/v (cross) projections are single fused GEMMs over weights stored adjacently in the blob.
#include <math.h>
#include <string.h>

#include <cstdlib>

#include "nets.cuh"

namespace cdx {

// ================================================================================================ inventory
namespace {

struct Inv {
  Net& n;
  explicit Inv(Net& net) : n(net) {}
  void add(const std::string& name, std::initializer_list<int64_t> dims, int segment = 0, bool conv3 = false) {
    Param p;
    p.name = name;
    p.rank = (int)dims.size();
    size_t ne = 1;
    int i = 0;
    for (int64_t d : dims) { p.dims[i++] = d; ne *= (size_t)d; }
    p.numel = ne;
    p.segment = segment;
    p.conv3 = conv3;
    n.index[name] = (int)n.params.size();
    n.params.push_back(p);
  }
  void conv(const std::string& name, int cin, int cout, int k) {
    add(name + ".weight", {cout, cin, k, k}, 0, k == 3);
    if (k == 3 && cin < 32) n.params.back().cin_pad = 32;      // conv_in layers (3 / 4 channels): run on the tensor-core path too
    add(name + ".bias", {cout});
  }
  void lin(const std::string& name, int cin, int cout, bool bias = true, int seg = 0) {
    add(name + ".weight", {cout, cin}, seg ? 1 : 0);
    if (bias) add(name + ".bias", {cout}, seg ? 2 : 0);
  }
  void norm(const std::string& name, int c) {
    add(name + ".weight", {c});
    add(name + ".bias", {c});
  }
};

bool contains(const int* arr, int n, int v) {
  for (int i = 0; i < n; ++i)
    if (arr[i] == v) return true;
  return false;
}

std::string S(const std::string& a, int i) { return a + std::to_string(i); }

void build_unet_inventory(Net& n) {
  const cdx_unet_config& c = n.ucfg;
  const bool oai = c.kind == CDX_UNET_OPENAI;
  Inv v(n);
  const int mc = c.model_channels, ted = 4 * mc;
  n.ted = ted;
  int emb_rows = 0;
  auto res = [&](const std::string& p, int cin, int cout) {
    v.norm(p + ".in_layers.0", cin);
    v.conv(p + ".in_layers.2", cin, cout, 3);
    const int erows = oai ? cout : 2 * cout;
    v.lin(p + ".emb_layers.1", ted, erows, true, 1);
    n.emb_off[p] = emb_rows;
    emb_rows += erows;
    v.norm(p + ".out_layers.0", cout);
    v.conv(p + ".out_layers.3", cout, cout, 3);
    if (cin != cout) v.conv(p + ".skip_connection", cin, cout, 1);
  };
  auto st = [&](const std::string& p, int ch) {
    v.norm(p + ".norm", ch);
    v.conv(p + ".proj_in", ch, ch, 1);
    const std::string t = p + ".transformer_blocks.0";
    for (int a = 1; a <= 2; ++a) {
      const std::string ap = t + ".attn" + std::to_string(a);
      const int kd = (a == 1) ? ch : c.context_dim;
      v.lin(ap + ".to_q", ch, ch, false);
      v.lin(ap + ".to_k", kd, ch, false);
      v.lin(ap + ".to_v", kd, ch, false);
      v.lin(ap + ".to_out.0", ch, ch);
    }
    v.lin(t + ".ff.net.0.proj", ch, 8 * ch);
    if ((4 * ch) % 64 == 0) {   // value / gate rows interleaved in blocks of 32: each epilogue thread's 64 columns then hold 32 values and their gates
      n.params[n.index.at(t + ".ff.net.0.proj.weight")].geglu = true;
      n.params[n.index.at(t + ".ff.net.0.proj.bias")].geglu = true;
    }
    v.lin(t + ".ff.net.2", 4 * ch, ch);
    v.norm(t + ".norm1", ch);
    v.norm(t + ".norm2", ch);
    v.norm(t + ".norm3", ch);
    v.conv(p + ".proj_out", ch, ch, 1);
  };
  auto attn = [&](const std::string& p, int ch) {   // i-DDPM AttentionBlock
    v.norm(p + ".norm", ch);
    v.add(p + ".qkv.weight", {3 * ch, ch, 1});
    v.add(p + ".qkv.bias", {3 * ch});
    v.add(p + ".proj_out.weight", {ch, ch, 1});
    v.add(p + ".proj_out.bias", {ch});
  };
  auto attention_layer = [&](const std::string& p, int ch) { (oai && c.context_dim > 0) ? st(p, ch) : attn(p, ch); };

  v.lin("time_embed.0", mc, ted);
  v.lin("time_embed.2", ted, ted);
  int ch = c.channel_mult[0] * mc;
  if (oai) ch = mc;
  v.conv("input_blocks.0.0", c.in_channels, ch, 3);
  std::vector<int> chans{ch};
  int ds = 1, bi = 1;
  for (int level = 0; level < c.n_mult; ++level) {
    const int m = c.channel_mult[level];
    for (int r = 0; r < c.num_res_blocks; ++r) {
      const std::string bp = S("input_blocks.", bi);
      res(bp + ".0", ch, m * mc);
      ch = m * mc;
      if (contains(c.attention_ds, c.n_attn, ds)) attention_layer(bp + ".1", ch);
      chans.push_back(ch);
      ++bi;
    }
    if (level != c.n_mult - 1) {
      const std::string bp = S("input_blocks.", bi);
      if (oai) v.conv(bp + ".0.op", ch, ch, 3);
      else res(bp + ".0", ch, ch);
      chans.push_back(ch);
      ++bi;
      ds *= 2;
    }
  }
  res("middle_block.0", ch, ch);
  attention_layer("middle_block.1", ch);
  res("middle_block.2", ch, ch);
  int bo = 0;
  for (int level = c.n_mult - 1; level >= 0; --level) {
    const int m = c.channel_mult[level];
    for (int i = 0; i <= c.num_res_blocks; ++i) {
      const int ich = chans.back();
      chans.pop_back();
      const std::string bp = S("output_blocks.", bo);
      res(bp + ".0", ch + ich, mc * m);
      ch = mc * m;
      int li = 1;
      if (contains(c.attention_ds, c.n_attn, ds)) { attention_layer(bp + "." + std::to_string(li), ch); ++li; }
      if (level && i == c.num_res_blocks) {
        if (oai) v.conv(bp + "." + std::to_string(li) + ".conv", ch, ch, 3);
        else res(bp + "." + std::to_string(li), ch, ch);
        ds /= 2;
      }
      ++bo;
    }
  }
  v.norm("out.0", ch);
  v.conv("out.2", oai ? mc : c.channel_mult[0] * mc, c.out_channels, 3);
  n.emb_rows = emb_rows;
}

// Ho et al. DDPM (ddpm/diffusion.py:192-297): temb.dense, conv_in, down.{l}.block / attn / downsample, mid, up.{l}.block / attn /
// upsample (num_res_blocks + 1 blocks per level, skip widths as built at :262-271), norm_out, conv_out
void build_ddpm_inventory(Net& n) {
  const cdx_unet_config& c = n.ucfg;
  Inv v(n);
  const int ch = c.model_channels, ted = 4 * ch, L = c.n_mult;
  n.ted = ted;
  int emb_rows = 0;
  auto res = [&](const std::string& p, int cin, int cout) {
    v.norm(p + ".norm1", cin);
    v.conv(p + ".conv1", cin, cout, 3);
    v.lin(p + ".temb_proj", ted, cout, true, 1);
    n.emb_off[p] = emb_rows;
    emb_rows += cout;
    v.norm(p + ".norm2", cout);
    v.conv(p + ".conv2", cout, cout, 3);
    if (cin != cout) v.conv(p + ".nin_shortcut", cin, cout, 1);
  };
  auto attn = [&](const std::string& p, int cch) {
    v.norm(p + ".norm", cch);
    for (const char* nm : {"q", "k", "v", "proj_out"}) v.conv(p + "." + nm, cch, cch, 1);
  };
  v.lin("temb.dense.0", ch, ted);
  v.lin("temb.dense.1", ted, ted);
  v.conv("conv_in", c.in_channels, ch, 3);
  int ds = 1, block_in = ch;
  for (int lvl = 0; lvl < L; ++lvl) {
    block_in = ch * (lvl == 0 ? 1 : c.channel_mult[lvl - 1]);
    const int block_out = ch * c.channel_mult[lvl];
    const std::string D = "down." + std::to_string(lvl);
    for (int b = 0; b < c.num_res_blocks; ++b) {
      res(D + ".block." + std::to_string(b), block_in, block_out);
      block_in = block_out;
    }
    // (ModuleList order inside a level: all blocks, then all attns, then the downsample -- names carry the indices)
    if (contains(c.attention_ds, c.n_attn, ds))
      for (int b = 0; b < c.num_res_blocks; ++b) attn(D + ".attn." + std::to_string(b), block_out);
    if (lvl != L - 1) { v.conv(D + ".downsample.conv", block_in, block_in, 3); ds *= 2; }
  }
  res("mid.block_1", block_in, block_in);
  attn("mid.attn_1", block_in);
  res("mid.block_2", block_in, block_in);
  // decoder levels are built top-down (reversed) but registered with insert(0): state_dict order is up.0 first; inventory order is free
  std::vector<std::pair<int, int>> geom((size_t)L);     // per level: (block_in at entry, ds)
  for (int lvl = L - 1; lvl >= 0; --lvl) {
    const int block_out = ch * c.channel_mult[lvl];
    const std::string U = "up." + std::to_string(lvl);
    int skip_in = block_out;
    for (int b = 0; b <= c.num_res_blocks; ++b) {
      if (b == c.num_res_blocks) skip_in = ch * (lvl == 0 ? 1 : c.channel_mult[lvl - 1]);
      res(U + ".block." + std::to_string(b), block_in + skip_in, block_out);
      block_in = block_out;
    }
    if (contains(c.attention_ds, c.n_attn, ds))
      for (int b = 0; b <= c.num_res_blocks; ++b) attn(U + ".attn." + std::to_string(b), block_out);
    if (lvl != 0) { v.conv(U + ".upsample.conv", block_in, block_in, 3); ds /= 2; }
  }
  v.norm("norm_out", block_in);
  v.conv("conv_out", block_in, c.out_channels, 3);
  n.emb_rows = emb_rows;
}

void build_vae_inventory(Net& n) {
  const cdx_vae_config& c = n.vcfg;
  Inv v(n);
  auto res = [&](const std::string& p, int cin, int cout) {
    v.norm(p + ".norm1", cin);
    v.conv(p + ".conv1", cin, cout, 3);
    v.norm(p + ".norm2", cout);
    v.conv(p + ".conv2", cout, cout, 3);
    if (cin != cout) v.conv(p + ".nin_shortcut", cin, cout, 1);
  };
  auto attn = [&](const std::string& p, int ch) {
    v.norm(p + ".norm", ch);
    v.conv(p + ".q", ch, ch, 1);
    v.conv(p + ".k", ch, ch, 1);
    v.conv(p + ".v", ch, ch, 1);
    v.conv(p + ".proj_out", ch, ch, 1);
  };
  const int ch = c.ch, L = c.n_mult;
  const std::string E = "encoder.", D = "decoder.";
  v.conv(E + "conv_in", c.in_channels, ch, 3);
  int block_in = ch;
  for (int lvl = 0; lvl < L; ++lvl) {
    block_in = ch * (lvl == 0 ? 1 : c.ch_mult[lvl - 1]);
    const int block_out = ch * c.ch_mult[lvl];
    for (int b = 0; b < c.num_res_blocks; ++b) {
      res(E + "down." + std::to_string(lvl) + ".block." + std::to_string(b), block_in, block_out);
      block_in = block_out;
    }
    if (lvl != L - 1) v.conv(E + "down." + std::to_string(lvl) + ".downsample.conv", block_in, block_in, 3);
  }
  res(E + "mid.block_1", block_in, block_in);
  attn(E + "mid.attn_1", block_in);
  res(E + "mid.block_2", block_in, block_in);
  v.norm(E + "norm_out", block_in);
  v.conv(E + "conv_out", block_in, (c.vq ? 1 : 2) * c.z_channels, 3);

  block_in = ch * c.ch_mult[L - 1];
  v.conv(D + "conv_in", c.z_channels, block_in, 3);
  res(D + "mid.block_1", block_in, block_in);
  attn(D + "mid.attn_1", block_in);
  res(D + "mid.block_2", block_in, block_in);
  for (int lvl = L - 1; lvl >= 0; --lvl) {
    const int block_out = ch * c.ch_mult[lvl];
    for (int b = 0; b <= c.num_res_blocks; ++b) {
      res(D + "up." + std::to_string(lvl) + ".block." + std::to_string(b), block_in, block_out);
      block_in = block_out;
    }
    if (lvl != 0) v.conv(D + "up." + std::to_string(lvl) + ".upsample.conv", block_in, block_in, 3);
  }
  v.norm(D + "norm_out", block_in);
  v.conv(D + "conv_out", block_in, c.out_ch, 3);
  if (c.vq) v.add("quantize.embedding.weight", {c.n_embed, c.embed_dim});
  v.conv("quant_conv", (c.vq ? 1 : 2) * c.z_channels, (c.vq ? 1 : 2) * c.embed_dim, 1);
  v.conv("post_quant_conv", c.embed_dim, c.z_channels, 1);
}

void assign_offsets(Net& n) {
  size_t off = 0;
  auto align = [&](size_t a) { off = (off + a - 1) / a * a; };
  // general segment: inventory order, 16-byte aligned starts (adjacent q/k/v weights stay contiguous)
  for (Param& p : n.params)
    if (p.segment == 0) { align(8); p.off = off; off += p.store(); }     // 8: the fp16 planes (2 B / element) must be 16-byte aligned for TMA
  align(64);
  n.emb_w_off = off;
  for (Param& p : n.params)
    if (p.segment == 1) { p.off = off; off += p.numel; }
  align(64);
  n.emb_b_off = off;
  for (Param& p : n.params)
    if (p.segment == 2) { p.off = off; off += p.numel; }
  align(64);
  n.blob_floats = off;
}

}  // namespace

const Param& Net::param(const std::string& name) const {
  auto it = index.find(name);
  if (it == index.end()) throw Error(CDX_E_INVALID, "unknown parameter '" + name + "'");
  return params[it->second];
}

Net* make_unet(Engine* e, const cdx_unet_config& cfg) {
  CDX_CHECK(cfg.kind == CDX_UNET_OPENAI || cfg.kind == CDX_UNET_IDDPM || cfg.kind == CDX_UNET_DDPM, "unet: bad kind %d", cfg.kind);
  CDX_CHECK(cfg.n_mult >= 1 && cfg.n_mult <= 8 && cfg.n_attn >= 0 && cfg.n_attn <= 8, "unet: bad level counts");
  CDX_CHECK(cfg.model_channels % 32 == 0, "unet: model_channels must be a multiple of 32 (GroupNorm32)");
  if (cfg.kind == CDX_UNET_OPENAI && cfg.context_dim > 0) {
    // SD v1 fixes the head count (num_heads), SD 2.x the head width (num_head_channels = 64, OAI:542-549): heads = C / width per level
    CDX_CHECK(cfg.num_heads > 0 || cfg.num_head_channels > 0, "unet: num_heads / num_head_channels");
    if (cfg.num_head_channels > 0)
      for (int l = 0; l < cfg.n_mult; ++l)
        CDX_CHECK((cfg.channel_mult[l] * cfg.model_channels) % cfg.num_head_channels == 0, "unet: %d channels are not whole heads of %d",
                  cfg.channel_mult[l] * cfg.model_channels, cfg.num_head_channels);
  }
  else if (cfg.kind != CDX_UNET_DDPM) CDX_CHECK(cfg.num_head_channels > 0 || cfg.num_heads > 0, "unet: num_head_channels / num_heads");
  Net* n = new Net();
  n->eng = e;
  n->kind = cfg.kind == CDX_UNET_OPENAI ? NET_UNET_OPENAI : cfg.kind == CDX_UNET_IDDPM ? NET_UNET_IDDPM : NET_UNET_DDPM;
  n->ucfg = cfg;
  if (cfg.kind == CDX_UNET_DDPM) build_ddpm_inventory(*n);
  else build_unet_inventory(*n);
  assign_offsets(*n);
  // default sinusoid frequencies (util.py:161-163); the host normally overrides them with torch's own values
  const int half = cfg.model_channels / 2;
  n->freqs_host.resize(half);
  const float sc = (float)(-log(10000.0));
  for (int i = 0; i < half; ++i) n->freqs_host[i] = expf(sc * (float)i / (float)half);
  return n;
}

Net* make_vae(Engine* e, const cdx_vae_config& cfg) {
  CDX_CHECK(cfg.n_mult >= 1 && cfg.n_mult <= 8, "vae: bad level count");
  CDX_CHECK(cfg.ch % 32 == 0, "vae: ch must be a multiple of 32");
  CDX_CHECK(!cfg.vq || cfg.n_embed > 0, "vae: vq needs n_embed");
  Net* n = new Net();
  n->eng = e;
  n->kind = NET_VAE;
  n->vcfg = cfg;
  build_vae_inventory(*n);
  assign_offsets(*n);
  return n;
}

// HF CLIPTextModel state_dict order (transformers modeling_clip.py: CLIPTextEmbeddings, CLIPEncoderLayer {self_attn k,v,q,out;
// layer_norm1; mlp fc1, fc2; layer_norm2}, final_layer_norm)
Net* make_text(Engine* e, const cdx_text_config& cfg) {
  CDX_CHECK(cfg.width > 0 && cfg.layers > 0 && cfg.heads > 0 && cfg.mlp_width > 0, "text: bad config");
  if (cfg.kind != CDX_CLIP_VISION) CDX_CHECK(cfg.vocab_size > 0 && cfg.max_len > 0, "text: bad config");
  CDX_CHECK(cfg.width % cfg.heads == 0 && cfg.width % 4 == 0 && cfg.mlp_width % 4 == 0, "text: width %d / heads %d", cfg.width, cfg.heads);
  Net* n = new Net();
  n->eng = e;
  n->kind = NET_CLIP_TEXT;
  n->tcfg = cfg;
  Inv v(*n);
  if (cfg.kind == CDX_TEXT_XTRANSFORMER) {
    // x_transformer TransformerWrapper(Encoder(dim, depth)) state_dict order (x_transformer.py:548-596, 370-480, 215-266, 194-208)
    CDX_CHECK(cfg.dim_head > 0 && (cfg.heads * cfg.dim_head) % 4 == 0, "text: dim_head %d", cfg.dim_head);
    const int inner = cfg.heads * cfg.dim_head;
    const std::string T = "transformer.";
    v.add(T + "token_emb.weight", {cfg.vocab_size, cfg.width});
    v.add(T + "pos_emb.emb.weight", {cfg.max_len, cfg.width});
    for (int l = 0; l < cfg.layers; ++l) {
      const std::string pa = T + "attn_layers.layers." + std::to_string(2 * l), pf = T + "attn_layers.layers." + std::to_string(2 * l + 1);
      v.norm(pa + ".0", cfg.width);
      v.lin(pa + ".1.to_q", cfg.width, inner, false);
      v.lin(pa + ".1.to_k", cfg.width, inner, false);
      v.lin(pa + ".1.to_v", cfg.width, inner, false);
      v.lin(pa + ".1.to_out", inner, cfg.width);
      v.norm(pf + ".0", cfg.width);
      v.lin(pf + ".1.net.0.0", cfg.width, cfg.mlp_width);
      v.lin(pf + ".1.net.2", cfg.mlp_width, cfg.width);
    }
    v.norm(T + "norm", cfg.width);
    assign_offsets(*n);
    return n;
  }
  if (cfg.kind == CDX_CLIP_VISION) {
    // HF CLIPVisionModel(+projection) state_dict order (modeling_clip.py: CLIPVisionEmbeddings {class_embedding, patch_embedding,
    // position_embedding}, pre_layrnorm [sic], encoder layers as the text tower, post_layernorm) == OpenAI clip VisionTransformer
    // (clip/model.py: conv1, class_embedding, positional_embedding, ln_pre, transformer, ln_post, proj)
    CDX_CHECK(cfg.patch > 0 && cfg.image_size % cfg.patch == 0 && cfg.proj_dim > 0 && (3 * cfg.patch * cfg.patch) % 4 == 0, "vision: patch %d size %d", cfg.patch, cfg.image_size);
    const int np = cfg.image_size / cfg.patch;
    const std::string V = "vision_model.";
    v.add(V + "embeddings.class_embedding", {cfg.width});
    v.add(V + "embeddings.patch_embedding.weight", {cfg.width, 3, cfg.patch, cfg.patch});
    v.add(V + "embeddings.position_embedding.weight", {np * np + 1, cfg.width});
    v.norm(V + "pre_layrnorm", cfg.width);
    for (int l = 0; l < cfg.layers; ++l) {
      const std::string p = V + "encoder.layers." + std::to_string(l);
      for (const char* nm : {"k_proj", "v_proj", "q_proj", "out_proj"}) v.lin(p + ".self_attn." + nm, cfg.width, cfg.width);
      v.norm(p + ".layer_norm1", cfg.width);
      v.lin(p + ".mlp.fc1", cfg.width, cfg.mlp_width);
      v.lin(p + ".mlp.fc2", cfg.mlp_width, cfg.width);
      v.norm(p + ".layer_norm2", cfg.width);
    }
    v.norm(V + "post_layernorm", cfg.width);
    v.lin("visual_projection", cfg.width, cfg.proj_dim, false);
    assign_offsets(*n);
    return n;
  }
  const std::string T = "text_model.";
  v.add(T + "embeddings.token_embedding.weight", {cfg.vocab_size, cfg.width});
  v.add(T + "embeddings.position_embedding.weight", {cfg.max_len, cfg.width});
  for (int l = 0; l < cfg.layers; ++l) {
    const std::string p = T + "encoder.layers." + std::to_string(l);
    for (const char* nm : {"k_proj", "v_proj", "q_proj", "out_proj"}) v.lin(p + ".self_attn." + nm, cfg.width, cfg.width);
    v.norm(p + ".layer_norm1", cfg.width);
    v.lin(p + ".mlp.fc1", cfg.width, cfg.mlp_width);
    v.lin(p + ".mlp.fc2", cfg.mlp_width, cfg.width);
    v.norm(p + ".layer_norm2", cfg.width);
  }
  v.norm(T + "final_layer_norm", cfg.width);
  if (cfg.proj_dim > 0) v.lin("text_projection", cfg.width, cfg.proj_dim, false);       // CLIPModel.text_projection (clip/model.py text_projection^T)
  assign_offsets(*n);
  return n;
}

void destroy_net(Net* n) {
  if (!n) return;
  if (n->blob) cudaFree(n->blob);
  if (n->blob_hi) cudaFree(n->blob_hi);
  if (n->blob_lo) cudaFree(n->blob_lo);
  if (n->blob_h_hi) cudaFree(n->blob_h_hi);
  if (n->blob_h_lo) cudaFree(n->blob_h_lo);
  if (n->freqs_dev) cudaFree(n->freqs_dev);
  if (n->ctxkv.buf) cudaFree(n->ctxkv.buf);
  if (n->ctxkv.amax) cudaFree(n->ctxkv.amax);
  delete n;
}

void net_ensure_blob(Net& n) {
  if (n.blob) return;
  CDX_CUDA(cudaSetDevice(n.eng->device));
  CDX_CUDA(cudaMalloc(&n.blob, n.blob_floats * sizeof(float)));
  CDX_CUDA(cudaMemset(n.blob, 0, n.blob_floats * sizeof(float)));
}

void net_load_param(Net& n, const char* name, const float* data, bool on_device, const int64_t* dims, int rank) {
  auto it = n.index.find(name);
  CDX_CHECK(it != n.index.end(), "load_param: unknown parameter '%s'", name);
  Param& p = n.params[it->second];
  CDX_CHECK(rank == p.rank, "load_param %s: rank %d != %d", name, rank, p.rank);
  for (int i = 0; i < rank; ++i) CDX_CHECK(dims[i] == p.dims[i], "load_param %s: dim %d is %lld, expected %lld", name, i, (long long)dims[i], (long long)p.dims[i]);
  net_ensure_blob(n);
  Engine& e = *n.eng;
  float* dst = n.blob + p.off;
  const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  if (p.conv3) {
    float* tmp = nullptr;
    CDX_CUDA(cudaMalloc(&tmp, p.numel * sizeof(float)));
    CDX_CUDA(cudaMemcpy(tmp, data, p.numel * sizeof(float), kind));
    repack_conv3x3(e, tmp, dst, (int)p.dims[0], (int)p.dims[1], 0, p.cin_pad);
    CDX_CUDA(cudaDeviceSynchronize());
    CDX_CUDA(cudaFree(tmp));
  } else if (p.geglu) {
    float* tmp = nullptr;
    CDX_CUDA(cudaMalloc(&tmp, p.numel * sizeof(float)));
    CDX_CUDA(cudaMemcpy(tmp, data, p.numel * sizeof(float), kind));
    interleave_geglu_rows(e, tmp, dst, (int)p.dims[0], p.rank == 2 ? (int)p.dims[1] : 1, 0);
    CDX_CUDA(cudaDeviceSynchronize());
    CDX_CUDA(cudaFree(tmp));
  } else {
    CDX_CUDA(cudaMemcpy(dst, data, p.numel * sizeof(float), kind));
  }
  p.loaded = true;
  n.finalized = false;
  n.planes_valid = false;
  n.ctxkv.valid = false;
}

void net_finalize(Net& n) {
  for (const Param& p : n.params) CDX_CHECK(p.loaded, "finalize: parameter '%s' was never loaded", p.name.c_str());
  if (n.kind != NET_VAE && !n.freqs_host.empty()) {
    if (!n.freqs_dev) CDX_CUDA(cudaMalloc(&n.freqs_dev, n.freqs_host.size() * sizeof(float)));
    CDX_CUDA(cudaMemcpy(n.freqs_dev, n.freqs_host.data(), n.freqs_host.size() * sizeof(float), cudaMemcpyHostToDevice));
  }
  if (!n.planes_valid) {
    // TF32 hi / lo planes of every weight for the TF32-plane kernel (3x the weight memory: 10.3 GB for SD v1-4 of the H100's 80 GB)
    if (!n.blob_hi) CDX_CUDA(cudaMalloc(&n.blob_hi, n.blob_floats * sizeof(float)));
    if (!n.blob_lo) CDX_CUDA(cudaMalloc(&n.blob_lo, n.blob_floats * sizeof(float)));
    split_planes(*n.eng, n.blob, n.blob_hi, n.blob_lo, n.blob_floats, 0);
    // fp16-split planes: one power-of-two scale per network, from the largest GEMM weight (+2 bytes x 2 per parameter)
    {
      float* slot = nullptr;
      CDX_CUDA(cudaMalloc(&slot, sizeof(float)));
      CDX_CUDA(cudaMemset(slot, 0, sizeof(float)));
      for (const Param& p : n.params)
        if (p.rank >= 2 && (p.store() % 4) == 0 && (p.off % 4) == 0) amax_rows(*n.eng, n.blob + p.off, 1, (int)std::min<size_t>(p.store(), (size_t)1 << 30), (long long)p.store(), slot, 0);
      float wmax = 0.f;
      CDX_CUDA(cudaMemcpy(&wmax, slot, sizeof(float), cudaMemcpyDeviceToHost));
      CDX_CUDA(cudaFree(slot));
      n.w_exp = h16_exp_host(wmax);
      if (!n.blob_h_hi) CDX_CUDA(cudaMalloc(&n.blob_h_hi, n.blob_floats * 2));
      if (!n.blob_h_lo) CDX_CUDA(cudaMalloc(&n.blob_h_lo, n.blob_floats * 2));
      split_planes_h16(*n.eng, n.blob, n.blob_h_hi, n.blob_h_lo, n.blob_floats, n.w_exp, 0);
    }
    CDX_CUDA(cudaDeviceSynchronize());
    n.planes_valid = true;
  }
  n.finalized = true;
}

// ================================================================================================ executors
void track_outputs(Engine& e, Tensor& t, GemmArgs& g, bool stats) {
  t.amax = e.amax_slot();
  g.c_amax = t.amax;
  if (stats && (t.C % 4) == 0) {          // (few-channel outputs -- a 3-channel VQ latent -- are never GroupNorm inputs)
    t.stats = e.stat_alloc((size_t)t.B * t.C * 2);
    g.c_stats = t.stats;
    g.rows_per_batch = t.H * t.W;
  }
}

namespace {

struct Exec {
  Net& n;
  Engine& e;
  cudaStream_t s;
  Exec(Net& net, cudaStream_t st) : n(net), e(*net.eng), s(st) {}

  Tensor alloc(int B, int H, int W, int C) { return alloc_tensor(e, B, H, W, C); }

  // weights living in the blob have pre-split TF32 planes at the same offset
  void run(GemmArgs& g) {
    if (n.planes_valid && g.Bw >= n.blob && g.Bw < n.blob + n.blob_floats) {
      const size_t off = (size_t)(g.Bw - n.blob);
      g.Bw_hi = n.blob_hi + off;
      g.Bw_lo = n.blob_lo + off;
      g.Bw_h_hi = (const char*)n.blob_h_hi + 2 * off;
      g.Bw_h_lo = (const char*)n.blob_h_lo + 2 * off;
      g.b_exp = n.w_exp;
    }
    gemm(e, g, s);
  }

  void track(Tensor& t, GemmArgs& g, bool stats) { track_outputs(e, t, g, stats); }

  // y = conv3x3(x) + bias (+ rowvec per sample) (+ residual); up: nearest-2x folded into the gather
  // out_nchw (optional): store y there in NCHW layout; into (optional): preallocated NHWC output, its range and statistics tracked
  Tensor conv3(const Tensor& x0, const std::string& name, int stride = 1, int pad = 1, int up = 1, const float* rowvec = nullptr,
               int ld_rowvec = 0, const float* residual = nullptr, float* out_nchw = nullptr, Tensor* into = nullptr) {
    const Param& w = n.param(name + ".weight");
    const int Cout = (int)w.dims[0];
    CDX_CHECK((int)w.dims[1] == x0.C, "conv %s: input has %d channels, weight expects %d", name.c_str(), x0.C, (int)w.dims[1]);
    Tensor x = x0;
    if (w.cin_pad && x0.C != w.cin_pad) {          // few-channel network inputs: zero-pad to the stored Cin (one small pass)
      x = alloc(x0.B, x0.H, x0.W, w.cin_pad);
      pad_channels(e, x0.p, x.p, (size_t)x0.rows(), x0.C, w.cin_pad, s);
      x.amax = x0.amax;                            // zero padding does not change the range
    }
    const int Cin = x.C;
    if (up == 2 && e.mma_mode == 1 && (Cin % 32) == 0 && !out_nchw) {
      // tensor-core path: the TMA box gather cannot express the >>1 source index, so materialise the nearest-2x upsample
      // (one extra write+read of the activation, <2% of the conv's time) and run the plain tensor-core conv on it
      Tensor xu = alloc(x.B, x.H * 2, x.W * 2, x.C);
      upsample2(e, x.p, xu.p, x.B, x.H, x.W, x.C, s);
      xu.amax = x.amax;
      return conv3(xu, name, stride, pad, 1, rowvec, ld_rowvec, residual, out_nchw, into);
    }
    const int Hl = x.H * up, Wl = x.W * up;
    int Ho, Wo;
    if (stride == 1) { Ho = Hl; Wo = Wl; }
    else { Ho = Hl / 2; Wo = Wl / 2; }
    Tensor y;
    if (out_nchw) { y.p = out_nchw; y.B = x.B; y.H = Ho; y.W = Wo; y.C = Cout; }
    else if (into) y = *into;
    else y = alloc(x.B, Ho, Wo, Cout);
    GemmArgs g;
    g.mode = 1;
    g.M = x.B * Ho * Wo; g.N = Cout; g.K = 9 * Cin;
    g.A = x.p; g.lda = x.C; g.C1 = x.C;
    g.Hin = x.H; g.Win = x.W; g.Hout = Ho; g.Wout = Wo; g.stride = stride; g.pad = pad; g.up = up;
    g.Bw = n.blob + w.off; g.ldb = 9 * Cin;
    g.Cout = y.p; g.ldc = Cout;
    g.bias = n.P(name + ".bias");
    g.rowvec = rowvec; g.ld_rowvec = ld_rowvec; g.rows_per_batch = Ho * Wo;
    g.residual = residual; g.ldr = Cout;
    if (out_nchw) { g.out_nchw = 1; g.rows_per_img = Ho * Wo; }
    else track(y, g, true);
    g.a_amax = x.amax;
    run(g);
    if (into) *into = y;
    return y;
  }

  // y[M,N] = x[M,K] (optionally [x | x2]) @ W[N,K]^T (+bias) (+residual)
  void linear_into(const float* x, int lda, int C1, const float* x2, int lda2, int C2, int M, const float* W, int N, const float* bias,
                   const float* residual, int ldr, float* y, int ldc, float* y_lo = nullptr, const float* a_amax = nullptr,
                   const float* a2_amax = nullptr, float* c_amax = nullptr, double* c_stats = nullptr, int rows_per_img = 0) {
    GemmArgs g;
    g.mode = 0;
    g.a_amax = a_amax; g.a2_amax = a2_amax; g.c_amax = c_amax; g.c_stats = c_stats;
    if (rows_per_img > 0) g.rows_per_batch = rows_per_img;
    g.Cout_lo = y_lo;            // if set: y / y_lo receive the TF32 hi / lo planes of the result
    g.M = M; g.N = N; g.K = C1 + C2;
    g.A = x; g.lda = lda; g.C1 = C1;
    g.A2 = x2; g.lda2 = lda2; g.C2 = C2;
    g.Bw = W; g.ldb = C1 + C2;
    g.Cout = y; g.ldc = ldc;
    g.bias = bias;
    g.residual = residual; g.ldr = ldr;
    run(g);
  }
  // single-source convenience: named weight [N,K(,1,1)], optional named bias
  // track: the result's range is recorded (it is the A operand of a later GEMM); stats: also its GroupNorm sums
  Tensor linear(const Tensor& x, const std::string& name, bool bias, const float* residual = nullptr, bool track_amax = false, bool stats = false) {
    const Param& w = n.param(name + ".weight");
    const int N = (int)w.dims[0], K = (int)w.dims[1];
    CDX_CHECK(K == x.C, "linear %s: input width %d, weight expects %d", name.c_str(), x.C, K);
    Tensor y = alloc(x.B, x.H, x.W, N);
    if (track_amax || stats) y.amax = e.amax_slot();
    if (stats) y.stats = e.stat_alloc((size_t)y.B * N * 2);
    linear_into(x.p, x.C, x.C, nullptr, 0, 0, x.rows(), n.blob + w.off, N, bias ? n.P(name + ".bias") : nullptr, residual, N, y.p, N, nullptr, x.amax,
                nullptr, y.amax, y.stats, x.H * x.W);
    return y;
  }

  // src_img (optional device [B]): image b of the result is image src_img[b]'s norm (groupnorm)
  Tensor gn(const Tensor& x, const Tensor* x2, const std::string& name, float eps, bool act, const float* scale = nullptr,
            const float* shift = nullptr, int ld_ss = 0, const int* src_img = nullptr) {
    const int C = x.C + (x2 ? x2->C : 0);
    Tensor y = alloc(x.B, x.H, x.W, C);
    y.amax = e.amax_slot();
    groupnorm(e, x.p, x.C, x2 ? x2->p : nullptr, x2 ? x2->C : 0, n.P(name + ".weight"), n.P(name + ".bias"), eps, act, scale, shift, ld_ss,
              y.p, x.B, x.H * x.W, s, x.stats, x2 ? x2->stats : nullptr, y.amax, nullptr, src_img);
    return y;
  }
  Tensor ln(const Tensor& x, const std::string& name) {
    Tensor y = alloc(x.B, x.H, x.W, x.C);
    y.amax = e.amax_slot();
    layernorm(e, x.p, n.P(name + ".weight"), n.P(name + ".bias"), y.p, x.rows(), x.C, s, y.amax);
    return y;
  }

  // GroupNorm(32)(+ scale-shift) + SiLU + conv3x3 (stride 1, pad 1) of x (optionally the channel concat [x | x2]): the ResBlock pattern
  // of all four network families (OAI:255-275, IU:241-261, AEM:121-141, ddpm/diffusion.py:117-139).  The GroupNorm kernel reads
  // both sources and writes the normalised concat, which the conv then reads as its one source.  `into` (optional): preallocated output.
  Tensor gn_silu_conv3(const Tensor& x, const Tensor* x2, const std::string& norm, float eps, const std::string& conv, const float* scale = nullptr,
                       const float* shift = nullptr, int ld_ss = 0, const float* rowvec = nullptr, int ld_rowvec = 0, const float* residual = nullptr,
                       Tensor* into = nullptr, float* out_nchw = nullptr, const int* src_img = nullptr) {
    const Tensor h = gn(x, x2, norm, eps, true, scale, shift, ld_ss, src_img);
    return conv3(h, conv, 1, 1, 1, rowvec, ld_rowvec, residual, out_nchw, into);
  }

  // AttnBlock (AEM:178-202): single head, d = C, scale C^-1/2
  Tensor attn(const Tensor& x, const std::string& p) {
    const int C = x.C, HW = x.H * x.W;
    Tensor out = alloc(x.B, x.H, x.W, C);
    Scope sc(e.arena);
    Tensor xn = gn(x, nullptr, p + ".norm", 1e-6f, false);
    Tensor q = linear(xn, p + ".q", true);
    Tensor k = linear(xn, p + ".k", true);
    Tensor v = linear(xn, p + ".v", true, nullptr, true);       // its range bounds the attention output
    Tensor a = alloc(x.B, x.H, x.W, C);
    a.amax = v.amax;
    const float scale = (float)pow((double)C, -0.5);
    bool done = false;
    if (e.mma_mode == 1 && (HW % 32) == 0 && HW >= 128) {
      // tensor-core path: S = q k^T, row softmax, O = P V with V transposed to [C, B*HW] (both P.V operands K-major)
      Scope sa(e.arena);
      float* vt = (float*)e.arena.alloc((size_t)C * x.rows() * sizeof(float));
      nhwc_to_nchw(e, v.p, vt, 1, C, x.rows(), s);
      done = attention_tc(e, q.p, C, k.p, C, C, vt, a.p, C, x.B, HW, HW, 1, C, scale, s);
    }
    if (!done) attention(e, q.p, C, k.p, C, v.p, C, a.p, C, x.B, HW, HW, 1, C, C, scale, s);
    out.amax = e.amax_slot();
    out.stats = e.stat_alloc((size_t)x.B * C * 2);
    linear_into(a.p, C, C, nullptr, 0, 0, x.rows(), n.P(p + ".proj_out.weight"), C, n.P(p + ".proj_out.bias"), x.p, C, out.p, C, nullptr, v.amax, nullptr,
                out.amax, out.stats, HW);
    return out;
  }

};

// ------------------------------------------------------------------------------------------------ U-Nets
struct UNetExec : Exec {
  const float* E = nullptr;   // [B, emb_rows] all ResBlock emb projections
  int ctx_len = 0;
  int ctx_lp = 0;                          // context rows per image, padded for the fused cross-attention
  bool kv_reuse = false, kv_hit = false;   // loop mode: context K / V live in n.ctxkv (kv_hit: already computed)
  const AttnControl* ctl = nullptr;        // attention control of this call, or null
  const AttnProbe* probe = nullptr;        // cross-attention probe of this call, or null
  int probed = 0;                          // layers probed so far in this call
  int st_layer = 0;                        // SpatialTransformers run so far in this call (AttnControl::start_layer counts them)
  // the contexts the cross-attention projects: [0] the call's context, [1] the V' context (AttnControl::ctx_v), [2] the refine
  // context (ctx_w); src null when absent.  pad: src zero-padded to ctx_lp rows per image (fused route only); amax: range slot of
  // src (A operand of the K / V projections)
  struct CtxIn {
    const float* src = nullptr;
    const float* pad = nullptr;
    float* amax = nullptr;
  } cx[3];
  size_t kv_off = 0;
  float* kv_take(size_t floats) {
    if (!kv_reuse) return (float*)e.arena.alloc(floats * sizeof(float));
    float* p = n.ctxkv.buf + kv_off;
    kv_off += (floats + 63) & ~(size_t)63;
    CDX_CHECK(kv_off <= n.ctxkv.cap, "context K/V cache overflow (%zu > %zu floats)", kv_off, n.ctxkv.cap);
    return p;
  }
  // range slots: of the contexts (CtxIn::amax) and of each layer's V (bounds the attention output).  In loop mode the projections
  // run only in the first call, so their slots live with the cached K / V, outside the per-call pool.
  int kv_layer = 0;
  float* kv_amax() {
    if (!kv_reuse) return e.amax_slot();
    CDX_CHECK(kv_layer < Net::CtxKV::MAX_LAYERS, "too many cross-attention layers for the context cache");
    return e.dry() ? reinterpret_cast<float*>((uintptr_t)0x100) : n.ctxkv.amax + 1 + kv_layer++;
  }
  // V' range slot = max(the layer's K | V range, max |V'|): starts as a copy of the K | V slot, the V' projection maxes into it, so
  // an identity token map leaves every exponent (and the output's range) as without control
  void v2_range(const float* kv_slot, float* v2_slot) {
    if (!e.dry()) CDX_CUDA(cudaMemcpyAsync(v2_slot, kv_slot, sizeof(float), cudaMemcpyDeviceToDevice, s));
  }
  // V^T planes of one padded context (Mk rows) in the engine's format for the fused cross-attention of block t, maxing its range
  // into `slot`; with k_hi also the K planes.  fp16: one fused K | V projection, K and V^T split from it with the slot of the whole
  // output -- a V' or V'' context takes the same projection with its K half unused, so an identity token map gives V' == V.
  // TF32: K and V^T = Wv . ctx^T (a swapped-role GEMM, so that both P.V operands are K-major) written as planes by the epilogues
  void context_planes(const CtxIn& x, const std::string& t, int C, int Mk, float* slot, float* k_hi, float* k_lo, float* vt_hi, float* vt_lo) {
    const int D = n.ucfg.context_dim;
    if (e.tc_kind >= 1) {
      Scope sk(e.arena);
      float* kvf = (float*)e.arena.alloc((size_t)Mk * 2 * C * sizeof(float));
      linear_into(x.pad, D, D, nullptr, 0, 0, Mk, n.P(t + ".attn2.to_k.weight"), 2 * C, nullptr, nullptr, 0, kvf, 2 * C, nullptr, x.amax, nullptr, slot);
      context_split_h16(e, kvf, Mk, C, slot, k_hi, k_lo, vt_hi, vt_lo, s);
    } else {
      if (k_hi) linear_into(x.pad, D, D, nullptr, 0, 0, Mk, n.P(t + ".attn2.to_k.weight"), C, nullptr, nullptr, 0, k_hi, C, k_lo, x.amax);
      linear_into(n.P(t + ".attn2.to_v.weight"), D, D, nullptr, 0, 0, C, x.pad, Mk, nullptr, nullptr, 0, vt_hi, Mk, vt_lo, nullptr, nullptr, slot);
    }
  }
  // the probe of one layer: the first probed layer of the call stores the map, later ones add
  void probe_layer(const ProbeOperands& po, int HW, int heads, int d, float scale) {
    attn_probe(e, po, probe->rows, probe->span, probe->weights, probe->n_rows, probe->map, HW, ctx_len, heads, d, scale, probed > 0, s);
    ++probed;
  }
  bool oai;
  UNetExec(Net& net, cudaStream_t st) : Exec(net, st), oai(net.kind == NET_UNET_OPENAI) {}

  // Plug-and-Play: the row table of output block k's ResBlock in this call, or null when it is not controlled
  const int* feature_row(int k) const {
    if (!ctl || !ctl->pnp_feat) return nullptr;
    for (int i = 0; i < ctl->n_feat; ++i)
      if (ctl->feat_blocks[i] == k) return ctl->pnp_row;
    return nullptr;
  }

  // ResBlock (OAI:255-275 / IU:241-261).  updown: 0 none, 1 down (avg-pool), 2 up (nearest).  feat_row (optional device [B],
  // Plug-and-Play feature injection): row r's out_layers run on row feat_row[r]'s in_layers output; the skip stays row r's own
  Tensor resblock(const Tensor& x, const Tensor* x2, const std::string& p, int updown = 0, const int* feat_row = nullptr) {
    const int Cout = n.dim0(p + ".in_layers.2.weight");
    const int eoff = n.emb_off.at(p);
    const int oH = updown == 1 ? x.H / 2 : (updown == 2 ? x.H * 2 : x.H);
    const int oW = updown == 1 ? x.W / 2 : (updown == 2 ? x.W * 2 : x.W);
    Tensor out = alloc(x.B, oH, oW, Cout);
    Scope sc(e.arena);
    Tensor xs = x;    // skip-path input after x_upd
    Tensor h1, h2;
    if (updown != 0) h1 = gn(x, x2, p + ".in_layers.0", 1e-5f, true);
    if (updown == 1) {
      CDX_CHECK(!x2, "res down with concat input");
      Tensor hp = alloc(x.B, oH, oW, x.C);
      avgpool2(e, h1.p, hp.p, x.B, x.H, x.W, x.C, s);
      hp.amax = h1.amax;                                         // |average| <= max
      xs = alloc(x.B, oH, oW, x.C);
      avgpool2(e, x.p, xs.p, x.B, x.H, x.W, x.C, s);
      xs.amax = x.amax;
      h2 = conv3(hp, p + ".in_layers.2");
    } else if (updown == 2) {
      CDX_CHECK(!x2, "res up with concat input");
      xs = alloc(x.B, oH, oW, x.C);
      upsample2(e, x.p, xs.p, x.B, x.H, x.W, x.C, s);
      xs.amax = x.amax;
      h2 = conv3(h1, p + ".in_layers.2", 1, 1, 2);
    } else if (oai) {
      h2 = gn_silu_conv3(x, x2, p + ".in_layers.0", 1e-5f, p + ".in_layers.2", nullptr, nullptr, 0, E + eoff, n.emb_rows);     // + emb_out (OAI:273)
    } else {
      h2 = gn_silu_conv3(x, x2, p + ".in_layers.0", 1e-5f, p + ".in_layers.2");
    }
    const float* residual;
    if (n.has(p + ".skip_connection.weight")) {
      Tensor sk = alloc(x.B, oH, oW, Cout);
      linear_into(xs.p, xs.C, xs.C, x2 ? x2->p : nullptr, x2 ? x2->C : 0, x2 ? x2->C : 0, xs.rows(), n.P(p + ".skip_connection.weight"), Cout,
                  n.P(p + ".skip_connection.bias"), nullptr, 0, sk.p, Cout, nullptr, xs.amax, x2 ? x2->amax : nullptr);
      residual = sk.p;
    } else {
      CDX_CHECK(!x2 && xs.C == Cout, "resblock %s: identity skip with mismatching channels", p.c_str());
      residual = xs.p;
    }
    // out_layers: GroupNorm (i-DDPM: scale-shift norm, IU:253-257) + SiLU + conv3x3 + residual, written into `out`
    if (oai) gn_silu_conv3(h2, nullptr, p + ".out_layers.0", 1e-5f, p + ".out_layers.3", nullptr, nullptr, 0, nullptr, 0, residual, &out, nullptr,
                           feat_row);
    else gn_silu_conv3(h2, nullptr, p + ".out_layers.0", 1e-5f, p + ".out_layers.3", E + eoff, E + eoff + Cout, n.emb_rows, nullptr, 0, residual, &out,
                       nullptr, feat_row);
    return out;
  }

  // SpatialTransformer (ATT:250-261) with one BasicTransformerBlock (ATT:211-215)
  Tensor spatial_transformer(const Tensor& x, const std::string& p) {
    const int C = x.C, heads = n.ucfg.num_head_channels > 0 ? C / n.ucfg.num_head_channels : n.ucfg.num_heads, d = C / heads;
    const int M = x.rows(), HW = x.H * x.W, B = x.B;
    Tensor out = alloc(B, x.H, x.W, C);
    Scope sc(e.arena);
    const float scale = (float)pow((double)d, -0.5);
    const std::string t = p + ".transformer_blocks.0";
    Tensor xn = gn(x, nullptr, p + ".norm", 1e-6f, false);
    Tensor h = linear(xn, p + ".proj_in", true);
    // --- self-attention: fused q|k|v projection (weights adjacent in the blob)
    Tensor h2;
    {
      Tensor n1 = ln(h, t + ".norm1");
      Tensor a = alloc(B, x.H, x.W, C);
      a.amax = e.amax_slot();                   // <- max |V| (written by whichever projection produces V)
      bool done = false;
      const bool flash_ok = flash_eligible(e, HW, HW, d, C);
      // Prompt-to-Prompt, or Plug-and-Play on layers >= pnp_layer: the controlled rows take their source rows' queries and keys
      const int* srow = (ctl && ctl->self && HW <= ctl->self_max_tokens)        ? ctl->qk_row
                        : (ctl && ctl->pnp_attn && st_layer >= ctl->pnp_layer) ? ctl->pnp_row
                                                                              : nullptr;
      // mutual self-attention: the controlled rows' queries over their source rows' keys and values
      const int* mrow = (ctl && ctl->mutual && st_layer >= ctl->start_layer) ? ctl->kv_row : nullptr;
      ++st_layer;
      CDX_CHECK((!srow && !mrow) || flash_ok, "attention control: self-attention at HW=%d d=%d would take the unfused route (mma mode and "
                "head width must run the fused kernel)", HW, d);
      if (flash_ok && e.tc_kind >= 1) {
        // fp16-split fused attention: ONE plain fp32 q|k|v projection (its range tracked by the epilogue), then one pass that
        // writes the fp16 hi / lo planes of q|k and of V^T (both P.V operands K-major for wgmma) with the tensor's exponent.
        // V^T keeps Nvs = HW rounded up to 8 keys per image (zero columns): its TMA map needs 16-byte key strides
        Scope sa(e.arena);
        float* qkv = (float*)e.arena.alloc((size_t)M * 3 * C * sizeof(float));
        linear_into(n1.p, C, C, nullptr, 0, 0, M, n.P(t + ".attn1.to_q.weight"), 3 * C, nullptr, nullptr, 0, qkv, 3 * C, nullptr, n1.amax, nullptr,
                    a.amax);                    // range of q | k | v (v bounds the attention output: a convex combination of V rows)
        // (mode 5: hi planes only, one-term kernel)
        done = self_attention_h16(e, qkv, a.amax, a.p, B, HW, C, heads, d, scale, !e.attn_one, s, srow, mrow);
        CDX_CHECK(done, "flash attention (fp16-split) rejected an eligible shape (HW=%d d=%d)", HW, d);
      } else if (flash_ok && (HW % 4) != 0) {
        // TF32 planes with a per-image key count off the 16-byte TMA granule: V row-major, copied into rows padded to Nvs keys
        // per image (zero rows), transposed and split; q|k planes from the projection's epilogue as below
        Scope sa(e.arena);
        const size_t nqk = (size_t)M * 2 * C;
        float* qk_hi = (float*)e.arena.alloc(nqk * sizeof(float));
        float* qk_lo = (float*)e.arena.alloc(nqk * sizeof(float));
        float* vr = (float*)e.arena.alloc((size_t)M * C * sizeof(float));
        linear_into(n1.p, C, C, nullptr, 0, 0, M, n.P(t + ".attn1.to_q.weight"), 2 * C, nullptr, nullptr, 0, qk_hi, 2 * C, qk_lo, n1.amax);
        linear_into(n1.p, C, C, nullptr, 0, 0, M, n.P(t + ".attn1.to_v.weight"), C, nullptr, nullptr, 0, vr, C, nullptr, n1.amax, nullptr, a.amax);
        done = self_attention_tf32_padded(e, qk_hi, qk_lo, vr, a.p, B, HW, C, heads, d, scale, s, srow, mrow);
        CDX_CHECK(done, "flash attention rejected an eligible shape (HW=%d d=%d)", HW, d);
      } else if (flash_ok) {
        // fused tensor-core attention: q|k projection and V^T (= Wv . X^T, a swapped-role GEMM, so that both P.V operands
        // are K-major for wgmma) are written by their GEMM epilogues directly as TF32 hi / lo planes
        Scope sa(e.arena);
        const size_t nqk = (size_t)M * 2 * C, nvt = (size_t)C * M;
        float* qk_hi = (float*)e.arena.alloc(nqk * sizeof(float));
        float* qk_lo = (float*)e.arena.alloc(nqk * sizeof(float));
        float* vt_hi = (float*)e.arena.alloc(nvt * sizeof(float));
        float* vt_lo = (float*)e.arena.alloc(nvt * sizeof(float));
        if ((2 * C) % 128 == 0 && M >= 64 && (C % 4) == 0) {
          // one fused q|k|v projection (weights adjacent in the blob): q|k stored row-major as planes, the v columns stored
          // transposed by the epilogue (thread = row, so a column is 32 consecutive floats per warp) -> V^T planes
          GemmArgs g;
          g.mode = 0;
          g.M = M; g.N = 3 * C; g.K = C;
          g.A = n1.p; g.lda = C; g.C1 = C;
          g.Bw = n.P(t + ".attn1.to_q.weight"); g.ldb = C;
          g.Cout = qk_hi; g.ldc = 2 * C; g.Cout_lo = qk_lo;
          g.Ct_hi = vt_hi; g.Ct_lo = vt_lo; g.t_col0 = 2 * C; g.ldt = M;
          g.a_amax = n1.amax;
          g.c_amax = a.amax;                    // range of q | k | v: bounds the attention output (a convex combination of V rows)
          run(g);
        } else {
          linear_into(n1.p, C, C, nullptr, 0, 0, M, n.P(t + ".attn1.to_q.weight"), 2 * C, nullptr, nullptr, 0, qk_hi, 2 * C, qk_lo, n1.amax);
          linear_into(n.P(t + ".attn1.to_v.weight"), C, C, nullptr, 0, 0, C, n1.p, M, nullptr, nullptr, 0, vt_hi, M, vt_lo, nullptr, nullptr,
                      a.amax);   // V^T = Wv . X^T
        }
        const AttnPlanes pl{AttnPlanes::TF32, qk_hi, qk_lo, 2 * C, qk_hi + C, qk_lo + C, 2 * C, vt_hi, vt_lo};
        done = flash_attention(e, pl, a.p, C, B, HW, HW, HW, HW, heads, d, scale, s, srow, nullptr, 0, mrow);
        CDX_CHECK(done, "flash attention rejected an eligible shape (HW=%d d=%d)", HW, d);
      } else if (e.mma_mode >= 1 && (HW % 32) == 0 && HW >= 128 && (d % 4) == 0) {
        // unfused tensor-core attention (mode 2, or shapes the fused kernel does not cover)
        Scope sa(e.arena);
        Tensor qk = alloc(B, x.H, x.W, 2 * C);
        linear_into(n1.p, C, C, nullptr, 0, 0, M, n.P(t + ".attn1.to_q.weight"), 2 * C, nullptr, nullptr, 0, qk.p, 2 * C, nullptr, n1.amax);
        float* vt = (float*)e.arena.alloc((size_t)C * M * sizeof(float));
        if (e.tc_kind >= 1) {
          // V by the ordinary (fp16-split, weight-planes) projection, then transposed: the swapped-role GEMM X . Wv^T -> V^T has an
          // activation as its B operand and runs on the TF32 SS path at ~85 TFLOP/s (0.08 ms per 16x16-level layer at batch 8)
          float* vr = (float*)e.arena.alloc((size_t)M * C * sizeof(float));
          linear_into(n1.p, C, C, nullptr, 0, 0, M, n.P(t + ".attn1.to_v.weight"), C, nullptr, nullptr, 0, vr, C, nullptr, n1.amax, nullptr, a.amax);
          nhwc_to_nchw(e, vr, vt, 1, C, M, s);
        } else {
          linear_into(n.P(t + ".attn1.to_v.weight"), C, C, nullptr, 0, 0, C, n1.p, M, nullptr, nullptr, 0, vt, M, nullptr, nullptr, nullptr, a.amax);
        }
        done = attention_tc(e, qk.p, 2 * C, qk.p + C, 2 * C, d, vt, a.p, C, B, HW, HW, heads, d, scale, s);
      }
      if (!done) {
        Scope sa(e.arena);
        Tensor qkv = alloc(B, x.H, x.W, 3 * C);
        linear_into(n1.p, C, C, nullptr, 0, 0, M, n.P(t + ".attn1.to_q.weight"), 3 * C, nullptr, nullptr, 0, qkv.p, 3 * C, nullptr, n1.amax, nullptr,
                    a.amax);
        attention(e, qkv.p, 3 * C, qkv.p + C, 3 * C, qkv.p + 2 * C, 3 * C, a.p, C, B, HW, HW, heads, d, d, scale, s);
      }
      h2 = linear(a, t + ".attn1.to_out.0", true, h.p);
    }
    // --- cross-attention: q from tokens, fused k|v projection of the context
    Tensor h3;
    {
      Tensor n2 = ln(h2, t + ".norm2");
      const int D = n.ucfg.context_dim;
      Tensor a = alloc(B, x.H, x.W, C);
      a.amax = kv_amax();                       // <- max |V| of the context projection (lives with the cached K / V in loop mode)
      // attention control: controlled rows attend with their source row's Q / K; with a V context every row reads V'^T (the
      // token-mapped context's projection; its range slot also bounds this call's output) instead of V^T
      const bool vmap = ctl && ctl->ctx_v;
      float* v2_amax = vmap ? kv_amax() : nullptr;
      // refine: the controlled rows also add their own attention over V''^T (the refine context's projection) into the output.
      // V'' takes its own slot, from zero: the context is zero outside the controlled rows, so own weights of zero give a zero
      // slot.  The output is no longer a convex combination of one tensor's rows, |out| <= max |V'| + max |V''|: its slot is the
      // sum, formed on the device with the projections (once per loop), and equal to the first term's slot when V'' is zero
      const bool wmap = ctl && ctl->ctx_w;
      float* v3_amax = wmap ? kv_amax() : nullptr;
      float* sum_amax = wmap ? kv_amax() : nullptr;
      const int* crow = (ctl && ctl->cross) ? ctl->qk_row : nullptr;
      const bool use_v2 = crow && vmap;
      const bool use_v3 = crow && wmap;
      bool done = false;
      Tensor q;
      // LEDITS++'s probe: this layer's Q and K as its route multiplied them
      const bool probe_here = probe && HW == probe->tokens && (p.rfind("input_blocks.", 0) == 0 || p.rfind("output_blocks.", 0) == 0);
      ProbeOperands po;
      const bool flash_ok = cx[0].pad && flash_eligible(e, HW, ctx_len, d, C);
      CDX_CHECK(!crow || flash_ok, "attention control: cross-attention at HW=%d d=%d would take the unfused route (mma mode "
                "and head width must run the fused kernel)", HW, d);
      if (flash_ok) {
        // fused attention over the zero-padded context (ctx_lp rows per image, keys >= ctx_len masked in the kernel).  fp16 planes:
        // q projected as plain fp32 (range tracked) and split; K and V share the layer's slot (one exponent for both).  TF32 planes:
        // q written as planes by its projection's epilogue.  In loop mode the context planes and slots are computed by the first call
        // only.  Mode 5: hi planes only (the cache then holds no lo planes; it lives for one loop, which runs in one mode)
        Scope sa(e.arena);
        const bool h16 = e.tc_kind >= 1, lo = !e.attn_one;
        const int Mk = B * ctx_lp;
        const size_t np = h16 ? (size_t)Mk * C / 2 : (size_t)Mk * C;     // floats per plane
        float* k_hi = kv_take(np);
        float* k_lo = lo ? kv_take(np) : nullptr;
        float* vt_hi = kv_take(np);
        float* vt_lo = lo ? kv_take(np) : nullptr;
        float* v2_hi = vmap ? kv_take(np) : nullptr;
        float* v2_lo = vmap && lo ? kv_take(np) : nullptr;
        float* v3_hi = wmap ? kv_take(np) : nullptr;
        float* v3_lo = wmap && lo ? kv_take(np) : nullptr;
        AttnPlanes pl{h16 ? AttnPlanes::H16 : AttnPlanes::TF32, nullptr, nullptr, C, k_hi, k_lo, C, nullptr, nullptr};
        if (h16) {
          Tensor qf = linear(n2, t + ".attn2.to_q", false, nullptr, true);
          void* q_hi = e.arena.alloc((size_t)M * C * 2);
          void* q_lo = lo ? e.arena.alloc((size_t)M * C * 2) : nullptr;
          split_rows_h16(e, qf.p, M, C, C, q_hi, q_lo, C, qf.amax, s);
          pl.q_hi = q_hi; pl.q_lo = q_lo; pl.q_amax = qf.amax;
          po.fmt = ProbeOperands::H16; po.q = qf.p;
        } else {
          float* q_hi = (float*)e.arena.alloc((size_t)M * C * sizeof(float));
          float* q_lo = (float*)e.arena.alloc((size_t)M * C * sizeof(float));
          linear_into(n2.p, C, C, nullptr, 0, 0, M, n.P(t + ".attn2.to_q.weight"), C, nullptr, nullptr, 0, q_hi, C, q_lo, n2.amax);
          pl.q_hi = q_hi; pl.q_lo = q_lo;
          po.fmt = ProbeOperands::TF32; po.q = q_hi; po.q_lo = q_lo;
        }
        if (!kv_hit) {
          context_planes(cx[0], t, C, Mk, a.amax, k_hi, k_lo, vt_hi, vt_lo);
          if (vmap) {
            v2_range(a.amax, v2_amax);
            context_planes(cx[1], t, C, Mk, v2_amax, nullptr, nullptr, v2_hi, v2_lo);
          }
          if (wmap) {             // V'', then the output's slot
            context_planes(cx[2], t, C, Mk, v3_amax, nullptr, nullptr, v3_hi, v3_lo);
            add(e, vmap ? v2_amax : a.amax, v3_amax, sum_amax, 1, s);
          }
        }
        pl.k_amax = a.amax;
        pl.vt_hi = use_v2 ? v2_hi : vt_hi; pl.vt_lo = use_v2 ? v2_lo : vt_lo; pl.v_amax = use_v2 ? v2_amax : a.amax;
        done = flash_attention(e, pl, a.p, C, B, HW, ctx_len, ctx_lp, ctx_lp, heads, d, scale, s, crow);
        CDX_CHECK(done, "flash cross-attention rejected an eligible shape (HW=%d d=%d L=%d)", HW, d, ctx_len);
        if (use_v3) {             // + the controlled rows' own attention over V'' (accumulating launch, those rows' CTAs only)
          pl.vt_hi = v3_hi; pl.vt_lo = v3_lo; pl.v_amax = v3_amax;
          done = flash_attention(e, pl, a.p, C, B, HW, ctx_len, ctx_lp, ctx_lp, heads, d, scale, s, nullptr, ctl->own_rows, ctl->n_own);
          CDX_CHECK(done, "flash cross-attention rejected the refine term (HW=%d d=%d L=%d)", HW, d, ctx_len);
        }
        if (probe_here) {
          po.ldq = C; po.k = k_hi; po.k_lo = k_lo; po.ldk = C; po.Lk = ctx_lp; po.k_amax = a.amax;
          probe_layer(po, HW, heads, d, scale);
        }
      }
      if (use_v3) a.amax = sum_amax;            // the sum of a convex combination of V' rows and one of V'' rows
      else if (use_v2) a.amax = v2_amax;        // the output is a convex combination of V' rows
      if (!done) q = linear(n2, t + ".attn2.to_q", false);
      if (!done) {
        Scope sa(e.arena);
        float* kv = kv_take((size_t)B * ctx_len * 2 * C);
        if (!kv_hit) linear_into(cx[0].src, D, D, nullptr, 0, 0, B * ctx_len, n.P(t + ".attn2.to_k.weight"), 2 * C, nullptr, nullptr, 0, kv, 2 * C,
                                 nullptr, cx[0].amax, nullptr, a.amax);
        attention(e, q.p, C, kv, 2 * C, kv + C, 2 * C, a.p, C, B, HW, ctx_len, heads, d, d, scale, s);
        if (probe_here) {
          po.fmt = ProbeOperands::F32; po.q = q.p; po.ldq = C; po.k = kv; po.ldk = 2 * C; po.Lk = ctx_len;
          probe_layer(po, HW, heads, d, scale);
        }
      }
      h3 = linear(a, t + ".attn2.to_out.0", true, h2.p);
    }
    // --- GEGLU feed-forward (ATT:37-64)
    Tensor h4;
    {
      Tensor n3 = ln(h3, t + ".norm3");
      Tensor g = alloc(B, x.H, x.W, 4 * C);
      if (n.param(t + ".ff.net.0.proj.weight").geglu) {
        // value * gelu(gate) applied in the projection's epilogue (weights stored [32 value | 32 gate] row blocks)
        GemmArgs ga;
        ga.mode = 0;
        ga.M = M; ga.N = 8 * C; ga.K = C;
        ga.A = n3.p; ga.lda = C; ga.C1 = C;
        ga.Bw = n.P(t + ".ff.net.0.proj.weight"); ga.ldb = C;
        ga.bias = n.P(t + ".ff.net.0.proj.bias");
        ga.geglu = 1;
        ga.Cout = g.p; ga.ldc = 4 * C;
        ga.a_amax = n3.amax;
        g.amax = e.amax_slot();
        ga.c_amax = g.amax;
        run(ga);
      } else {
        Tensor f = linear(n3, t + ".ff.net.0.proj", true);
        geglu(e, f.p, g.p, M, 4 * C, s);        // (range of g not tracked here: the consumer measures it)
      }
      h4 = linear(g, t + ".ff.net.2", true, h3.p, true);
    }
    out.amax = e.amax_slot();
    out.stats = e.stat_alloc((size_t)B * C * 2);
    linear_into(h4.p, C, C, nullptr, 0, 0, M, n.P(p + ".proj_out.weight"), C, n.P(p + ".proj_out.bias"), x.p, C, out.p, C, nullptr, h4.amax, nullptr,
                out.amax, out.stats, HW);
    return out;
  }

  // i-DDPM AttentionBlock + QKVAttentionLegacy (IU:304-310, 342-363): qkv channels are [head][q|k|v][d]
  Tensor attention_block(const Tensor& x, const std::string& p) {
    const int C = x.C, d = n.ucfg.num_head_channels > 0 ? n.ucfg.num_head_channels : C / n.ucfg.num_heads, heads = C / d;
    const int M = x.rows(), HW = x.H * x.W, B = x.B;
    Tensor out = alloc(B, x.H, x.W, C);
    Scope sc(e.arena);
    Tensor xn = gn(x, nullptr, p + ".norm", 1e-5f, false);
    Tensor qkv = alloc(B, x.H, x.W, 3 * C);
    qkv.amax = e.amax_slot();
    linear_into(xn.p, C, C, nullptr, 0, 0, M, n.P(p + ".qkv.weight"), 3 * C, n.P(p + ".qkv.bias"), nullptr, 0, qkv.p, 3 * C, nullptr, xn.amax, nullptr,
                qkv.amax);
    const float sq = (float)(1.0 / sqrt(sqrt((double)d)));
    Tensor a = alloc(B, x.H, x.W, C);
    attention(e, qkv.p, 3 * C, qkv.p + d, 3 * C, qkv.p + 2 * d, 3 * C, a.p, C, B, HW, HW, heads, d, 3 * d, sq * sq, s);
    out.amax = e.amax_slot();
    out.stats = e.stat_alloc((size_t)B * C * 2);
    // |attention output| <= max |V| <= max |qkv|
    linear_into(a.p, C, C, nullptr, 0, 0, M, n.P(p + ".proj_out.weight"), C, n.P(p + ".proj_out.bias"), x.p, C, out.p, C, nullptr, qkv.amax, nullptr,
                out.amax, out.stats, HW);
    return out;
  }

  Tensor attn_layer(const Tensor& x, const std::string& p) { return (oai && n.ucfg.context_dim > 0) ? spatial_transformer(x, p) : attention_block(x, p); }

  // ResnetBlock.forward (ddpm/diffusion.py:117-139): conv1(swish(norm1 x)) + temb_proj(swish temb); conv2(swish(norm2 h)); + shortcut
  Tensor ddpm_resblock(const Tensor& x, const Tensor* x2, const std::string& p) {
    const int Cout = n.dim0(p + ".conv1.weight");
    Tensor out = alloc(x.B, x.H, x.W, Cout);
    Scope sc(e.arena);
    Tensor h2 = gn_silu_conv3(x, x2, p + ".norm1", 1e-6f, p + ".conv1", nullptr, nullptr, 0, E + n.emb_off.at(p), n.emb_rows);
    const float* residual;
    if (n.has(p + ".nin_shortcut.weight")) {
      Tensor sk = alloc(x.B, x.H, x.W, Cout);
      linear_into(x.p, x.C, x.C, x2 ? x2->p : nullptr, x2 ? x2->C : 0, x2 ? x2->C : 0, x.rows(), n.P(p + ".nin_shortcut.weight"), Cout,
                  n.P(p + ".nin_shortcut.bias"), nullptr, 0, sk.p, Cout, nullptr, x.amax, x2 ? x2->amax : nullptr);
      residual = sk.p;
    } else {
      CDX_CHECK(!x2 && x.C == Cout, "ddpm resblock %s: identity skip with mismatching channels", p.c_str());
      residual = x.p;
    }
    gn_silu_conv3(h2, nullptr, p + ".norm2", 1e-6f, p + ".conv2", nullptr, nullptr, 0, nullptr, 0, residual, &out);
    return out;
  }

  // DDPM.forward (ddpm/diffusion.py:299-337)
  void forward_ddpm(const float* x_nchw, const float* t_dev, float* out_nchw, int B, int H, int W) {
    const cdx_unet_config& c = n.ucfg;
    const int ch = c.model_channels, half = ch / 2, ted = n.ted, L = c.n_mult;
    Scope top(e.arena);
    e.pools_reset(s);
    Tensor temb = alloc(B, 1, 1, ch);
    timestep_embedding(e, t_dev, n.freqs_dev, temb.p, B, half, s, true);          // [sin | cos]
    Tensor e1 = linear(temb, "temb.dense.0", true);
    silu(e, e1.p, e1.p, e1.numel(), s);
    Tensor emb = linear(e1, "temb.dense.1", true);
    silu(e, emb.p, emb.p, emb.numel(), s);   // every ResnetBlock applies the swish before its temb_proj (:125)
    Tensor Eall = alloc(B, 1, 1, n.emb_rows);
    linear_into(emb.p, ted, ted, nullptr, 0, 0, B, n.blob + n.emb_w_off, n.emb_rows, n.blob + n.emb_b_off, nullptr, 0, Eall.p, n.emb_rows);
    E = Eall.p;
    Tensor xin = alloc(B, H, W, c.in_channels);
    nchw_to_nhwc(e, x_nchw, xin.p, B, c.in_channels, H * W, s);
    std::vector<Tensor> hs;
    hs.push_back(conv3(xin, "conv_in"));
    int ds = 1;
    for (int lvl = 0; lvl < L; ++lvl) {
      const std::string D = "down." + std::to_string(lvl);
      const bool at = contains(c.attention_ds, c.n_attn, ds);
      for (int b = 0; b < c.num_res_blocks; ++b) {
        Tensor h = ddpm_resblock(hs.back(), nullptr, D + ".block." + std::to_string(b));
        if (at) h = attn(h, D + ".attn." + std::to_string(b));
        hs.push_back(h);
      }
      if (lvl != L - 1) { hs.push_back(conv3(hs.back(), D + ".downsample.conv", 2, 0)); ds *= 2; }      // pad (0,1,0,1), :60-64
    }
    Tensor h = hs.back();
    h = ddpm_resblock(h, nullptr, "mid.block_1");
    h = attn(h, "mid.attn_1");
    h = ddpm_resblock(h, nullptr, "mid.block_2");
    for (int lvl = L - 1; lvl >= 0; --lvl) {
      const std::string U = "up." + std::to_string(lvl);
      const bool at = contains(c.attention_ds, c.n_attn, ds);
      for (int b = 0; b <= c.num_res_blocks; ++b) {
        const Tensor skip = hs.back();
        hs.pop_back();
        h = ddpm_resblock(h, &skip, U + ".block." + std::to_string(b));
        if (at) h = attn(h, U + ".attn." + std::to_string(b));
      }
      if (lvl != 0) { h = conv3(h, U + ".upsample.conv", 1, 1, 2); ds /= 2; }
    }
    gn_silu_conv3(h, nullptr, "norm_out", 1e-6f, "conv_out", nullptr, nullptr, 0, nullptr, 0, nullptr, nullptr, out_nchw);
  }

  void forward(const float* x_nchw, const float* t_dev, const float* context, int L, float* out_nchw, int B, int H, int W) {
    const cdx_unet_config& c = n.ucfg;
    ctx_len = L;
    ctx_lp = (L + 7) & ~7;                // (fp16 planes: 16-byte TMA strides need 8 keys)
    const int mc = c.model_channels, half = mc / 2, ted = n.ted;
    Scope top(e.arena);
    e.pools_reset(s);
    kv_off = 0;
    kv_hit = false;
    if (kv_reuse && context && L > 0) {
      Net::CtxKV& kc = n.ctxkv;
      size_t sumC = 0;
      for (const Param& pp : n.params)
        if (pp.name.size() > 17 && pp.name.compare(pp.name.size() - 17, 17, "attn2.to_k.weight") == 0) sumC += (size_t)pp.dims[0] + 64;
      const size_t need = (4 + (ctl && ctl->ctx_v ? 2 : 0) + (ctl && ctl->ctx_w ? 2 : 0)) * (size_t)B * ctx_lp * sumC;   // K, V (V', V'') hi + lo
      if (kc.cap < need) {
        CDX_CUDA(cudaDeviceSynchronize());
        if (kc.buf) CDX_CUDA(cudaFree(kc.buf));
        kc.buf = nullptr; kc.cap = 0; kc.valid = false;
        CDX_CUDA(cudaMalloc(&kc.buf, need * sizeof(float)));
        kc.cap = need;
      }
      kv_hit = kc.valid && kc.ctx == context && kc.ctx_v == (ctl ? ctl->ctx_v : nullptr) && kc.ctx_w == (ctl ? ctl->ctx_w : nullptr) && kc.L == L &&
               kc.B == B && !e.dry();
      if (!kc.amax) {
        CDX_CUDA(cudaMalloc(&kc.amax, (Net::CtxKV::MAX_LAYERS + 1) * sizeof(float)));
        CDX_CUDA(cudaMemset(kc.amax, 0, (Net::CtxKV::MAX_LAYERS + 1) * sizeof(float)));
      }
      if (!kv_hit && !e.dry()) CDX_CUDA(cudaMemsetAsync(kc.amax, 0, (Net::CtxKV::MAX_LAYERS + 1) * sizeof(float), s));
    }
    kv_layer = 0;
    if (context && L > 0) {
      // each context's range (A operand of the K / V projections) and, for the fused route, its rows padded with zeros to ctx_lp per
      // image (TMA needs 16-byte strides for K and V^T); in loop mode both once per loop
      const size_t D = (size_t)c.context_dim;
      const float* src[3] = {context, ctl ? ctl->ctx_v : nullptr, ctl ? ctl->ctx_w : nullptr};
      for (int i = 0; i < 3; ++i) {
        if (!src[i]) continue;
        CtxIn& x = cx[i];
        x.src = src[i];
        // the context's slot is the cache's first; the V' and V'' contexts take the next ones
        x.amax = i ? kv_amax() : kv_reuse ? (e.dry() ? reinterpret_cast<float*>((uintptr_t)0x100) : n.ctxkv.amax) : e.amax_slot();
        if (!kv_hit) amax_rows(e, x.src, (long long)B * L, c.context_dim, c.context_dim, x.amax, s);
        if (e.mma_mode != 1 || !e.flash_attn) continue;
        float* pad = (float*)e.arena.alloc((size_t)B * ctx_lp * D * sizeof(float));
        if (!e.dry() && !kv_hit) {
          if (ctx_lp != L) CDX_CUDA(cudaMemsetAsync(pad, 0, (size_t)B * ctx_lp * D * sizeof(float), s));
          CDX_CUDA(cudaMemcpy2DAsync(pad, (size_t)ctx_lp * D * 4, x.src, (size_t)L * D * 4, (size_t)L * D * 4, B, cudaMemcpyDeviceToDevice, s));
        }
        x.pad = pad;
      }
    }
    // --- timestep embedding MLP + all ResBlock emb projections in one GEMM
    Tensor temb = alloc(B, 1, 1, mc);
    timestep_embedding(e, t_dev, n.freqs_dev, temb.p, B, half, s);
    Tensor e1 = linear(temb, "time_embed.0", true);
    silu(e, e1.p, e1.p, e1.numel(), s);
    Tensor emb = linear(e1, "time_embed.2", true);
    silu(e, emb.p, emb.p, emb.numel(), s);   // every consumer applies SiLU first (OAI:219, IU:205)
    Tensor Eall = alloc(B, 1, 1, n.emb_rows);
    linear_into(emb.p, ted, ted, nullptr, 0, 0, B, n.blob + n.emb_w_off, n.emb_rows, n.blob + n.emb_b_off, nullptr, 0, Eall.p, n.emb_rows);
    E = Eall.p;

    Tensor xin = alloc(B, H, W, c.in_channels);
    nchw_to_nhwc(e, x_nchw, xin.p, B, c.in_channels, H * W, s);

    std::vector<Tensor> hs;
    Tensor h = conv3(xin, "input_blocks.0.0");
    hs.push_back(h);
    int ds = 1, bi = 1;
    for (int level = 0; level < c.n_mult; ++level) {
      for (int r = 0; r < c.num_res_blocks; ++r) {
        const std::string bp = S("input_blocks.", bi);
        h = resblock(h, nullptr, bp + ".0");
        if (contains(c.attention_ds, c.n_attn, ds)) h = attn_layer(h, bp + ".1");
        hs.push_back(h);
        ++bi;
      }
      if (level != c.n_mult - 1) {
        const std::string bp = S("input_blocks.", bi);
        if (oai) h = conv3(h, bp + ".0.op", 2, 1);
        else h = resblock(h, nullptr, bp + ".0", 1);
        hs.push_back(h);
        ++bi;
        ds *= 2;
      }
    }
    h = resblock(h, nullptr, "middle_block.0");
    h = attn_layer(h, "middle_block.1");
    h = resblock(h, nullptr, "middle_block.2");
    int bo = 0;
    for (int level = c.n_mult - 1; level >= 0; --level) {
      for (int i = 0; i <= c.num_res_blocks; ++i) {
        const Tensor skip = hs.back();
        hs.pop_back();
        const std::string bp = S("output_blocks.", bo);
        h = resblock(h, &skip, bp + ".0", 0, feature_row(bo));
        int li = 1;
        if (contains(c.attention_ds, c.n_attn, ds)) { h = attn_layer(h, bp + "." + std::to_string(li)); ++li; }
        if (level && i == c.num_res_blocks) {
          if (oai) h = conv3(h, bp + "." + std::to_string(li) + ".conv", 1, 1, 2);
          else h = resblock(h, nullptr, bp + "." + std::to_string(li), 2);
          ds /= 2;
        }
        ++bo;
      }
    }
    gn_silu_conv3(h, nullptr, "out.0", 1e-5f, "out.2", nullptr, nullptr, 0, nullptr, 0, nullptr, nullptr, out_nchw);
  }
};

// ------------------------------------------------------------------------------------------------ VAE
struct VaeExec : Exec {
  VaeExec(Net& net, cudaStream_t st) : Exec(net, st) {}

  Tensor resnet(const Tensor& x, const std::string& p) {
    const int Cout = n.dim0(p + ".conv1.weight");
    Tensor out = alloc(x.B, x.H, x.W, Cout);
    Scope sc(e.arena);
    Tensor h2 = gn_silu_conv3(x, nullptr, p + ".norm1", 1e-6f, p + ".conv1");
    const float* residual = x.p;
    if (n.has(p + ".nin_shortcut.weight")) {
      Tensor sk = linear(x, p + ".nin_shortcut", true);
      residual = sk.p;
    }
    gn_silu_conv3(h2, nullptr, p + ".norm2", 1e-6f, p + ".conv2", nullptr, nullptr, 0, nullptr, 0, residual, &out);
    return out;
  }

  void encode(const float* img_nchw, float* moments_nchw, int B, int H, int W) {
    const cdx_vae_config& c = n.vcfg;
    Scope top(e.arena);
    e.pools_reset(s);
    const std::string E = "encoder.";
    Tensor xin = alloc(B, H, W, c.in_channels);
    nchw_to_nhwc(e, img_nchw, xin.p, B, c.in_channels, H * W, s);
    Tensor h = conv3(xin, E + "conv_in");
    for (int lvl = 0; lvl < c.n_mult; ++lvl) {
      for (int b = 0; b < c.num_res_blocks; ++b) h = resnet(h, E + "down." + std::to_string(lvl) + ".block." + std::to_string(b));
      if (lvl != c.n_mult - 1) h = conv3(h, E + "down." + std::to_string(lvl) + ".downsample.conv", 2, 0);   // pad (0,1,0,1), AEM:72-76
    }
    h = resnet(h, E + "mid.block_1");
    h = attn(h, E + "mid.attn_1");
    h = resnet(h, E + "mid.block_2");
    Tensor m = gn_silu_conv3(h, nullptr, E + "norm_out", 1e-6f, E + "conv_out");
    Tensor q = linear(m, "quant_conv", true);
    nhwc_to_nchw(e, q.p, moments_nchw, B, q.C, q.H * q.W, s);
  }

  void decode(const float* z_nchw, float* img_nchw, int B, int hsz, int wsz) {
    const cdx_vae_config& c = n.vcfg;
    Scope top(e.arena);
    e.pools_reset(s);
    const std::string D = "decoder.";
    Tensor zin = alloc(B, hsz, wsz, c.embed_dim);
    nchw_to_nhwc(e, z_nchw, zin.p, B, c.embed_dim, hsz * wsz, s);
    if (c.vq) {       // VQModelInterface.decode: quantise first (autoencoder.py:272-281)
      Tensor zq = alloc(B, hsz, wsz, c.embed_dim);
      vq_quantize(e, zin.p, n.P("quantize.embedding.weight"), zq.p, (size_t)B * hsz * wsz, c.embed_dim, c.n_embed, s);
      zin = zq;
    }
    Tensor h = linear(zin, "post_quant_conv", true);
    h = conv3(h, D + "conv_in");
    h = resnet(h, D + "mid.block_1");
    h = attn(h, D + "mid.attn_1");
    h = resnet(h, D + "mid.block_2");
    for (int lvl = c.n_mult - 1; lvl >= 0; --lvl) {
      for (int b = 0; b <= c.num_res_blocks; ++b) h = resnet(h, D + "up." + std::to_string(lvl) + ".block." + std::to_string(b));
      if (lvl != 0) h = conv3(h, D + "up." + std::to_string(lvl) + ".upsample.conv", 1, 1, 2);
    }
    gn_silu_conv3(h, nullptr, D + "norm_out", 1e-6f, D + "conv_out", nullptr, nullptr, 0, nullptr, 0, nullptr, nullptr, img_nchw);
  }
};

}  // namespace

void unet_forward(Net& n, const float* x_nchw, const float* t_dev, const float* ctx, int ctx_len, float* out_nchw, int B, int H, int W,
                  cudaStream_t s, bool reuse_ctx, const AttnControl* ctl, const AttnProbe* probe) {
  CDX_CHECK(n.kind == NET_UNET_OPENAI || n.kind == NET_UNET_IDDPM || n.kind == NET_UNET_DDPM, "unet_forward on a non-U-Net");
  CDX_CHECK(n.finalized, "unet_forward before finalize");
  if (n.kind == NET_UNET_OPENAI && n.ucfg.context_dim > 0) CDX_CHECK(ctx != nullptr && ctx_len > 0, "unet_forward: the SD/LDM U-Net needs a context");
  const int down = 1 << (n.ucfg.n_mult - 1);
  CDX_CHECK(H % down == 0 && W % down == 0, "unet_forward: %dx%d not divisible by %d", H, W, down);
  UNetExec ex(n, s);
  ex.kv_reuse = reuse_ctx && n.kind == NET_UNET_OPENAI && n.ucfg.context_dim > 0;
  CDX_CHECK(!ctl || (!ctl->qk_row && !ctl->kv_row && !ctl->pnp_row) || (n.kind == NET_UNET_OPENAI && n.ucfg.context_dim > 0 && ctx_len > 0),
            "attention control: SD / LDM U-Nets with a context only");
  CDX_CHECK(!ctl || (!!ctl->qk_row + !!ctl->kv_row + !!ctl->pnp_row) <= 1,
            "attention control: Prompt-to-Prompt, mutual self-attention and Plug-and-Play are exclusive in one call");
  ex.ctl = ctl;
  CDX_CHECK(!probe || (n.kind == NET_UNET_OPENAI && n.ucfg.context_dim > 0 && ctx_len > 0 && probe->rows && !probe->span != !probe->weights && probe->map &&
                       probe->n_rows >= 1 && probe->tokens >= 1),
            "attention probe: SD / LDM U-Nets with a context, and a row list, spans or weights and a map");
  ex.probe = probe;
  if (n.kind == NET_UNET_DDPM) { ex.forward_ddpm(x_nchw, t_dev, out_nchw, B, H, W); return; }
  ex.forward(x_nchw, t_dev, ctx, ctx_len, out_nchw, B, H, W);
  CDX_CHECK(!probe || ex.probed > 0, "attention probe: no cross-attention of %d tokens in the input or output blocks (a %dx%d latent)",
            probe->tokens, H, W);
  if (ex.kv_reuse && !n.eng->dry()) {
    n.ctxkv.valid = true;
    n.ctxkv.ctx = ctx; n.ctxkv.ctx_v = ctl ? ctl->ctx_v : nullptr; n.ctxkv.ctx_w = ctl ? ctl->ctx_w : nullptr; n.ctxkv.L = ctx_len; n.ctxkv.B = B;
  }
}

// CLIPEncoderLayer stack (HF modeling_clip.py; OpenAI clip ResidualAttentionBlock): pre-LN, self-attention (q scaled by d^-1/2; causal
// for the text tower), quick-GELU MLP (exact-erf GELU for the OpenCLIP tower).  x [B, L, W] -> returns the last layer's output tensor.
static Tensor clip_layers(Exec& ex, Net& n, const std::string& prefix, Tensor x, int B, int L, int W, int heads, int layers, int mlp_width,
                          bool causal, cudaStream_t s, bool erf_gelu = false) {
  Engine& e = *n.eng;
  const int d = W / heads;
  const float scale = (float)pow((double)d, -0.5);
  for (int l = 0; l < layers; ++l) {
    const std::string p = prefix + "encoder.layers." + std::to_string(l);
    Tensor y = ex.alloc(B, L, 1, W);          // layer output (outlives the layer's temporaries)
    {
      Scope sc(e.arena);
      Tensor n1 = ex.ln(x, p + ".layer_norm1");
      Tensor q = ex.linear(n1, p + ".self_attn.q_proj", true);
      Tensor k = ex.linear(n1, p + ".self_attn.k_proj", true);
      Tensor v = ex.linear(n1, p + ".self_attn.v_proj", true, nullptr, true);
      Tensor a = ex.alloc(B, L, 1, W);
      a.amax = v.amax;
      attention(e, q.p, W, k.p, W, v.p, W, a.p, W, B, L, L, heads, d, d, scale, s, causal);
      Tensor h = ex.linear(a, p + ".self_attn.out_proj", true, x.p);                 // + residual
      Tensor n2 = ex.ln(h, p + ".layer_norm2");
      Tensor f = ex.linear(n2, p + ".mlp.fc1", true, nullptr, true);
      if (erf_gelu) gelu(e, f.p, f.p, f.numel(), s);    // |gelu(x)| <= |x|
      else quick_gelu(e, f.p, f.p, f.numel(), s);      // |x sigmoid(1.702 x)| <= |x|
      const Param& w2 = n.param(p + ".mlp.fc2.weight");
      ex.linear_into(f.p, mlp_width, mlp_width, nullptr, 0, 0, B * L, n.blob + w2.off, W, n.P(p + ".mlp.fc2.bias"), h.p, W, y.p, W, nullptr, f.amax);
    }
    x = y;
  }
  return x;
}

// CLIPTextTransformer.forward (HF modeling_clip.py; call site ldm/modules/encoders/modules.py:152-157): embeddings, pre-LN
// encoder layers with causal self-attention (q scaled by d^-1/2) and quick-GELU MLP, final LayerNorm -> last_hidden_state
void text_encode(Net& n, const int* ids, float* out, int B, int L, cudaStream_t s) {
  CDX_CHECK(n.kind == NET_CLIP_TEXT && n.finalized, "text_encode: not a finalized text encoder");
  const cdx_text_config& c = n.tcfg;
  CDX_CHECK(L >= 1 && L <= c.max_len, "text_encode: %d tokens, the position table has %d", L, c.max_len);
  Exec ex(n, s);
  Engine& e = *n.eng;
  e.pools_reset(s);
  if (c.kind == CDX_TEXT_XTRANSFORMER) {
    // TransformerWrapper.forward(return_embeddings=True) (x_transformer.py:598-626) over AttentionLayers.forward (481-523):
    // x = tok + pos; per layer x += to_out(softmax(q k^T d^-1/2) v) of LN(x), x += W2 gelu(W1 LN(x)); final LN
    const int W = c.width, inner = c.heads * c.dim_head;
    const std::string T = "transformer.";
    Scope top(e.arena);
    Tensor x = ex.alloc(B, L, 1, W);
    embed_tokens(e, ids, n.P(T + "token_emb.weight"), n.P(T + "pos_emb.emb.weight"), x.p, B, L, W, c.vocab_size, s);
    const float scale = (float)pow((double)c.dim_head, -0.5);
    for (int l = 0; l < c.layers; ++l) {
      const std::string pa = T + "attn_layers.layers." + std::to_string(2 * l), pf = T + "attn_layers.layers." + std::to_string(2 * l + 1);
      Tensor y = ex.alloc(B, L, 1, W);
      {
        Scope sc(e.arena);
        Tensor n1 = ex.ln(x, pa + ".0");
        Tensor q = ex.linear(n1, pa + ".1.to_q", false);
        Tensor k = ex.linear(n1, pa + ".1.to_k", false);
        Tensor v = ex.linear(n1, pa + ".1.to_v", false, nullptr, true);
        Tensor a = ex.alloc(B, L, 1, inner);
        a.amax = v.amax;                              // |softmax-weighted mean of V rows| <= max |V|
        attention(e, q.p, inner, k.p, inner, v.p, inner, a.p, inner, B, L, L, c.heads, c.dim_head, c.dim_head, scale, s, false);
        Tensor h = ex.linear(a, pa + ".1.to_out", true, x.p);                         // + residual
        Tensor n2 = ex.ln(h, pf + ".0");
        Tensor f = ex.linear(n2, pf + ".1.net.0.0", true, nullptr, true);
        gelu(e, f.p, f.p, f.numel(), s);                 // |gelu(x)| <= |x|: the tracked range stays valid
        const Param& w2 = n.param(pf + ".1.net.2.weight");
        ex.linear_into(f.p, c.mlp_width, c.mlp_width, nullptr, 0, 0, B * L, n.blob + w2.off, W, n.P(pf + ".1.net.2.bias"), h.p, W, y.p, W, nullptr, f.amax);
      }
      x = y;
    }
    layernorm(e, x.p, n.P(T + "norm.weight"), n.P(T + "norm.bias"), out, B * L, W, s);
    return;
  }
  const int W = c.width;
  const std::string T = "text_model.";
  Scope top(e.arena);
  Tensor x = ex.alloc(B, L, 1, W);
  embed_tokens(e, ids, n.P(T + "embeddings.token_embedding.weight"), n.P(T + "embeddings.position_embedding.weight"), x.p, B, L, W, c.vocab_size, s);
  x = clip_layers(ex, n, T, x, B, L, W, c.heads, c.layers, c.mlp_width, true, s, c.kind == CDX_TEXT_OPENCLIP);
  // final LayerNorm straight into the caller's buffer
  layernorm(e, x.p, n.P(T + "final_layer_norm.weight"), n.P(T + "final_layer_norm.bias"), out, B * L, W, s);
}

// CLIP.encode_text (clip/model.py:343-356; call site clean_clip.py:24-27): x[arange(B), text.argmax(-1)] of the final-LN states, then
// @ text_projection
void text_features(Net& n, const int* ids, float* out, int B, int L, cudaStream_t s) {
  CDX_CHECK(n.kind == NET_CLIP_TEXT && n.finalized && n.tcfg.kind != CDX_TEXT_XTRANSFORMER && n.tcfg.kind != CDX_CLIP_VISION && n.tcfg.proj_dim > 0,
            "text_features: needs a CLIP text tower built with proj_dim > 0");
  Engine& e = *n.eng;
  const int W = n.tcfg.width;
  Scope top(e.arena);
  float* hs = (float*)e.arena.alloc((size_t)B * L * W * sizeof(float));
  int* rows = (int*)e.arena.alloc((size_t)B * sizeof(int));
  text_encode(n, ids, hs, B, L, s);
  eot_rows(e, ids, rows, B, L, s);
  Exec ex(n, s);
  Tensor pooled = ex.alloc(B, 1, 1, W);
  gather_rows(e, hs, rows, pooled.p, B, L, W, s);
  ex.linear_into(pooled.p, W, W, nullptr, 0, 0, B, n.P("text_projection.weight"), n.tcfg.proj_dim, nullptr, nullptr, 0, out, n.tcfg.proj_dim);
}

// CLIP.encode_image (clip/model.py VisionTransformer.forward; call site clean_clip.py:28-31): patch embedding as one GEMM, class token
// + positions, ln_pre, the layer stack (full attention), ln_post of the class token, @ proj.  pixels [B,3,S,S] already preprocessed.
void clip_image_features(Net& n, const float* pixels, float* out, int B, cudaStream_t s) {
  CDX_CHECK(n.kind == NET_CLIP_TEXT && n.finalized && n.tcfg.kind == CDX_CLIP_VISION, "clip_image_features: not a finalized CLIP vision tower");
  const cdx_text_config& c = n.tcfg;
  Engine& e = *n.eng;
  e.pools_reset(s);
  Exec ex(n, s);
  const int W = c.width, P = c.patch, S = c.image_size, np = S / P, N = np * np, K = 3 * P * P;
  const std::string V = "vision_model.";
  Scope top(e.arena);
  float* pm = (float*)e.arena.alloc((size_t)B * N * K * sizeof(float));
  patchify(e, pixels, pm, B, S, P, s);
  float* pe = (float*)e.arena.alloc((size_t)B * N * W * sizeof(float));
  ex.linear_into(pm, K, K, nullptr, 0, 0, B * N, n.P(V + "embeddings.patch_embedding.weight"), W, nullptr, nullptr, 0, pe, W);
  Tensor x = ex.alloc(B, N + 1, 1, W);
  vit_tokens(e, pe, n.P(V + "embeddings.class_embedding"), n.P(V + "embeddings.position_embedding.weight"), x.p, B, N, W, s);
  Tensor x1 = ex.ln(x, V + "pre_layrnorm");
  Tensor y = clip_layers(ex, n, V, x1, B, N + 1, W, c.heads, c.layers, c.mlp_width, false, s);
  Tensor cls = ex.alloc(B, 1, 1, W);
  gather_rows(e, y.p, nullptr, cls.p, B, N + 1, W, s);
  Tensor pooled = ex.ln(cls, V + "post_layernorm");
  ex.linear_into(pooled.p, W, W, nullptr, 0, 0, B, n.P("visual_projection.weight"), c.proj_dim, nullptr, nullptr, 0, out, c.proj_dim, nullptr, pooled.amax);
}

void vae_encode(Net& n, const float* img, float* moments, int B, int H, int W, cudaStream_t s) {
  CDX_CHECK(n.kind == NET_VAE && n.finalized, "vae_encode: not a finalized VAE");
  const int down = 1 << (n.vcfg.n_mult - 1);
  CDX_CHECK(H > 0 && W > 0 && H % down == 0 && W % down == 0, "vae_encode: image %dx%d, both sides must be multiples of %d", H, W, down);
  VaeExec ex(n, s);
  ex.encode(img, moments, B, H, W);
}

void vae_decode(Net& n, const float* z, float* img, int B, int h, int w, cudaStream_t s) {
  CDX_CHECK(n.kind == NET_VAE && n.finalized, "vae_decode: not a finalized VAE");
  CDX_CHECK(h > 0 && w > 0, "vae_decode: latent %dx%d", h, w);
  VaeExec ex(n, s);
  ex.decode(z, img, B, h, w);
}

}  // namespace cdx
