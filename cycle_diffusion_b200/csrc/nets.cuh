// nets.cuh -- network objects: parameter inventory, packed weight blob, forward executors.
#pragma once
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"

namespace cdx {

struct Param {
  std::string name;
  int64_t dims[4] = {0, 0, 0, 0};
  int rank = 0;
  size_t numel = 0;
  size_t off = 0;        // float offset into the blob
  int segment = 0;       // 0 general, 1 emb-proj weights (concatenated), 2 emb-proj biases (concatenated)
  bool conv3 = false;    // stored repacked O,kh,kw,I
  int cin_pad = 0;       // 3x3 conv with < 32 input channels: stored with Cin zero-padded to this (tensor-core K blocks are 32 wide)
  size_t store() const { return cin_pad ? (size_t)dims[0] * 9 * cin_pad : numel; }   // floats occupied in the blob
  bool geglu = false;    // GEGLU projection: rows stored as alternating blocks of 32 value rows | their 32 gate rows
  bool loaded = false;
};

enum NetKind { NET_UNET_OPENAI = 1, NET_UNET_IDDPM = 2, NET_VAE = 3, NET_CLIP_TEXT = 4, NET_UNET_DDPM = 5 };

struct Net {
  Engine* eng = nullptr;
  int kind = 0;
  cdx_unet_config ucfg{};
  cdx_vae_config vcfg{};
  cdx_text_config tcfg{};
  std::vector<Param> params;
  std::unordered_map<std::string, int> index;
  float* blob = nullptr;
  float* blob_hi = nullptr;     // rn_tf32(blob)            } pre-split planes for the TF32-plane (KIND_TS) kernel,
  float* blob_lo = nullptr;     // rn_tf32(blob - blob_hi)  } same offsets as `blob`, derived at finalize
  bool planes_valid = false;
  // fp16-split planes (MODE_H16): hi = fp16(w * 2^w_exp), lo = fp16(w * 2^w_exp - hi), element index = float index into `blob`;
  // w_exp from the largest |weight| of the GEMM operands (rank >= 2 parameters) so that every scaled weight is < 2^15
  void* blob_h_hi = nullptr;
  void* blob_h_lo = nullptr;
  int w_exp = 0;
  size_t blob_floats = 0;
  bool finalized = false;
  // output parameterisation of an SD U-Net (cdx_unet_set_prediction): 0 eps, 1 v with sqrt(abar_t) / sqrt(1 - abar_t) per timestep t
  int pred = 0;
  std::vector<float> sa_v, s1_v;
  // timestep embedding
  std::vector<float> freqs_host;
  float* freqs_dev = nullptr;
  // cross-attention K / V of a context that stays fixed over a sampling loop (set up by the loop drivers in cabi.cu):
  // computed by the first U-Net call of the loop, reused by the others (the reference recomputes them every step)
  struct CtxKV {
    static constexpr int MAX_LAYERS = 127;   // range slots after [0] (up to four per layer under refine control)
    bool valid = false; const float* ctx = nullptr; const float* ctx_v = nullptr; const float* ctx_w = nullptr; int L = 0, B = 0;
    float* buf = nullptr; size_t cap = 0;
    // [0]: max |context|, then per layer max |K, V| of its context projection and, with a V context (AttnControl::ctx_v), max |V'|;
    // with a refine context (AttnControl::ctx_w) also max |V''| and the bound of the output (see UNetExec)
    float* amax = nullptr;
  } ctxkv;
  // concatenated ResBlock emb projections: weights [emb_rows][ted] at emb_w_off, biases at emb_b_off
  size_t emb_w_off = 0, emb_b_off = 0;
  int emb_rows = 0, ted = 0;
  std::unordered_map<std::string, int> emb_off;   // ResBlock prefix -> row offset

  const Param& param(const std::string& name) const;
  float* P(const std::string& name) const { return blob + param(name).off; }
  bool has(const std::string& name) const { return index.find(name) != index.end(); }
  int dim0(const std::string& name) const { return (int)param(name).dims[0]; }
};

Net* make_unet(Engine* e, const cdx_unet_config& cfg);
Net* make_vae(Engine* e, const cdx_vae_config& cfg);
Net* make_text(Engine* e, const cdx_text_config& cfg);
void destroy_net(Net* n);
void net_load_param(Net& n, const char* name, const float* data, bool on_device, const int64_t* dims, int rank);
void net_finalize(Net& n);
void net_ensure_blob(Net& n);

// side outputs of a GEMM that writes tensor t: its range slot (for a consumer fp16-split GEMM) and, with `stats`, its per-(image,
// channel) sums (for a consumer GroupNorm) -- both produced by the epilogue that holds the tile in registers where it can
void track_outputs(Engine& e, Tensor& t, GemmArgs& g, bool stats);

// Attention control of one SD / LDM U-Net call (Prompt-to-Prompt's "replace" and "refine" edits, driven by the lock-step loop in cabi.cu).
// Row r's fused attention takes its Q and K from row qk_row[r], so its probabilities are that row's; its V stays its own.  Only the
// fused kernels can do this: a layer that would take another route while control is on is an error.
struct AttnControl {
  const int* qk_row = nullptr;          // device [B]; null: no control
  bool cross = false;                   // remap the cross-attention layers in this call
  bool self = false;                    // remap the self-attention layers of at most self_max_tokens tokens in this call
  int self_max_tokens = 0;
  // optional device [B, L, D]: the context the cross-attention V' is projected from (a controlled row holds A_b . c_tgt[b], every
  // other row its own context).  Given, the context cache also holds V'^T (own range slot), and cross-controlled calls read it
  // instead of V^T.  Fixed over the loop, like the context
  const float* ctx_v = nullptr;
  // refine (optional): the context of the second term, device [B, L, D] (a controlled row holds diag(w_b) . c_tgt[b], every other
  // row zeros), and the controlled rows, device [n_own].  Given, the context cache also holds V''^T (own range slot) and the
  // range slot of the sum, and every cross-controlled layer adds softmax(Q K^T) . V'' of those rows into its output
  const float* ctx_w = nullptr;
  const int* own_rows = nullptr;
  int n_own = 0;
  // mutual self-attention (MasaCtrl; exclusive with qk_row): with `mutual`, the self-attention of every SpatialTransformer whose
  // index in forward order (input blocks, middle block, output blocks) is >= start_layer takes row r's K and V from row kv_row[r]
  const int* kv_row = nullptr;          // device [B]
  bool mutual = false;                  // control the self-attention layers >= start_layer in this call
  int start_layer = 0;
  // Plug-and-Play (Tumanyan et al., 2023; exclusive with qk_row and kv_row).  With `pnp_feat`, the ResBlock output_blocks.k.0 of
  // each k in feat_blocks normalises row pnp_row[r]'s out_layers input on row r (so its conv adds row r's own skip to row
  // pnp_row[r]'s out_layers); with `pnp_attn`, the self-attention of every SpatialTransformer whose index in forward order is
  // >= pnp_layer takes row r's Q and K from row pnp_row[r] and keeps its own V
  const int* pnp_row = nullptr;         // device [B]
  bool pnp_feat = false;                // control the ResBlocks of feat_blocks in this call
  const int* feat_blocks = nullptr;     // host [n_feat]: output-block indices
  int n_feat = 0;
  bool pnp_attn = false;                // control the self-attention layers >= pnp_layer in this call
  int pnp_layer = 0;
};

// Cross-attention probe of one SD / LDM U-Net call (LEDITS++'s implicit masks, driven by the semantic-guidance loop in cabi.cu).  It
// changes no output: the cross-attention of every SpatialTransformer in the input and output blocks (never the middle block) whose
// token count is `tokens` also runs attn_probe on the operands its route multiplied, for the listed rows: the first such layer
// stores map [n_rows, tokens], later ones add.  A call in which no layer matches is an error.  LocalBlend's loop gives weights
// instead of span: entry i's map is then sum_j weights[i, j] * softmax_j of row rows[i].
struct AttnProbe {
  const int* rows = nullptr;            // device [n_rows]: U-Net rows
  const int* span = nullptr;            // device [n_rows]: tokens 1..span[i] of row i's context
  const float* weights = nullptr;       // device [n_rows, L], exclusive with span
  int n_rows = 0;
  float* map = nullptr;                 // device [n_rows, tokens]
  int tokens = 0;
};

// forward executors (enqueue only; caller handles arena dry-run)
// reuse_ctx: the caller guarantees `ctx` is unchanged since the previous call with reuse_ctx (and n.ctxkv was invalidated
// at the start of the loop) -> context K / V projections are taken from n.ctxkv instead of being recomputed
void unet_forward(Net& n, const float* x_nchw, const float* t_dev, const float* ctx, int ctx_len, float* out_nchw, int B, int H,
                  int W, cudaStream_t s, bool reuse_ctx = false, const AttnControl* ctl = nullptr, const AttnProbe* probe = nullptr);void vae_encode(Net& n, const float* img_nchw, float* moments_nchw, int B, int H, int W, cudaStream_t s);
void vae_decode(Net& n, const float* z_nchw, float* img_nchw, int B, int h, int w, cudaStream_t s);
void text_encode(Net& n, const int* ids, float* out, int B, int L, cudaStream_t s);
void text_features(Net& n, const int* ids, float* out, int B, int L, cudaStream_t s);                // CLIP.encode_text   -> [B, proj_dim]
void clip_image_features(Net& n, const float* pixels, float* out, int B, cudaStream_t s);            // CLIP.encode_image  -> [B, proj_dim]

}  // namespace cdx
