// common.cuh -- engine-wide declarations: error plumbing, workspace arena, tensor views, op prototypes.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>
#include <stdexcept>

#include "../../include/cdx.h"

namespace cdx {

// ------------------------------------------------------------------------------------------------
// errors: C++ exceptions inside the library, translated to CDX_E_* + thread-local message at the ABI
// ------------------------------------------------------------------------------------------------
struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
void set_last_error(const std::string& m);

#define CDX_CHECK(cond, ...)                                                     \
  do {                                                                           \
    if (!(cond)) {                                                               \
      char _b[512];                                                              \
      snprintf(_b, sizeof(_b), __VA_ARGS__);                                     \
      throw ::cdx::Error(CDX_E_INVALID, std::string(_b) + " [" #cond "]");       \
    }                                                                            \
  } while (0)

#define CDX_CUDA(expr)                                                                         \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      char _b[512];                                                                            \
      snprintf(_b, sizeof(_b), "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      throw ::cdx::Error(CDX_E_CUDA, _b);                                                      \
    }                                                                                          \
  } while (0)

// ------------------------------------------------------------------------------------------------
// workspace arena: stack (mark/release) allocator over one device slab, sized by a dry run of the call.
// All work of an engine is enqueued on a single stream, so memory released to the stack can be reused
// by later launches without extra synchronisation.
// ------------------------------------------------------------------------------------------------
struct Arena {
  char* base = nullptr;
  size_t cap = 0, off = 0, high = 0;
  bool dry = false;
  void* alloc(size_t bytes);
  size_t mark() const { return off; }
  void release(size_t m) { off = m; }
  void begin_dry();   // start a sizing pass: allocations only advance the offset
  void end_dry();     // grow the slab to the recorded high-water mark, rewind
  void destroy();
};

// per-kernel-family timing with CUDA events on the launching stream (bench.py's roofline numbers)
enum ProfTag {
  PROF_CONV_FFMA = 0, PROF_DENSE_FFMA = 1, PROF_BATCHED_FFMA = 2, PROF_CONV_TC = 3, PROF_DENSE_TC = 4, PROF_BATCHED_TC = 5,
  PROF_GROUPNORM = 6, PROF_LAYERNORM = 7, PROF_SOFTMAX = 8, PROF_ELEMENTWISE = 9, PROF_NTAGS = 10
};
struct ProfRec { cudaEvent_t a, b; int tag; double flops, bytes; int launches; char note[56]; };
struct Profiler {
  bool on = false;
  std::vector<ProfRec> recs;
  std::vector<cudaEvent_t> pool;
};

struct Engine {
  Profiler prof;
  int device = 0;
  int num_sms = 132;
  bool flash_attn = true;        // fused wgmma attention kernel (kernels_attn.cu); false -> unfused QK^T / softmax / PV
  int mma_mode = 1;              // 0 SIMT FFMA (exact fp32), 1 tensor cores (wgmma)
  int tc_kind = 1;               // tensor-core product scheme: 0 3xTF32, 1 3x fp16-split at the f16 rate (default), 2 1x fp16 (fast, not fp32-faithful)
  bool attn_one = false;         // mode 5 ("autocast"): fused fp16 attention with one product term on hi planes only (no lo planes written)
  bool persist = true;           // persistent tensor-core GEMM for unsplit dense fp16-split work (CDX_PERSIST=0 at creation: one CTA per item)
  int persist_grid = 0;          // > 0: at most this many persistent CTAs (tests: one CTA walks many work items); 0: one per SM
  // tracked |max| scalars of activation tensors (operand range of the fp16-split GEMMs): a pool of device floats, handed out
  // per tensor by the graph executors and zeroed at the start of every network call
  float* amax_pool = nullptr;
  int amax_cap = 1 << 15, amax_used = 0, amax_high = 0;
  float* amax_slot();
  // per-(image, channel) fp64 statistics buffers of activation tensors (GroupNorm inputs), same life cycle as the amax slots
  double* stat_pool = nullptr;
  size_t stat_cap = (size_t)8 << 20, stat_used = 0, stat_high = 0;      // doubles (64 MB)
  size_t stat_dry = 0;      // doubles the sizing passes have asked for, ever: a driver checks one call's share against stat_cap
  double* stat_alloc(size_t n);
  void pools_reset(cudaStream_t s);   // start of a network call: zero what the previous call dirtied, rewind
  Arena arena;
  cudaStream_t last_stream = nullptr;   // stream of the previous arena-using call and the event recorded at its end
  cudaEvent_t done_ev = nullptr;
  bool ev_recorded = false;
  // second stream (non-blocking, created on first use) on which the two-model loops run this engine's U-Net calls when the other
  // chain's net lives in another engine; fork / join events order it against the caller's stream once per step
  cudaStream_t side = nullptr;
  cudaEvent_t fork_ev = nullptr, join_ev = nullptr;
  uint64_t launches = 0;
  bool dry() const { return arena.dry; }
};

// RAII: time everything enqueued between construction and destruction under one tag (no-op unless profiling)
struct ProfScope {
  Engine& e;
  cudaStream_t s;
  int idx = -1;
  ProfScope(Engine& eng, cudaStream_t st, int tag, double flops, double bytes, int launches);
  ~ProfScope();
  void note(const char* fmt, ...);     // free-form shape note, printed per launch when CDX_PROF_DUMP is set
};

struct Scope {   // RAII arena scope
  Arena& a;
  size_t m;
  explicit Scope(Arena& ar) : a(ar), m(ar.mark()) {}
  ~Scope() { a.release(m); }
};

// NHWC activation view: p[((b*H + y)*W + x)*C + c]; a [M,C] token matrix is H=M/B, W=1.
struct Tensor {
  float* p = nullptr;
  int B = 0, H = 0, W = 0, C = 0;
  float* amax = nullptr;      // device scalar >= max |element| (maintained by the producing kernel), or null when not tracked
  double* stats = nullptr;    // per-(image, channel) fp64 {sum, sum of squares} accumulated by the producing kernel, or null
  size_t numel() const { return (size_t)B * H * W * C; }
  int rows() const { return B * H * W; }
};
inline Tensor alloc_tensor(Engine& e, int B, int H, int W, int C) {
  Tensor t;
  t.B = B; t.H = H; t.W = W; t.C = C;
  t.p = (float*)e.arena.alloc(t.numel() * sizeof(float));
  return t;
}

// ------------------------------------------------------------------------------------------------
// dense contraction (implicit GEMM) arguments, shared by the SIMT and wgmma back ends
//   C[m,n] = alpha * sum_k A(m,k) * W(n,k)  (+ bias[n]) (+ rowvec[m / rows_per_batch, n]) (+ residual[m,n])
// A is either a dense row matrix (two channel-concatenated sources allowed) or the implicit im2col of
// a 3x3 convolution over an NHWC tensor (k = tap*Cin + c).
// ------------------------------------------------------------------------------------------------
struct GemmArgs {
  int M = 0, N = 0, K = 0;
  int mode = 0;                       // 0 dense rows, 1 conv3x3 gather
  const float* A = nullptr;  int lda = 0;  int C1 = 0;   // first source: C1 channels, row/pixel stride lda
  const float* A2 = nullptr; int lda2 = 0; int C2 = 0;   // optional second source (channel concat; dense mode only)
  // conv geometry (mode 1): stored input [B,Hin,Win,*], logical input is up x larger (nearest)
  int Hin = 0, Win = 0, Hout = 0, Wout = 0, stride = 1, pad = 1, up = 1;
  const float* Bw = nullptr; int ldb = 0; int b_kn = 0;   // weights [N][K] (b_kn=0) or [K][N] (b_kn=1)
  const float* Bw_hi = nullptr; const float* Bw_lo = nullptr;   // optional pre-split TF32 planes of Bw (same geometry)
  // optional fp16-split planes of Bw, pre-scaled by 2^b_exp (same geometry, element index = float index), and the tracked max |A|
  // scalars (device) of the A operand(s); c_amax: device scalar that receives max |C| (atomic max) for a consumer GEMM
  const void* Bw_h_hi = nullptr; const void* Bw_h_lo = nullptr; int b_exp = 0;
  const float* a_amax = nullptr; const float* a2_amax = nullptr;
  float* c_amax = nullptr;
  double* c_stats = nullptr;         // optional: += per-(image, channel) {sum, sum sq} of C (rows_per_batch rows per image), zeroed by the caller
  float* Cout = nullptr; int ldc = 0;
  float* Cout_lo = nullptr;           // if set: Cout receives rn_tf32(C) and Cout_lo rn_tf32(C - hi) (operand planes for the tensor-core kernels)
  // optional: columns n >= t_col0 are stored TRANSPOSED as TF32 planes, Ct_hi / Ct_lo [(n - t_col0) * ldt + m] (dense mode,
  // no split-K): the value projection of a fused q|k|v GEMM lands directly as the K-major V^T operand of the attention kernel
  float* Ct_hi = nullptr; float* Ct_lo = nullptr; int t_col0 = 0; long long ldt = 0;
  const float* bias = nullptr;
  const float* rowvec = nullptr; int ld_rowvec = 0; int rows_per_batch = 1;
  const float* residual = nullptr; int ldr = 0;
  float alpha = 1.f;
  int geglu = 0;                     // columns are [32 value | 32 gate] blocks: store value * gelu(gate) as [M, N/2] (attention.py:42-44)
  int out_nchw = 0;                  // store C as [B, N, rows_per_img] instead of [M, N]
  int rows_per_img = 0;
  // batching over blockIdx.z = zb*heads + zh
  int batch = 1, heads = 1;
  long long sA_b = 0, sA_h = 0, sB_b = 0, sB_h = 0, sC_b = 0, sC_h = 0;
};
// route (optional): how the call ran, known on the host at enqueue time -- bits 0-2, 4-5, 8-23 as gemm_tc's side_done, bit 3:
// tensor cores (0: the FFMA tiles, side outputs by the standalone passes; bits 8-15 then hold the FFMA tile side, 128 or 64, and
// bits 16-23 a split count of 1)
void gemm(Engine& e, const GemmArgs& a, cudaStream_t s, int* route = nullptr);
// wgmma back end (kernels_tc.cu); returns false when the shape is not eligible
// side_done bit 0: c_amax fused, bit 1: c_stats fused, bit 2: split-K (partial sums + reduce kernel); the plan it ran:
// bits 4-5 operand kind (ROUTE_KIND_*), bits 8-15 tile width (128 or 64), bits 16-23 split-K factor
bool gemm_tc(Engine& e, const GemmArgs& a, cudaStream_t s, int* side_done = nullptr);
enum { ROUTE_KIND_SS = 0, ROUTE_KIND_TS = 1, ROUTE_KIND_H16 = 2, ROUTE_KIND_H16_FAST = 3 };
inline int route_plan(int kind, int width, int splits) { return kind << 4 | width << 8 | splits << 16; }
// fused attention (kernels_attn.cu): true when the engine's mode runs N queries over Nk keys at head width d (C channels) fused
bool flash_eligible(const Engine& e, int N, int Nk, int d, int C);
// The fused kernel's operands: hi / lo planes of q [B*N, ldq] and k [B*Nks, ldk] (head h at column h*d; Nks stored keys per image
// >= Nk) and of V^T [heads*d, B*Nvs] (Nvs keys per image, the padding columns zero).  Self-attention: q and k are two column ranges
// of one fused projection.
// TF32: planes rn_tf32(x), rn_tf32(x - hi), as the GEMM epilogues write them; ldq, ldk and Nvs multiples of 4.
// H16 (the default scheme): fp16 planes made by split_rows_h16 / split_transpose_h16 from fp32 q | k and v, each scaled by
// 2^h16_exp_of(*amax) of its tensor's range slot (device); halves the tensor-pipe time and the operand bytes of the TF32 planes.
// ldq, ldk and Nvs multiples of 8.  q_lo, k_lo and vt_lo all null: one-term products on the hi planes (mode 5; the split functions
// then write hi only).
struct AttnPlanes {
  enum Fmt { TF32, H16 } fmt;
  const void* q_hi; const void* q_lo; int ldq;
  const void* k_hi; const void* k_lo; int ldk;
  const void* vt_hi; const void* vt_lo;
  const float* q_amax = nullptr; const float* k_amax = nullptr; const float* v_amax = nullptr;   // H16 only
};
// out [B, N, ldo], head h at column h*d.  False when the planes or the shape do not fit an instantiation.
// qk_row (optional device [B]): image b takes its Q and K from image qk_row[b] and keeps its own V and output -- its probabilities
// are image qk_row[b]'s (attention control).  Null: every image its own.
// acc_rows (optional device [n_acc]): the accumulating launch, out[r] += attention of image r for the listed images only (CTAs for
// those alone); ordered after the stream's previous launch, whose out it reads after the dependent-launch wait.
// kv_row (optional device [B]): image b takes its K and V from image kv_row[b] and keeps its own Q and output -- its queries attend
// over image kv_row[b]'s keys and values (mutual self-attention).  Giving both qk_row and kv_row is an error.
bool flash_attention(Engine& e, const AttnPlanes& a, float* out, int ldo, int B, int N, int Nk, int Nks, int Nvs, int heads, int d, float scale,
                     cudaStream_t s, const int* qk_row = nullptr, const int* acc_rows = nullptr, int n_acc = 0, const int* kv_row = nullptr);
void split_rows_h16(Engine& e, const float* src, long long rows, int cols, long long ld, void* hi, void* lo, long long ldh, const float* amax,
                    cudaStream_t s);
// R rows = `images` images of R / images rows each; Rp > 0: each image's columns padded with zeros to a stride of Rp (V^T key stride)
void split_transpose_h16(Engine& e, const float* src, int R, int Cc, long long ld, void* hi, void* lo, const float* amax, cudaStream_t s,
                         int images = 1, int Rp = 0);
// The fused kernel variant flash_attention runs for head width d, plane format and N queries: queries per CTA, ragged last query
// tile, key split across the two consumer warpgroups, K / V ring depth (all zero: no instantiation)
struct FlashPlan { int qrows, rag, ksplit, ring; };
FlashPlan flash_plan(int d, bool h16, bool one, int N);
// The network executors' operand preparation after the projection, shared by UNetExec::spatial_transformer and
// cdx_op_attention_net so that the op test feeds the kernel exactly as the network does.
// Self-attention, fp16 planes: one plain fp32 q|k|v projection qkv [B*HW, 3C] whose single range slot sets the exponent of all
// three operands.  q|k split in place at ld 3C; K keeps the per-image key stride HW (Nks = HW: an image's last 64-key box reads
// into the next image, masked by Nk); V^T split per image at Nvs = HW rounded up to 8 keys.  lo = false: hi planes only (one-term)
bool self_attention_h16(Engine& e, const float* qkv, const float* slot, float* out, int B, int HW, int C, int heads, int d, float scale, bool lo,
                        cudaStream_t s, const int* qk_row, const int* kv_row, const int* acc_rows = nullptr, int n_acc = 0, int* Nvs_out = nullptr);
// Self-attention, TF32 planes, HW % 4 != 0: q|k planes [B*HW, 2C] from the projection's epilogue and V row-major [B*HW, C], copied
// into rows padded to Nvs = HW rounded up to 4 keys per image (zero rows), transposed and split
bool self_attention_tf32_padded(Engine& e, const float* qk_hi, const float* qk_lo, const float* vr, float* out, int B, int HW, int C, int heads,
                                int d, float scale, cudaStream_t s, const int* qk_row, const int* kv_row, const int* acc_rows = nullptr,
                                int n_acc = 0, int* Nvs_out = nullptr);
// Cross-attention, fp16 planes: K (when k_hi) and V^T of one fused K | V context projection kv [Mk, 2C] (Mk padded context rows),
// both with the exponent of the one slot of the whole projection
void context_split_h16(Engine& e, const float* kv, int Mk, int C, const float* slot, void* k_hi, void* k_lo, void* vt_hi, void* vt_lo,
                       cudaStream_t s);
// LEDITS++'s cross-attention probe (attn_probe): the Q and K of one cross-attention layer in the form its route holds them, so the
// probabilities are those of the operands the layer multiplied.  F32 (unfused routes): fp32 q, fp32 k.  H16 (fused fp16 planes):
// fp32 q (the projection before its split), K as __half planes of k * 2^e with e = h16_exp_of(*k_amax), k = (hi + lo) * 2^-e (hi
// only when k_lo is null: mode 5).  TF32 (fused TF32 planes): q = q_hi + q_lo, k = k_hi + k_lo.  Image b's query p at row b*N + p
// of ldq, its key j at row b*Lk + j of ldk (Lk: the stored keys per image, the padded context on the fused routes); head h at column
// h*d of both.
struct ProbeOperands {
  enum Fmt { F32, H16, TF32 } fmt = F32;
  const float* q = nullptr; const float* q_lo = nullptr; int ldq = 0;
  const void* k = nullptr; const void* k_lo = nullptr; int ldk = 0; int Lk = 0;
  const float* k_amax = nullptr;
};
// map[i, p] (= or += with accumulate) sum over heads h (in order) of sum over j in 1..span[i] of softmax_j(scale * q_p . k_j) over
// all L keys, for the U-Net row rows[i] (device [n_rows] both).  One warp owns each (i, p): the dot in channel order, the softmax
// sums in a fixed lane order, no atomics, so a row's map does not depend on the other rows or their count.  Weighted form
// (LocalBlend; span null): the inner sum is sum over all j of weights[i, j] * softmax_j (device [n_rows, L]).
void attn_probe(Engine& e, const ProbeOperands& o, const int* rows, const int* span, const float* weights, int n_rows, float* map, int N, int L,
                int heads, int d, float scale, bool accumulate, cudaStream_t s);
void split_planes(Engine& e, const float* w, float* hi, float* lo, size_t n, cudaStream_t s);   // hi = rn_tf32(w), lo = rn_tf32(w - hi)
// fp16 split of w * 2^exp: hi = fp16(w'), lo = fp16(w' - hi)  (hi / lo: __half arrays)
void split_planes_h16(Engine& e, const float* w, void* hi, void* lo, size_t n, int exp, cudaStream_t s);
// slot <- max(slot, max |x[r, 0..C)|) over `rows` rows of stride ld (atomic max on the bit pattern)
void amax_rows(Engine& e, const float* x, long long rows, int C, long long ld, float* slot, cudaStream_t s);
int h16_exp_host(float amax);   // exponent e with amax * 2^e in [2^14, 2^15)
bool attention_tc(Engine& e, const float* q, int ldq, const float* k, int ldk, int head_stride, const float* vt, float* out, int ldo, int B,
                  int Nq, int Nk, int heads, int d, float scale, cudaStream_t s);

// ------------------------------------------------------------------------------------------------
// normalisation / softmax / elementwise ops (kernels_norm.cu, kernels_elem.cu)
// ------------------------------------------------------------------------------------------------
// GroupNorm(32) over NHWC, optionally over the channel-concat of two sources; y = [silu]( gn(x)*(1+scale)+shift )
// st1 / st2: per-(image, channel) fp64 {sum, sum of squares} of the sources when their producer already accumulated them
// (stats[(b*C + c)*2 + k]); null -> computed here by one extra read.  amax: optional device scalar <- atomic max |y|.
// ab_out: optional [B, C1+C2] table of the (a, o) the norm applies, y = silu?(x*a + o).
// src_img: optional device [B]; image b of y is image src_img[b]'s norm (its input, statistics and scale / shift), bit for bit.
// amax then covers the images written.  Null: every image its own.
void groupnorm(Engine& e, const float* x1, int C1, const float* x2, int C2, const float* gamma, const float* beta,
               float eps, bool silu, const float* scale, const float* shift, int ld_ss, float* y, int B, int HW,
               cudaStream_t s, const double* st1 = nullptr, const double* st2 = nullptr, float* amax = nullptr, float2* ab_out = nullptr,
               const int* src_img = nullptr);
double* gn_channel_stats(Engine& e, const float* x, int C, int B, int HW, cudaStream_t s);
void gn_channel_stats_into(Engine& e, const float* x, int C, int B, int HW, double* stats, cudaStream_t s);   // stats += (zeroed by the caller)
void layernorm(Engine& e, const float* x, const float* gamma, const float* beta, float* y, int M, int C, cudaStream_t s, float* amax = nullptr);
// in place; causal_nq > 0: row r may only see columns j <= r % causal_nq (the rest become 0)
void softmax_rows(Engine& e, float* x, long long rows, int L, int ld, cudaStream_t s, int causal_nq = 0);
void silu(Engine& e, const float* x, float* y, size_t n, cudaStream_t s);
// x [M,2C] -> y [M,C] = value * gelu(gate); plain: value = x[:, :C], gate = x[:, C:]; interleaved: blocks of [32 value | 32 gate]
void geglu(Engine& e, const float* x, float* y, int M, int C, cudaStream_t s, bool interleaved = false);
void interleave_geglu_rows(Engine& e, const float* src, float* dst, int rows, int rowlen, cudaStream_t s);
void add(Engine& e, const float* a, const float* b, float* y, size_t n, cudaStream_t s);
void avgpool2(Engine& e, const float* x, float* y, int B, int H, int W, int C, cudaStream_t s);      // -> [B,H/2,W/2,C]
void upsample2(Engine& e, const float* x, float* y, int B, int H, int W, int C, cudaStream_t s);     // -> [B,2H,2W,C]
void nchw_to_nhwc(Engine& e, const float* x, float* y, int B, int C, int HW, cudaStream_t s);
void nhwc_to_nchw(Engine& e, const float* x, float* y, int B, int C, int HW, cudaStream_t s);
void timestep_embedding(Engine& e, const float* t, const float* freqs, float* emb, int B, int half, cudaStream_t s, bool sin_first = false);
void repack_conv3x3(Engine& e, const float* w, float* o, int O, int I, cudaStream_t s, int Ipad = 0);   // OIHW -> O,kh,kw,I (I zero-padded to Ipad)
void pad_channels(Engine& e, const float* x, float* y, size_t rows, int C, int Cp, cudaStream_t s);
void embed_tokens(Engine& e, const int* ids, const float* tok, const float* pos, float* out, int B, int L, int W, int vocab, cudaStream_t s);
void quick_gelu(Engine& e, const float* x, float* y, size_t n, cudaStream_t s);     // x * sigmoid(1.702 x)
void gelu(Engine& e, const float* x, float* y, size_t n, cudaStream_t s);           // exact erf GELU     // [rows,C] -> [rows,Cp], zero fill
void copy_rows(Engine& e, const float* src, float* dst, size_t n, cudaStream_t s);
// taming VectorQuantizer2.forward on NHWC latents: per pixel the first argmin_k of (|z|^2 + |e_k|^2) - 2 z.e_k, output z + (e_k - z)
void vq_quantize(Engine& e, const float* z, const float* codebook, float* out, size_t npix, int dim, int n_embed, cudaStream_t s);
// ---- Directional-CLIP / metric kernels (kernels_elem.cu; SURVEY 8f-3)
void clip_preprocess(Engine& e, const float* img, int B, int R, int size, float* out, cudaStream_t s);
void patchify(Engine& e, const float* img, float* out, int B, int S, int P, cudaStream_t s);            // [B,3,S,S] -> [B*(S/P)^2, 3*P*P]
void vit_tokens(Engine& e, const float* patches, const float* cls, const float* pos, float* out, int B, int N, int W, cudaStream_t s);
void gather_rows(Engine& e, const float* x, const int* row_of_batch, float* out, int B, int L, int W, cudaStream_t s);   // out[b] = x[b, row[b]]
void eot_rows(Engine& e, const int* ids, int* rows, int B, int L, cudaStream_t s);                      // first argmax of ids per sample
void dclip_scores(Engine& e, const float* img_f, const float* orig_f, const float* enc_f, const float* dec_f, int B, int D, float* clip_out,
                  float* dclip_out, cudaStream_t s);
void image_metrics(Engine& e, const float* a, const float* b, int B, int H, int W, float* out, cudaStream_t s);
void attention(Engine& e, const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo,
               int B, int Nq, int Nk, int heads, int d, int head_stride, float scale, cudaStream_t s, bool causal = false);

// scheduler kernels (kernels_elem.cu)
void affine(Engine& e, const float* x, float a, float b, float* out, size_t n, cudaStream_t s);
void shift_scale(Engine& e, const float* x, float b, float a, float* out, size_t n, cudaStream_t s);
void q_sample(Engine& e, const float* x0, const float* noise, float sa, float s1ma, float* out, size_t n, cudaStream_t s);
void vae_posterior(Engine& e, const float* moments, const float* noise, float sf, float* out, int B, int C, int hw, cudaStream_t s);
void ddim_posterior_sample(Engine& e, const float* x0, const float* xt, const float* noise, const cdx_ddim_coef& c, float* out, size_t n, cudaStream_t s);
void ddim_compute_eps(Engine& e, const float* xt, const float* xt_next, const float* e_c, const float* e_uc, float scale,
                      const cdx_ddim_coef& c, float* out, size_t n, cudaStream_t s);
void ddim_step_with_eps(Engine& e, const float* x, const float* e_c, const float* e_uc, float scale, const float* eps,
                        const cdx_ddim_coef& c, float* out, size_t n, cudaStream_t s);
// The latent sampling loops (DPM-Encoder, decode, or both in lock-step) run n_src element groups: one source chain per group (when the
// loop has one) drives the group's K target chains (chain j*K + k) with the noise it recovers.  One fused elementwise launch per step
// recovers the noise of step i from the U-Net output (compute_eps), draws the next posterior sample of the source chain
// (sample_xt_next), advances every target chain with the recovered noise (p_sample_ddim_with_eps) and writes the next U-Net input
// batch.  Op order inside is that of the three single-purpose kernels above (bit-exact against the reference formulas).
// A chain finds its U-Net rows through its Chain entry: `row` is the cond row (the uncond row when the chain runs at scale 0 on one
// row), `row2` the uncond row of a chain under classifier-free guidance, else -1.  eps-hat is e(row) when row2 < 0 or scale == 1,
// e(row2) when scale == 0 -- EXACTLY, as the reference's single-forward branches (ddim.py:550-551) -- else
// e(row2) + scale * (e(row) - e(row2)) (ddim.py:559).
struct Chain { int row, row2; float scale; };
struct LatentChains {
  size_t n = 0; int chw = 0, n_src = 0, K = 0;   // n = n_src*chw elements; one thread element carries its source and K targets
  const Chain* chains = nullptr;                 // [n_src] source chains, then [n_src*K] target chains
  int src = 0;                                   // a source chain runs this step; else the recovered noise is read from eps_in
  const float* x0 = nullptr;
  const float* eout = nullptr;                   // step: U-Net output [rows, chw]
  cdx_ddim_coef c{};                             // step: coefficients of this step (both chains share the schedule)
  const float* noise0 = nullptr; float sa = 0.f, s1 = 0.f;     // init with a source: x_T = sa*x0 + s1*noise0 (ddim.py:477-479)
  float* xt = nullptr; float* xn = nullptr;      // source x_t, x_{t-1} (init writes both, step reads them)
  int next = 0;                                  // 0 none, 1 posterior sample x_{t-2} from (x0, xn, noise_next), 2 x_{t-2} = x0 (index 0)
  const float* noise_next = nullptr; cdx_ddim_coef cnext{};
  float* xn2 = nullptr;                          // step: next x_{t-1} of the source chains
  float* z_out = nullptr; long long z_stride = 0;     // optional: x_T (init) / recovered noise (step) -> z_out[j*z_stride + r]
  const float* eps_in = nullptr; long long eps_stride = 0;    // no source: x_T (init) / the step's noise <- eps_in[j*eps_stride + r]
  float* yt = nullptr; float* y_out = nullptr;   // target chains [n_src*K, chw]: init writes yt = x_T; step reads yt, writes y_out
  float* xin = nullptr;                          // next U-Net input [rows, chw]
  // v-prediction (SD 2.x "-v" models): the U-Net output is v; after the guidance combine, e_t = vsa*v + vs1*x_t and
  // pred_x0 = vsa*x_t - vs1*v with vsa = sqrt(abar_t), vs1 = sqrt(1 - abar_t) of the step's timestep (both chains share the step)
  int pred = 0; float vsa = 0.f, vs1 = 0.f;
  // masked editing (step, source chain present): a target chain's x_{t-1} becomes m*y + (1 - m)*x of its group's source x_{t-1},
  // m = mask[j*hw + p] for latent pixel p, broadcast over the C channels; m == 1 keeps y and m == 0 takes x exactly.  Kept last
  // so that the offsets of the fields above, and the unmasked kernels' code, do not change.
  const float* mask = nullptr; int hw = 0;
  // semantic guidance (SEGA; cdx_cycle_lockstep_semantic), sg_m > 0: target chain t has sg_m concept rows sg_rows[t*sg_m + k] at its
  // own x_t (init and step write them as the chain's rows).  With o_uc the chain's uncond row (row2, or row when it runs on one row
  // at scale 0) and o_k concept k's row, per element of channel c = r / hw:
  //   psi_k = sg_scale[k]*(o_k - o_uc);  g_k = (bit k of sg_active and |psi_k| >= sg_thr[(t*sg_m + k)*C + c]) ? psi_k : 0
  //   G = (g_0 + ... + g_{m-1}) + sg_mu*nu;  nu <- sg_beta*nu + sg_beta1*G  (nu = sg_nu[t*chw + r]);  o-hat += G when sg_apply
  // the threshold of each (chain, concept, channel) plane written by semantic_thresholds from the same step's eout.  Kept after the
  // mask so that the earlier offsets, and the code of the kernels without concepts, do not change.
  int sg_m = 0;
  const int* sg_rows = nullptr;                  // device [n_src*K*sg_m]
  float* sg_thr = nullptr;                       // device [n_src*K*sg_m*C]
  float* sg_nu = nullptr;                        // device [n_src*K, chw], zero before the first step
  float sg_scale[8] = {};                        // signed edit scales
  float sg_lambda[8] = {};                       // percentile thresholds in [0, 1)
  unsigned sg_active = 0;                        // bit k: concept k is before its cooldown step
  int sg_apply = 0;                              // the step is past the warmup: o-hat += G
  float sg_mu = 0.f, sg_beta = 0.f, sg_beta1 = 0.f;
  // LEDITS++'s implicit masks (cdx_cycle_lockstep_semantic_attn), sg_mask > 0: concept k of target chain t keeps psi_k at latent
  // pixel (y, x) where the smoothed cross-attention map of its row, sm(y/4, x/4) (ledits_smooth over sg_map[t*sg_m + k], an sg_gh x
  // sg_gw grid), reaches sg_thr[(t*sg_m + k)*2]; with sg_mask == 2 also where the channel sum of |psi_k| at (y, x) reaches
  // sg_thr[(t*sg_m + k)*2 + 1].  The per-channel thresholds are then not used.  Kept last, as the fields above.
  int sg_mask = 0;
  const float* sg_map = nullptr;                 // device [n_src*K*sg_m, sg_gh*sg_gw]: the probe's raw maps
  int sg_gh = 0, sg_gw = 0;
  int w = 0;                                     // latent width: pixel r % hw = y*w + x
  // edit-friendly inversion (cdx_cycle_lockstep_sampler).  solver 0: the DDIM step on the posterior chain; 1: the DDIM step on
  // independent draws; 2: the SDE-DPM-Solver++ step under dc on independent draws.  Under 1 and 2 the source's next x is next == 3,
  // q_sample(x0, noise_next, qa, q1), or next == 2, x0; next == 1 is solver 0's.  Solver 2: D = pred_x0 of each chain,
  // mu = a*x + b*D (+ c*(D - D_prev) at order 2), z = (xn - mu_src) / n, y_next = mu_y + n*z; D_prev is read from d_src / d_tgt
  // ([n_src, chw] / [n_src*K, chw]) and overwritten with D in place.  Kept last, as the fields above.
  int solver = 0;
  cdx_dpm_coef dc{};
  float* d_src = nullptr; float* d_tgt = nullptr;
  float qa = 0.f, q1 = 0.f;
};
constexpr int SEMANTIC_MAX_CONCEPTS = 8;
void latent_chains_init(Engine& e, const LatentChains& a, cudaStream_t s);
void latent_chains_step(Engine& e, const LatentChains& a, cudaStream_t s);
// SEGA's threshold stage: one launch, one CTA per (target chain, concept, channel) plane of hw elements.  theta = Q(sg_lambda[k],
// |psi_k| over the plane): r = lambda*(hw - 1) in fp32, the floor(r)-th and ceil(r)-th smallest values found exactly by a radix
// select over the float bit patterns (re-read from eout each pass: no shared-memory limit on the plane size), then torch.quantile's
// linear interpolation with ATen's scalar lerp, each op rounded.  Writes a.sg_thr.  With sg_mask > 0 the planes are instead, per
// (target chain, concept), the smoothed attention map (sg_gh*sg_gw values) and, with sg_mask == 2, the channel sum of |psi_k| (hw
// values): one or two CTAs per concept row, still one launch.
void semantic_thresholds(Engine& e, const LatentChains& a, cudaStream_t s);
// Prompt-to-Prompt's LocalBlend (cdx_cycle_lockstep_blend).  blend_weights: one probe weight row out [L] <- A . v (A [L, L]
// row-major, one fmaf per n ascending), or d * v elementwise, or v.  local_blend_mask: one launch, one CTA per image b.  maps
// [B*n_vec*n_terms, G] (G = (h/4)(w/4), entry (b*n_vec + v)*n_terms + t); run [B*n_vec, G] += (term 0 + term 1 + ...); then per
// vector v (0 / 1: blend words of the source / target prompt, 2 / 3: subtract words) its maximum mx_v over the grid, and per cell
// keep = OR_{v<2} (maxpool3x3(run_v) / mx_v > th_blend) AND NOT OR_{v>=2} (run_v / mx_v > th_sub) (fp32 division; a map whose
// maximum is 0 adds nothing); mask [B,1,h,w] <- keep of cell (y/4, x/4), times umask [B,1,h,w] when given.
void blend_weights(Engine& e, const float* v, const float* A, const float* d, float* out, int L, cudaStream_t s);
void local_blend_mask(Engine& e, const float* maps, int n_terms, int n_vec, float* run, const float* umask, float th_blend, float th_sub,
                      float* mask, int B, int h, int w, cudaStream_t s);
// image-resolution mask [B,1,H,W] -> [B,1,H/f,W/f]: mean of each f x f block, summed row by row then divided by f*f (avg_pool2d)
void mask_pool(Engine& e, const float* mask, float* out, int B, int H, int W, int f, cudaStream_t s);
// paste-back at image resolution: out = m*clamp((dec + 1)*0.5, 0, 1) + (1 - m)*image, mask [B,1,H,W] broadcast over C channels;
// m == 0 gives image, m == 1 the clamped decode, exactly
void mask_composite(Engine& e, const float* dec, const float* image, const float* mask, float* out, int B, int C, int H, int W,
                    cudaStream_t s);
// DiffEdit mask (cdx_edit_map / cdx_edit_mask).  Pairs q = k*B + b (map k of image b) in map-major order.
// edit_rows: pairs [p0, p1) -> xin rows 2*(q - p0) and 2*(q - p0) + 1 both = q_sample(x0[b], noise[b, k]), noise [B, n_maps, chw]
void edit_rows(Engine& e, const float* x0, const float* noise, float sa, float s1, float* xin, int B, int n_maps, int chw, int p0, int p1,
               cudaStream_t s);
// edit_map_accum: acc [B, hw] += sum_c |vscale*(tgt - src)| per pair of [p0, p1) in map order; pair q's [C, hw] predictions at
// src / tgt + b*sb + k*sk - off0
void edit_map_accum(Engine& e, const float* src, const float* tgt, long long sb, long long sk, long long off0, float vscale, float* acc, int B,
                    int C, int hw, int p0, int p1, cudaStream_t s);
// edit_mask: one block per image -> map = acc / (n_maps*C), latent mask and (img_out non-null) the mask nearest-upsampled by f
void edit_mask(Engine& e, const float* acc, int n_maps, float ratio, float* map_out, float* mask_out, float* img_out, int f, int B, int C, int h,
               int w, cudaStream_t s);
// Running per-sample best of the ensemble search over candidates that arrive in chunks, in any order: candidate c of the chunk
// (image images[c], score scores[c], reference candidate index cand[c], sample sample[c]) replaces the best of its sample when it
// wins under torch.argmax's rule over the [B, n_total] score matrix (larger score; NaN beats any number; ties and NaNs: lower
// index).  best_idx < 0: no candidate yet.  Scores are also written to score_mat[sample, cand].
void ensemble_select(Engine& e, int n, const float* scores, const long long* cand, const int* sample, const float* images, float* best_score,
                     long long* best_idx, float* best_img, float* score_mat, int B, int n_total, size_t img_n, cudaStream_t s);

void pixel_posterior_sample(Engine& e, const float* x0, const float* xt, const float* noise, const cdx_pixel_coef& c, float* out, size_t n, cudaStream_t s);
void pixel_compute_eps(Engine& e, const float* xt, const float* xt_next, const float* et, const cdx_pixel_coef& c, float* out,
                       int B, int chw, int net_chw, cudaStream_t s);
void pixel_step_with_eps(Engine& e, const float* xt, const float* et, const float* eps, const cdx_pixel_coef& c, float* out,
                         int B, int chw, int net_chw, cudaStream_t s);
// one step of the two-model pixel loop (identical schedules): x_{t-1} = sample_xt_next(x0, xs, noise), eps = compute_eps(xs, x_{t-1},
// et_src), ys <- denoising_step_with_eps(ys, et_tgt, eps), xs <- x_{t-1}; bit-identical to the three kernels above
void pixel_lockstep_step(Engine& e, const float* x0, float* xs, float* ys, const float* et_src, const float* et_tgt, const float* noise,
                         const cdx_pixel_coef& c, int B, int chw, int net_chw_src, int net_chw_tgt, cudaStream_t s);

inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

}  // namespace cdx
