// cabi.cu -- the extern "C" surface declared in include/cdx.h, plus the in-library loop drivers
// (DPM-Encoder inversion and decode-with-recovered-noise) so that a whole chain is enqueued without
// returning to the host language between steps.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "nets.cuh"

struct cdx_engine { cdx::Engine e; };
struct cdx_net { cdx::Net* n; cdx_engine* owner; };

namespace cdx {
const std::string& last_error();

namespace {

template <class F>
int guard(F&& f) {
  try {
    f();
    return CDX_OK;
  } catch (const Error& err) {
    set_last_error(err.what());
    return err.code;
  } catch (const std::exception& err) {
    set_last_error(std::string("internal error: ") + err.what());
    return CDX_E_INVALID;
  }
}

// run `f` once in sizing mode, grow the arena, then for real
// The arena, the context K/V cache and the weight planes are reused from call to call with no synchronisation of their own,
// which is only safe in stream order.  A caller that switches streams between calls is handed over explicitly: every call
// records an event at its end, and a call arriving on a different stream first waits for it.
// `e2`: the engine of a second net taking part in the same call (two-model loops); both arenas are sized by the one dry pass, and
// both engines are handed over on `s`.
template <class F>
void with_arena(Engine& e, cudaStream_t s, F&& f, Engine* e2 = nullptr) {
  Engine* const engs[2] = {&e, e2 == &e ? nullptr : e2};
  if (engs[1]) CDX_CHECK(engs[1]->device == e.device, "the two nets of a call live on devices %d and %d", e.device, engs[1]->device);
  CDX_CUDA(cudaSetDevice(e.device));
  for (Engine* x : engs) if (x) x->arena.begin_dry();
  try {
    f();
  } catch (...) {
    for (Engine* x : engs) if (x) { x->arena.dry = false; x->arena.off = 0; }
    throw;
  }
  for (Engine* x : engs) {
    if (!x) continue;
    x->arena.end_dry();
    if (!x->done_ev) CDX_CUDA(cudaEventCreateWithFlags(&x->done_ev, cudaEventDisableTiming));
    if (x->ev_recorded && x->last_stream != s) CDX_CUDA(cudaStreamWaitEvent(s, x->done_ev, 0));
  }
  f();
  for (Engine* x : engs) {
    if (!x) continue;
    x->arena.off = 0;
    CDX_CUDA(cudaEventRecord(x->done_ev, s));
    x->ev_recorded = true;
    x->last_stream = s;
  }
}

// Streams of the two U-Net calls of one two-model step.  The calls are independent (each reads its own chain's x_t); only the
// elementwise step after them joins the chains.  Nets of different engines share no arena, pools or caches, so the target's call
// runs on the target engine's side stream, forked from and joined back into `s` once per step.  Nets of one engine run in order
// on `s`.
struct PairStreams {
  Engine& tgt;
  cudaStream_t s;
  bool two;
  PairStreams(Engine& src_eng, Engine& tgt_eng, cudaStream_t st) : tgt(tgt_eng), s(st), two(&src_eng != &tgt_eng) {
    if (!two || tgt.dry() || tgt.side) return;
    CDX_CUDA(cudaStreamCreateWithFlags(&tgt.side, cudaStreamNonBlocking));     // overlaps a caller on the legacy default stream
    CDX_CUDA(cudaEventCreateWithFlags(&tgt.fork_ev, cudaEventDisableTiming));
    CDX_CUDA(cudaEventCreateWithFlags(&tgt.join_ev, cudaEventDisableTiming));
  }
  cudaStream_t target_stream() const { return two ? tgt.side : s; }
  void fork() {
    if (!two || tgt.dry()) return;
    CDX_CUDA(cudaEventRecord(tgt.fork_ev, s));
    CDX_CUDA(cudaStreamWaitEvent(tgt.side, tgt.fork_ev, 0));
  }
  void join() {
    if (!two || tgt.dry()) return;
    CDX_CUDA(cudaEventRecord(tgt.join_ev, tgt.side));
    CDX_CUDA(cudaStreamWaitEvent(s, tgt.join_ev, 0));
  }
};

inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// fill a device float vector with one value per row, repeated `rep` times (timestep vector for [x;x] CFG batches)
void upload_timesteps(Engine& e, const float* t_host, int n_steps, int reps, float* dev, cudaStream_t s) {
  if (e.dry()) return;
  std::vector<float> h((size_t)n_steps * reps);
  for (int i = 0; i < n_steps; ++i)
    for (int r = 0; r < reps; ++r) h[(size_t)i * reps + r] = t_host[i];
  // pageable source: the runtime stages the copy before returning, so `h` may die afterwards
  CDX_CUDA(cudaMemcpyAsync(dev, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice, s));
}

// dst[b, slot, :] = src[b, :]  for a [B, n_slots, chw] tensor
void scatter_slot(Engine& e, const float* src, float* dst, int B, int chw, int n_slots, int slot, cudaStream_t s) {
  if (e.dry()) return;
  CDX_CUDA(cudaMemcpy2DAsync(dst + (size_t)slot * chw, (size_t)n_slots * chw * sizeof(float), src, (size_t)chw * sizeof(float),
                             (size_t)chw * sizeof(float), B, cudaMemcpyDeviceToDevice, s));
}
void gather_slot(Engine& e, const float* src, float* dst, int B, int chw, int n_slots, int slot, cudaStream_t s) {
  if (e.dry()) return;
  CDX_CUDA(cudaMemcpy2DAsync(dst, (size_t)chw * sizeof(float), src + (size_t)slot * chw, (size_t)n_slots * chw * sizeof(float),
                             (size_t)chw * sizeof(float), B, cudaMemcpyDeviceToDevice, s));
}
void copy_dd(Engine& e, const float* src, float* dst, size_t n, cudaStream_t s) {
  if (e.dry()) return;
  CDX_CUDA(cudaMemcpyAsync(dst, src, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
}

// test hooks: the tensor-core weight planes of an ad-hoc weight matrix, built on the fly (networks do this once at finalize):
// TF32 hi / lo, and in the fp16-split modes the fp16 planes of w * 2^b_exp with b_exp from max(w_range, max |w|) -- w_range stands
// in for the net-wide weight range a network's planes take their exponent from
void hook_weight_planes(Engine& e, const float* w, size_t n, GemmArgs& g, cudaStream_t s, float w_range = 0.f) {
  if (e.mma_mode != 1) return;
  float* thi = (float*)e.arena.alloc(n * sizeof(float));
  float* tlo = (float*)e.arena.alloc(n * sizeof(float));
  split_planes(e, w, thi, tlo, n, s);
  g.Bw_hi = thi; g.Bw_lo = tlo;
  if (e.tc_kind < 1 || (n & 7)) return;
  void* hi = e.arena.alloc(n * 2);
  void* lo = e.arena.alloc(n * 2);
  if (e.dry()) { g.Bw_h_hi = hi; g.Bw_h_lo = lo; return; }
  float* slot = e.amax_slot();
  amax_rows(e, w, 1, (int)n, (long long)n, slot, s);
  float wmax = 0.f;
  CDX_CUDA(cudaMemcpyAsync(&wmax, slot, sizeof(float), cudaMemcpyDeviceToHost, s));
  CDX_CUDA(cudaStreamSynchronize(s));
  g.b_exp = h16_exp_host(std::max(wmax, w_range));
  split_planes_h16(e, w, hi, lo, n, g.b_exp, s);
  g.Bw_h_hi = hi; g.Bw_h_lo = lo;
}

// ---------------------------------------------------------------------------------------------------------------------
// The latent sampling loops (DDIMSampler._ddpm_ddim_encoding ddim.py:450-501, ddim_sampling_with_eps ddim.py:395-448, and the
// ensemble search SDW:189-204 / :146-165) as ONE driver over chains.  Each of the n_src element groups has at most one source chain
// (the DPM-Encoder under the source condition) and K target chains (decoders under the target condition); the noise the source
// recovers at step i is consumed by its targets in registers, so lock-step needs no z buffer -- the Diffusers
// CycleDiffusionPipeline loop shape.  K == 0 is the DPM-Encoder alone, no source chain the decoder alone (noise read from z_in /
// extra), K == 1 the single-image cycle, K > 1 one recovered chain driving several decoder scales.
// Per step: one U-Net call over exactly the rows the chains need (a chain contributes [uncond, cond] when it runs with
// classifier-free guidance, ddim.py:550-559, else one row) and ONE fused elementwise launch (latent_chains_step).
// ---------------------------------------------------------------------------------------------------------------------
// Plug-and-Play injection of one loop (cdx.h, cdx_cycle_lockstep_pnp): the ResBlocks of output blocks blocks[0 .. n_blocks) at
// steps < feature_steps, the self-attention of layers >= start_layer at steps < attention_steps
struct PnpLoop {
  int feature_steps = 0, attention_steps = 0, start_layer = 0;
  const int* blocks = nullptr;                      // host [n_blocks]
  int n_blocks = 0;
};

struct ChainLoopArgs {
  int n_src = 0, K = 0;                            // element groups; target chains per group
  bool src = false;                                // a source chain per group
  const float* x0 = nullptr;                       // src
  // contexts [n_src, L, D]: every chain of group j runs under c_src[j] / c_tgt[j], its uncond row under uc[j]
  const float* c_src = nullptr; const float* c_tgt = nullptr; const float* uc = nullptr; int L = 0;
  // guidance scales [n_src] / [n_src*K], from the host or on the device.  Host scales decide the rows: with `uc`, a chain at a
  // scale other than 0 and 1 has a cond and an uncond row, else one.  Device scales cannot (nothing is read back), so with `uc`
  // every chain has both rows and the step kernel picks the row of a chain at scale 0 or 1.
  const float* s_scales = nullptr; const float* t_scales = nullptr; bool scales_on_device = false;
  const cdx_ddim_coef* coef = nullptr; const float* t_host = nullptr; int n_steps = 0;
  int n_rec = 0; const float* noise = nullptr; float sa = 0.f, s1 = 0.f;      // src: steps the source runs; noise [n_rec+1, n_src, chw]
  float* z_out = nullptr;                           // src: [n_src, n_rec+1, chw], optional when K > 0
  const float* z_in = nullptr; int n_eps = 0;       // no src: [n_src, n_eps+1, chw], x_T then the recovered noises
  const float* extra = nullptr;                     // noise of the steps past n_eps (no src) / past n_rec (src)
  float* x_out = nullptr;                           // K > 0: [n_src*K, chw]
  const float* mask = nullptr;                      // optional [n_src, 1, h, w]: masked editing (LatentChains::mask)
  const cdx_attn_control* ctl = nullptr;           // optional: attention control of each target chain's cond row (cdx.h)
  const float* own_weight = nullptr;                // optional with ctl: [n_src, L], refine's weights of the rows' own attention
  // optional, exclusive with ctl: mutual self-attention (cdx.h, cdx_cycle_lockstep_mutual) at steps >= start_step, layers >= start_layer
  bool mutual = false; int start_step = 0, start_layer = 0;
  const PnpLoop* pnp = nullptr;                     // optional, exclusive with ctl and mutual: Plug-and-Play
  // optional, exclusive with ctl, mutual and pnp: semantic guidance (cdx.h, cdx_cycle_lockstep_semantic), concept contexts
  // c_edit [n_src, m, L, D]: every target chain of group j runs concept k under c_edit[j, k]
  const cdx_semantic_guidance* sega = nullptr; const float* c_edit = nullptr;
  const cdx_semantic_attn_mask* sega_mask = nullptr;    // optional with sega: LEDITS++'s implicit masks (cdx_cycle_lockstep_semantic_attn)
  const cdx_local_blend* blend = nullptr;           // optional, with ctl / own_weight or alone: P2P's LocalBlend (cdx_cycle_lockstep_blend)
  int C = 0, h = 0, w = 0;
  // optional: the source chain's sampler (cdx.h, cdx_cycle_lockstep_sampler); NULL or CDX_SAMPLER_DDIM_POSTERIOR is the DPM-Encoder
  const cdx_sampler* sampler = nullptr;
};

// RAII: the engine's contractions on the exact-fp32 FFMA path for one scope
struct ExactFp32 {
  Engine& e;
  int mode;
  explicit ExactFp32(Engine& eng) : e(eng), mode(eng.mma_mode) { e.mma_mode = 0; }
  ~ExactFp32() { e.mma_mode = mode; }
};

// v-prediction nets (cdx_unet_set_prediction): every U-Net timestep of the loop must index the net's sqrt(abar) tables
void check_v_steps(const Net& u, const float* t_host, int n) {
  if (!u.pred) return;
  for (int i = 0; i < n; ++i) {
    const int t = (int)t_host[i];
    CDX_CHECK((float)t == t_host[i] && t >= 0 && t < (int)u.sa_v.size(), "v-prediction: timestep %g outside the %d-entry table", t_host[i],
              (int)u.sa_v.size());
  }
}
void set_v(const Net& u, float t, LatentChains& st) {
  if (!u.pred) return;
  st.pred = 1; st.vsa = u.sa_v[(int)t]; st.vs1 = u.s1_v[(int)t];
}

// `tgt_net`: the target chains run under their own net (two-model translation, context-free): the step's U-Net call is split into a
// source call and a target call over the source rows and the target rows of `xin` / `eout`.  With n_rec < n_steps the target chains
// continue alone after the last recovered step, with `extra` noise (ddim.py:640).
void run_latent_chains(Net& unet, const ChainLoopArgs& a, cudaStream_t s, Net* tgt_net = nullptr) {
  Engine& e = *unet.eng;
  const int chw = a.C * a.h * a.w, n_tgt_chains = a.n_src * a.K;
  const size_t n = (size_t)a.n_src * chw;
  const size_t ctx_n = (size_t)a.L * unet.ucfg.context_dim;
  if (a.sega) {
    const cdx_semantic_guidance& g = *a.sega;
    CDX_CHECK(!a.ctl && !a.mutual && !a.pnp, "semantic guidance and attention control are exclusive in one loop");
    CDX_CHECK(a.src && a.K > 0 && a.n_rec == a.n_steps && !tgt_net && !a.scales_on_device,
              "semantic guidance: needs the lock-step loop with a source chain at every step");
    CDX_CHECK(ctx_n > 0 && a.c_tgt && a.c_edit, "semantic guidance: needs a net with a context and the concept contexts");
    CDX_CHECK(a.uc, "semantic guidance: needs the unconditional context (its terms are taken against the uncond row)");
    CDX_CHECK(g.m >= 1 && g.m <= SEMANTIC_MAX_CONCEPTS, "semantic guidance: m=%d concepts, 1 to %d", g.m, SEMANTIC_MAX_CONCEPTS);
    for (int k = 0; k < g.m; ++k)
      CDX_CHECK(g.threshold[k] >= 0.0f && g.threshold[k] < 1.0f, "semantic guidance: threshold[%d]=%g outside [0, 1)", k, g.threshold[k]);
  }
  if (a.sega_mask) {
    CDX_CHECK(a.sega, "attention masks: semantic guidance only");
    CDX_CHECK(a.h % 4 == 0 && a.w % 4 == 0 && a.h >= 8 && a.w >= 8, "attention masks: a %dx%d latent, multiples of 4 of at least 8 needed", a.h,
              a.w);
    for (int k = 0; k < a.sega->m; ++k)
      CDX_CHECK(a.sega_mask->n_tokens[k] >= 1 && a.sega_mask->n_tokens[k] <= a.L - 2, "attention masks: n_tokens[%d]=%d outside 1..%d", k,
                a.sega_mask->n_tokens[k], a.L - 2);
  }
  if (a.blend) {
    const cdx_local_blend& lb = *a.blend;
    CDX_CHECK(!a.sega && !a.mutual && !a.pnp, "LocalBlend: Prompt-to-Prompt edits (or none) only, not semantic guidance, MasaCtrl or PnP");
    CDX_CHECK(a.src && a.K == 1 && a.n_rec == a.n_steps && !tgt_net && !a.scales_on_device,
              "LocalBlend: needs the lock-step loop with one target chain per source chain (K=%d)", a.K);
    CDX_CHECK(unet.kind == NET_UNET_OPENAI && ctx_n > 0 && a.c_src && a.c_tgt, "LocalBlend: needs a U-Net with a context and both prompts");
    CDX_CHECK(lb.alpha_src && lb.alpha_tgt && !lb.sub_src == !lb.sub_tgt, "LocalBlend: null blend-word vector, or one subtract vector alone");
    CDX_CHECK(a.h % 4 == 0 && a.w % 4 == 0, "LocalBlend: a %dx%d latent, multiples of 4 needed", a.h, a.w);
    CDX_CHECK(lb.start_step >= 0 && lb.start_step <= a.n_steps, "LocalBlend: start_step=%d (of %d)", lb.start_step, a.n_steps);
    CDX_CHECK(lb.th_blend >= 0.f && lb.th_blend < 1.f && lb.th_sub >= 0.f && lb.th_sub < 1.f, "LocalBlend: thresholds %g, %g outside [0, 1)",
              lb.th_blend, lb.th_sub);
  }
  // the chain table: all source-chain rows first, then all target-chain rows (the two-model loop runs the two blocks under two
  // nets); inside a block the uncond rows come first, cat([uc, c]) as ddim.py:555-557
  std::vector<Chain> ch((size_t)a.n_src + n_tgt_chains, Chain{-1, -1, 1.f});
  int rows = 0;
  // need_uc: the chains need their uncond row's output even at scale 1 (semantic guidance forms its terms against it)
  auto place = [&](Chain* c, int count, const float* scales, bool need_uc) {
    for (int k = 0; k < count; ++k) {
      if (!a.scales_on_device && scales) c[k].scale = scales[k];
      if (a.uc && (a.scales_on_device || (c[k].scale != 0.0f && (c[k].scale != 1.0f || need_uc)))) c[k].row2 = rows++;
    }
    for (int k = 0; k < count; ++k) c[k].row = rows++;
  };
  if (a.src) place(ch.data(), a.n_src, a.s_scales, false);
  const int rows_src = rows;
  place(ch.data() + a.n_src, n_tgt_chains, a.t_scales, a.sega != nullptr);
  // semantic guidance: the m concept rows of every target chain after the whole target block, chain-major, so that no other row moves
  const int sg_m = a.sega ? a.sega->m : 0;
  std::vector<int> sg_rows((size_t)n_tgt_chains * sg_m);
  for (int& r : sg_rows) r = rows++;
  const int loop_steps = a.K ? a.n_steps : a.n_rec;
  CDX_CHECK(!tgt_net || (!unet.pred && !tgt_net->pred), "two-model latent loop: eps-prediction U-Nets only");
  // a masked target chain takes its source chain's x_{t-1} outside the mask, so every step needs one
  CDX_CHECK(!a.mask || (a.src && a.K > 0 && a.n_rec == a.n_steps && !tgt_net), "masked latent loop: needs a source chain at every step");
  check_v_steps(unet, a.t_host, loop_steps);
  if (a.ctl) {
    const cdx_attn_control& c = *a.ctl;
    CDX_CHECK(a.src && a.K > 0 && a.n_rec == a.n_steps && !tgt_net && !a.scales_on_device,
              "attention control: needs the lock-step loop with a source chain at every step");
    CDX_CHECK(ctx_n > 0 && a.c_src && a.c_tgt, "attention control: needs a net with a context and both prompts");
    CDX_CHECK(e.mma_mode == 1 && e.flash_attn, "attention control: needs the fused attention kernel (mma modes 1, 3, 4 or 5)");
    CDX_CHECK(c.cross_steps >= 0 && c.cross_steps <= a.n_steps && c.self_steps >= 0 && c.self_steps <= a.n_steps && c.self_max_tokens >= 0,
              "attention control: cross_steps=%d self_steps=%d (of %d) self_max_tokens=%d", c.cross_steps, c.self_steps, a.n_steps,
              c.self_max_tokens);
  }
  CDX_CHECK(!a.own_weight || a.ctl, "refine: own_weight needs an attention control");
  if (a.mutual) {
    CDX_CHECK(!a.ctl, "mutual self-attention and Prompt-to-Prompt control are exclusive in one loop");
    CDX_CHECK(a.src && a.K > 0 && a.n_rec == a.n_steps && !tgt_net && !a.scales_on_device,
              "mutual self-attention: needs the lock-step loop with a source chain at every step");
    CDX_CHECK(unet.kind == NET_UNET_OPENAI && ctx_n > 0 && a.c_src && a.c_tgt, "mutual self-attention: needs a U-Net with SpatialTransformers");
    CDX_CHECK(e.mma_mode == 1 && e.flash_attn, "mutual self-attention: needs the fused attention kernel (mma modes 1, 3, 4 or 5)");
    CDX_CHECK(a.start_step >= 0 && a.start_layer >= 0, "mutual self-attention: start_step=%d start_layer=%d", a.start_step, a.start_layer);
  }
  if (a.pnp) {
    const PnpLoop& p = *a.pnp;
    CDX_CHECK(!a.ctl && !a.mutual, "Plug-and-Play, Prompt-to-Prompt and mutual self-attention are exclusive in one loop");
    CDX_CHECK(a.src && a.K > 0 && a.n_rec == a.n_steps && !tgt_net && !a.scales_on_device,
              "Plug-and-Play: needs the lock-step loop with a source chain at every step");
    CDX_CHECK(unet.kind == NET_UNET_OPENAI && ctx_n > 0 && a.c_src && a.c_tgt, "Plug-and-Play: needs a U-Net with SpatialTransformers");
    CDX_CHECK(e.mma_mode == 1 && e.flash_attn, "Plug-and-Play: needs the fused attention kernel (mma modes 1, 3, 4 or 5)");
    CDX_CHECK(p.feature_steps >= 0 && p.feature_steps <= a.n_steps && p.attention_steps >= 0 && p.attention_steps <= a.n_steps &&
              p.start_layer >= 0 && p.n_blocks >= 0 && (p.blocks || p.n_blocks == 0),
              "Plug-and-Play: feature_steps=%d attention_steps=%d (of %d) attention_start_layer=%d n_blocks=%d", p.feature_steps,
              p.attention_steps, a.n_steps, p.start_layer, p.n_blocks);
    const int n_out = unet.ucfg.n_mult * (unet.ucfg.num_res_blocks + 1);
    for (int i = 0; i < p.n_blocks; ++i) {
      CDX_CHECK(p.blocks[i] >= 0 && p.blocks[i] < n_out, "Plug-and-Play: feature block %d outside the net's %d output blocks", p.blocks[i], n_out);
      for (int j = 0; j < i; ++j) CDX_CHECK(p.blocks[j] != p.blocks[i], "Plug-and-Play: feature block %d given twice", p.blocks[i]);
    }
  }
  // edit-friendly inversion: independent draws of the source's x at every step (solver 1 and 2), the DPM table (solver 2)
  const int solver = a.sampler ? a.sampler->kind : 0;
  if (solver) {
    const cdx_sampler& sp = *a.sampler;
    CDX_CHECK(solver == CDX_SAMPLER_DDIM_DRAWS || solver == CDX_SAMPLER_DPMSOLVER_DRAWS, "sampler: kind %d", solver);
    CDX_CHECK(a.src && a.K > 0 && a.n_rec == a.n_steps && !tgt_net && a.noise,
              "edit-friendly inversion: needs the lock-step loop with a source chain at every step");
    CDX_CHECK(sp.qa && sp.q1 && sp.qa[0] == a.sa && sp.q1[0] == a.s1,
              "edit-friendly inversion: the draw scalars qa / q1 must be given, their step 0 the x_T scalars");
    if (solver == CDX_SAMPLER_DPMSOLVER_DRAWS) {
      CDX_CHECK(sp.dpm, "SDE-DPM-Solver++: null coefficient table");
      for (int i = 0; i < a.n_steps; ++i) {
        const cdx_dpm_coef& d = sp.dpm[i];
        CDX_CHECK(d.n > 0.f && std::isfinite(d.n) && (d.order == 1 || d.order == 2), "SDE-DPM-Solver++: step %d n=%g order %d", i, d.n, d.order);
        CDX_CHECK(i > 0 || d.order == 1, "SDE-DPM-Solver++: order %d on the loop's first step (no previous x0-prediction)", d.order);
      }
    }
  }
  Scope sc(e.arena);
  unet.ctxkv.valid = false;                    // the conditioning is fixed for this loop: its K / V are computed by the first step only
  struct Invalidate { Net& u; ~Invalidate() { u.ctxkv.valid = false; } } inval{unet};
  float* xin = (float*)e.arena.alloc((size_t)rows * chw * sizeof(float));
  float* eout = (float*)e.arena.alloc((size_t)rows * chw * sizeof(float));
  float* ctx_in = (float*)e.arena.alloc((size_t)rows * ctx_n * sizeof(float));
  float* xb[3] = {nullptr, nullptr, nullptr};
  float* yb[2] = {nullptr, nullptr};
  if (a.src) for (float*& p : xb) p = (float*)e.arena.alloc(n * sizeof(float));
  if (a.K) for (float*& p : yb) p = (float*)e.arena.alloc((size_t)n_tgt_chains * chw * sizeof(float));
  float* tdev = (float*)e.arena.alloc((size_t)std::max(loop_steps, 1) * rows * sizeof(float));
  Chain* chd = (Chain*)e.arena.alloc(ch.size() * sizeof(Chain));
  upload_timesteps(e, a.t_host, loop_steps, rows, tdev, s);
  if (!e.dry()) {   // pageable source: staged before the call returns
    CDX_CUDA(cudaMemcpyAsync(chd, ch.data(), ch.size() * sizeof(Chain), cudaMemcpyHostToDevice, s));
    auto scales_to = [&](Chain* c, const float* scales, int count) {
      CDX_CUDA(cudaMemcpy2DAsync(&c->scale, sizeof(Chain), scales, sizeof(float), sizeof(float), count, cudaMemcpyDeviceToDevice, s));
    };
    if (a.scales_on_device && a.src) scales_to(chd, a.s_scales, a.n_src);
    if (a.scales_on_device && a.K) scales_to(chd + a.n_src, a.t_scales, n_tgt_chains);
  }
  if (ctx_n) {   // one context per row: the chain's condition on its cond row, uc on its uncond row; unconditional models carry none
    auto ctx_rows = [&](const Chain& c, const float* cond, int j) {
      const bool uncond_only = a.uc && !a.scales_on_device && c.scale == 0.0f;
      copy_dd(e, (uncond_only ? a.uc : cond) + j * ctx_n, ctx_in + (size_t)c.row * ctx_n, ctx_n, s);
      if (c.row2 >= 0) copy_dd(e, a.uc + j * ctx_n, ctx_in + (size_t)c.row2 * ctx_n, ctx_n, s);
    };
    for (int j = 0; j < a.n_src; ++j) {
      if (a.src) ctx_rows(ch[j], a.c_src, j);
      for (int k = 0; k < a.K; ++k) ctx_rows(ch[a.n_src + (size_t)j * a.K + k], a.c_tgt, j);
    }
    for (int t = 0; t < n_tgt_chains; ++t)
      for (int q = 0; q < sg_m; ++q)
        copy_dd(e, a.c_edit + ((size_t)(t / a.K) * sg_m + q) * ctx_n, ctx_in + (size_t)sg_rows[(size_t)t * sg_m + q] * ctx_n, ctx_n, s);
  }
  // semantic guidance: the concept row table, the thresholds of the step and the momentum of every target chain, fixed for the loop
  int* sg_rows_dev = nullptr;
  float *sg_thr = nullptr, *sg_nu = nullptr;
  // attention masks: each concept row's span and raw map, written by the probe of every step's U-Net call
  AttnProbe probe;
  const int sg_mask = a.sega_mask ? 1 + (a.sega_mask->intersect != 0) : 0, gh = a.h / 4, gw = a.w / 4;
  if (sg_m) {
    sg_rows_dev = (int*)e.arena.alloc(sg_rows.size() * sizeof(int));
    sg_thr = (float*)e.arena.alloc(sg_rows.size() * std::max(a.C, 2) * sizeof(float));
    sg_nu = (float*)e.arena.alloc((size_t)n_tgt_chains * chw * sizeof(float));
    if (!e.dry()) {
      CDX_CUDA(cudaMemcpyAsync(sg_rows_dev, sg_rows.data(), sg_rows.size() * sizeof(int), cudaMemcpyHostToDevice, s));   // (pageable: staged)
      CDX_CUDA(cudaMemsetAsync(sg_nu, 0, (size_t)n_tgt_chains * chw * sizeof(float), s));
    }
  }
  if (sg_mask) {
    std::vector<int> span(sg_rows.size());
    for (size_t r = 0; r < span.size(); ++r) span[r] = a.sega_mask->n_tokens[r % sg_m];
    int* span_dev = (int*)e.arena.alloc(span.size() * sizeof(int));
    if (!e.dry()) CDX_CUDA(cudaMemcpyAsync(span_dev, span.data(), span.size() * sizeof(int), cudaMemcpyHostToDevice, s));
    probe.rows = sg_rows_dev; probe.span = span_dev; probe.n_rows = (int)sg_rows.size(); probe.tokens = gh * gw;
    probe.map = (float*)e.arena.alloc(sg_rows.size() * gh * gw * sizeof(float));
  }
  // attention control: the row table maps each target chain's cond row to its group's source row (every other row to itself); with
  // a token map, the V context holds A_j . c_tgt[j] on those rows and every other row's own context.  Both fixed for the loop
  AttnControl actl;
  if (a.ctl) {
    std::vector<int> qk(rows);
    for (int r = 0; r < rows; ++r) qk[r] = r;
    for (int j = 0; j < a.n_src; ++j) {
      CDX_CHECK(!a.uc || ch[j].scale != 0.0f, "attention control: the source chain at scale 0 has no source-prompt row");
      for (int k = 0; k < a.K; ++k) {
        const Chain& t = ch[a.n_src + (size_t)j * a.K + k];
        CDX_CHECK(!a.uc || t.scale != 0.0f, "attention control: the target chain at scale 0 has no target-prompt row");
        qk[t.row] = ch[j].row;
      }
    }
    int* qk_dev = (int*)e.arena.alloc((size_t)rows * sizeof(int));
    if (!e.dry()) CDX_CUDA(cudaMemcpyAsync(qk_dev, qk.data(), qk.size() * sizeof(int), cudaMemcpyHostToDevice, s));   // (pageable: staged)
    actl.qk_row = qk_dev;
    actl.self_max_tokens = a.ctl->self_max_tokens;
    // out[row] = A_j [L, L] . c_tgt[j] [L, D] on each target chain's cond row, in exact fp32 (A_j at A + j L L)
    auto ctx_products = [&](const float* A, float* out) {
      const int D = unet.ucfg.context_dim;
      ExactFp32 exact(e);
      for (int j = 0; j < a.n_src; ++j)
        for (int k = 0; k < a.K; ++k) {
          GemmArgs g;
          g.mode = 0;
          g.M = a.L; g.N = D; g.K = a.L;
          g.A = A + (size_t)j * a.L * a.L; g.lda = a.L; g.C1 = a.L;
          g.Bw = a.c_tgt + (size_t)j * ctx_n; g.ldb = D; g.b_kn = 1;
          g.Cout = out + (size_t)ch[a.n_src + (size_t)j * a.K + k].row * ctx_n; g.ldc = D;
          gemm(e, g, s);
        }
    };
    if (a.ctl->token_map) {
      float* cv = (float*)e.arena.alloc((size_t)rows * ctx_n * sizeof(float));
      copy_dd(e, ctx_in, cv, (size_t)rows * ctx_n, s);
      ctx_products(a.ctl->token_map, cv);
      actl.ctx_v = cv;
    }
    if (a.own_weight) {
      // refine: the second term's context holds diag(w_j) . c_tgt[j] on the controlled rows and zeros elsewhere (those rows run no
      // second term, and zeros keep them out of its range slot), formed by the same exact-fp32 GEMM with a diagonal A
      float* cw = (float*)e.arena.alloc((size_t)rows * ctx_n * sizeof(float));
      float* dg = (float*)e.arena.alloc((size_t)a.n_src * a.L * a.L * sizeof(float));
      std::vector<int> own;
      for (int j = 0; j < a.n_src; ++j)
        for (int k = 0; k < a.K; ++k) own.push_back(ch[a.n_src + (size_t)j * a.K + k].row);
      int* own_dev = (int*)e.arena.alloc(own.size() * sizeof(int));
      if (!e.dry()) {
        CDX_CUDA(cudaMemcpyAsync(own_dev, own.data(), own.size() * sizeof(int), cudaMemcpyHostToDevice, s));   // (pageable: staged)
        CDX_CUDA(cudaMemsetAsync(cw, 0, (size_t)rows * ctx_n * sizeof(float), s));
        CDX_CUDA(cudaMemsetAsync(dg, 0, (size_t)a.n_src * a.L * a.L * sizeof(float), s));
        for (int j = 0; j < a.n_src; ++j)      // w_j onto the diagonal: a stride of L + 1 floats
          CDX_CUDA(cudaMemcpy2DAsync(dg + (size_t)j * a.L * a.L, (size_t)(a.L + 1) * sizeof(float), a.own_weight + (size_t)j * a.L, sizeof(float),
                                     sizeof(float), a.L, cudaMemcpyDeviceToDevice, s));
      }
      ctx_products(dg, cw);
      actl.ctx_w = cw;
      actl.own_rows = own_dev;
      actl.n_own = (int)own.size();
    }
  }
  // mutual self-attention and Plug-and-Play: each target chain's cond row reads its group's source cond row, its uncond row the
  // source's uncond row (the source's only row when it runs without one); every other row its own.  Fixed for the loop
  if (a.mutual || a.pnp) {
    std::vector<int> src_row(rows);
    for (int r = 0; r < rows; ++r) src_row[r] = r;
    for (int j = 0; j < a.n_src; ++j)
      for (int k = 0; k < a.K; ++k) {
        const Chain& t = ch[a.n_src + (size_t)j * a.K + k];
        src_row[t.row] = ch[j].row;
        if (t.row2 >= 0) src_row[t.row2] = ch[j].row2 >= 0 ? ch[j].row2 : ch[j].row;
      }
    int* dev = (int*)e.arena.alloc((size_t)rows * sizeof(int));
    if (!e.dry()) CDX_CUDA(cudaMemcpyAsync(dev, src_row.data(), src_row.size() * sizeof(int), cudaMemcpyHostToDevice, s));   // (pageable: staged)
    if (a.mutual) {
      actl.kv_row = dev;
      actl.start_layer = a.start_layer;
    } else {
      actl.pnp_row = dev;
      actl.pnp_layer = a.pnp->start_layer;
      actl.feat_blocks = a.pnp->blocks;
      actl.n_feat = a.pnp->n_blocks;
    }
  }
  // LocalBlend: the probe's entry tables, [0] the rows' own maps and [1] the maps of an edited step, uploaded once.  Entry
  // (j*n_vec + v)*T + t of image j, vector v (source / target blend words, then source / target subtract words), term t.  A source
  // vector probes the source row; a target vector the target row, or at an edited step the source row with A_j v (the map P_src A_j
  // contracted with v) plus, under refine (T = 2), the target row with own_weight_j * v.  The running sums and the step's mask
  AttnProbe bprobe[2];
  int bl_terms[2] = {1, 1};
  const int bl_vec = a.blend ? (a.blend->sub_src ? 4 : 2) : 0;
  float *bl_run = nullptr, *bl_mask = nullptr;
  if (a.blend) {
    const int G = gh * gw, L = a.L;
    const float* vecs[4] = {a.blend->alpha_src, a.blend->alpha_tgt, a.blend->sub_src, a.blend->sub_tgt};
    for (int j = 0; j < a.n_src; ++j) {
      CDX_CHECK(!a.uc || ch[j].scale != 0.0f, "LocalBlend: the source chain at scale 0 has no source-prompt row");
      CDX_CHECK(!a.uc || ch[a.n_src + j].scale != 0.0f, "LocalBlend: the target chain at scale 0 has no target-prompt row");
    }
    bl_terms[1] = a.own_weight ? 2 : 1;
    for (int tab = 0; tab < (a.ctl ? 2 : 1); ++tab) {
      const int T = bl_terms[tab], n_ent = a.n_src * bl_vec * T;
      std::vector<int> rows_h((size_t)n_ent);
      float* wts = (float*)e.arena.alloc((size_t)n_ent * L * sizeof(float));
      if (!e.dry()) CDX_CUDA(cudaMemsetAsync(wts, 0, (size_t)n_ent * L * sizeof(float), s));
      for (int j = 0; j < a.n_src; ++j)
        for (int v = 0; v < bl_vec; ++v)
          for (int t = 0; t < T; ++t) {
            const int idx = (j * bl_vec + v) * T + t, src_row = ch[j].row, tgt_row = ch[a.n_src + j].row;
            const float* vec = vecs[v] + (size_t)j * L;
            float* out = wts + (size_t)idx * L;
            if (!(v & 1)) {                       // source vector: the source row's own map (a refine term 1 stays zero)
              rows_h[idx] = src_row;
              if (t == 0) blend_weights(e, vec, nullptr, nullptr, out, L, s);
            } else if (tab == 0) {
              rows_h[idx] = tgt_row;
              blend_weights(e, vec, nullptr, nullptr, out, L, s);
            } else if (t == 0) {
              rows_h[idx] = src_row;
              blend_weights(e, vec, a.ctl->token_map ? a.ctl->token_map + (size_t)j * L * L : nullptr, nullptr, out, L, s);
            } else {
              rows_h[idx] = tgt_row;
              blend_weights(e, vec, nullptr, a.own_weight + (size_t)j * L, out, L, s);
            }
          }
      int* rows_dev = (int*)e.arena.alloc(rows_h.size() * sizeof(int));
      if (!e.dry()) CDX_CUDA(cudaMemcpyAsync(rows_dev, rows_h.data(), rows_h.size() * sizeof(int), cudaMemcpyHostToDevice, s));   // (pageable: staged)
      AttnProbe& p = bprobe[tab];
      p.rows = rows_dev; p.weights = wts; p.n_rows = n_ent; p.tokens = G;
      p.map = (float*)e.arena.alloc((size_t)n_ent * G * sizeof(float));
    }
    bl_run = (float*)e.arena.alloc((size_t)a.n_src * bl_vec * G * sizeof(float));
    bl_mask = (float*)e.arena.alloc((size_t)a.n_src * a.h * a.w * sizeof(float));
    if (!e.dry()) CDX_CUDA(cudaMemsetAsync(bl_run, 0, (size_t)a.n_src * bl_vec * G * sizeof(float), s));
  }
  auto next_kind = [&](int i_next) {             // how x_{t-1} of iteration i_next is obtained (0: that iteration does not exist)
    if (i_next >= a.n_rec) return 0;
    return (a.n_steps - 1 - i_next) == 0 ? 2 : solver ? 3 : 1;                  // ddim.py:583-584; 3: an independent draw
  };
  // solver 2: each chain's previous x0-prediction, written by every step before the second-order steps read it
  float *d_src = nullptr, *d_tgt = nullptr;
  if (solver == CDX_SAMPLER_DPMSOLVER_DRAWS) {
    d_src = (float*)e.arena.alloc(n * sizeof(float));
    d_tgt = (float*)e.arena.alloc((size_t)n_tgt_chains * chw * sizeof(float));
  }
  // the noise of a step no source chain recovers: the z_in slots while they last, then `extra`
  const int n_given = a.src ? a.n_rec : a.n_eps;
  LatentChains f;
  f.n = n; f.chw = chw; f.n_src = a.n_src; f.K = a.K; f.chains = chd; f.x0 = a.x0; f.xin = xin; f.mask = a.mask; f.hw = a.h * a.w;
  f.z_stride = (long long)(a.n_rec + 1) * chw;
  f.solver = solver; f.d_src = d_src; f.d_tgt = d_tgt;
  if (sg_m) {
    const cdx_semantic_guidance& g = *a.sega;
    f.sg_m = sg_m; f.sg_rows = sg_rows_dev; f.sg_thr = sg_thr; f.sg_nu = sg_nu;
    for (int q = 0; q < sg_m; ++q) { f.sg_scale[q] = g.scale[q]; f.sg_lambda[q] = g.threshold[q]; }
    f.sg_mu = g.momentum_scale; f.sg_beta = g.beta; f.sg_beta1 = g.beta1;
    f.sg_mask = sg_mask; f.sg_map = probe.map; f.sg_gh = gh; f.sg_gw = gw; f.w = a.w;
  }
  {
    LatentChains in = f;
    in.src = a.src;
    in.noise0 = a.noise; in.sa = a.sa; in.s1 = a.s1; in.z_out = a.z_out;
    in.eps_in = a.z_in; in.eps_stride = (long long)(a.n_eps + 1) * chw;                // x_T = eps_list[:, 0], SDW:153
    in.xt = xb[0]; in.xn = xb[1]; in.yt = yb[0];
    in.next = a.src ? next_kind(0) : 0;
    if (in.next) { in.noise_next = a.noise + n; in.cnext = a.coef[0]; }
    if (in.next == 3) { in.qa = a.sampler->qa[1]; in.q1 = a.sampler->q1[1]; }
    latent_chains_init(e, in, s);
  }
  const int iters = e.dry() ? std::min(loop_steps, 1) : loop_steps;
  PairStreams ps(e, tgt_net ? *tgt_net->eng : e, s);
  for (int i = 0; i < iters; ++i) {
    const bool src_i = a.src && i < a.n_rec;
    if (!tgt_net) {
      actl.cross = a.ctl && i < a.ctl->cross_steps;
      actl.self = a.ctl && i < a.ctl->self_steps;
      actl.mutual = a.mutual && i >= a.start_step;
      actl.pnp_feat = a.pnp && i < a.pnp->feature_steps;
      actl.pnp_attn = a.pnp && i < a.pnp->attention_steps;
      const size_t stat0 = e.stat_dry;
      const AttnProbe* pr = sg_mask ? &probe : a.blend ? &bprobe[actl.cross ? 1 : 0] : nullptr;
      unet_forward(unet, xin, tdev + (size_t)i * rows, ctx_in, a.L, eout, rows, a.h, a.w, s, true,
                   a.ctl || a.mutual || a.pnp ? &actl : nullptr, pr);
      CDX_CHECK(!sg_m || !e.dry() || e.stat_dry - stat0 <= e.stat_cap,
                "semantic guidance: a %d-row U-Net call needs %zu GroupNorm statistics doubles, the pool holds %zu: fewer images or concepts",
                rows, e.stat_dry - stat0, e.stat_cap);
    } else {
      ps.fork();
      if (src_i) unet_forward(unet, xin, tdev + (size_t)i * rows, nullptr, 0, eout, rows_src, a.h, a.w, s);
      unet_forward(*tgt_net, xin + (size_t)rows_src * chw, tdev + (size_t)i * rows + rows_src, nullptr, 0, eout + (size_t)rows_src * chw,
                   rows - rows_src, a.h, a.w, ps.target_stream());
      ps.join();
    }
    LatentChains st = f;
    st.src = src_i; st.eout = eout; st.c = a.coef[i];
    if (src_i) {
      st.xt = xb[0]; st.xn = xb[1]; st.xn2 = xb[2];
      if (a.z_out) st.z_out = a.z_out + (size_t)(1 + i) * chw;
      st.next = next_kind(i + 1);
      if (st.next) { st.noise_next = a.noise + (size_t)(2 + i) * n; st.cnext = a.coef[i + 1]; }
      if (st.next == 3) { st.qa = a.sampler->qa[i + 2]; st.q1 = a.sampler->q1[i + 2]; }
      if (solver == CDX_SAMPLER_DPMSOLVER_DRAWS) st.dc = a.sampler->dpm[i];
    } else if (i < n_given) {
      st.eps_in = a.z_in + (size_t)(1 + i) * chw; st.eps_stride = (long long)(a.n_eps + 1) * chw;
    } else {
      st.eps_in = a.extra + (size_t)(i - n_given) * n; st.eps_stride = chw;
    }
    st.yt = yb[0]; st.y_out = (i == loop_steps - 1) ? a.x_out : yb[1];
    set_v(unet, a.t_host[i], st);
    if (sg_m) {                                   // this step's flags, then the thresholds of this step's outputs
      for (int q = 0; q < sg_m; ++q) st.sg_active |= (unsigned)(i < a.sega->cooldown[q]) << q;
      st.sg_apply = i >= a.sega->warmup;
      semantic_thresholds(e, st, s);
    }
    if (a.blend) {                                // this step's maps into the running sums, then the mask the step blends under
      const int tab = actl.cross ? 1 : 0;
      local_blend_mask(e, bprobe[tab].map, bl_terms[tab], bl_vec, bl_run, a.mask, a.blend->th_blend, a.blend->th_sub, bl_mask, a.n_src, a.h,
                       a.w, s);
      if (i >= a.blend->start_step) st.mask = bl_mask;
    }
    latent_chains_step(e, st, s);
    if (src_i) { float* t0 = xb[0]; xb[0] = xb[1]; xb[1] = xb[2]; xb[2] = t0; }
    std::swap(yb[0], yb[1]);
  }
}

// DiffEdit's mask statistics (Couairon et al., 2022): for each image b and map k, x_t = q_sample(x0[b], noise[b, k]) at timestep t
// runs under c_src[b] and c_tgt[b], and acc[b] += sum_c |e_tgt - e_src| (v nets: sa_v[t]*(v_tgt - v_src), in eps units).  The
// (map, image) pairs are walked map-major, as many whole pairs per U-Net call as rows_per_call allows (two rows each): per call one
// launch builds the rows, one U-Net call, one launch accumulates.  The accumulate kernel adds the maps of an image in map order, so
// acc does not depend on rows_per_call.
void run_edit_map(Net& unet, const float* x0, const float* c_src, const float* c_tgt, int L, float t, float sa, float s1, const float* noise,
                  int n_maps, int rows_per_call, float* acc, int B, int C, int h, int w, cudaStream_t s) {
  Engine& e = *unet.eng;
  const int chw = C * h * w, hw = h * w, n_pairs = n_maps * B, per_call = std::min(rows_per_call / 2, n_pairs), rows = 2 * per_call;
  const size_t ctx_n = (size_t)L * unet.ucfg.context_dim;
  check_v_steps(unet, &t, 1);
  const float vscale = unet.pred ? unet.sa_v[(int)t] : 1.f;
  Scope sc(e.arena);
  float* xin = (float*)e.arena.alloc((size_t)rows * chw * sizeof(float));
  float* eout = (float*)e.arena.alloc((size_t)rows * chw * sizeof(float));
  float* ctx_in = (float*)e.arena.alloc((size_t)rows * ctx_n * sizeof(float));
  float* tdev = (float*)e.arena.alloc((size_t)rows * sizeof(float));
  upload_timesteps(e, &t, 1, rows, tdev, s);
  if (!e.dry()) CDX_CUDA(cudaMemsetAsync(acc, 0, (size_t)B * hw * sizeof(float), s));
  // the sizing pass runs the first call, the largest
  const int calls = e.dry() ? 1 : cdiv(n_pairs, per_call);
  for (int c = 0; c < calls; ++c) {
    const int p0 = c * per_call, p1 = std::min(p0 + per_call, n_pairs), nr = 2 * (p1 - p0);
    for (int q = p0; q < p1; ++q) {
      const int b = q % B, r = 2 * (q - p0);
      copy_dd(e, c_src + (size_t)b * ctx_n, ctx_in + (size_t)r * ctx_n, ctx_n, s);
      copy_dd(e, c_tgt + (size_t)b * ctx_n, ctx_in + (size_t)(r + 1) * ctx_n, ctx_n, s);
    }
    edit_rows(e, x0, noise, sa, s1, xin, B, n_maps, chw, p0, p1, s);
    const size_t stat0 = e.stat_dry;
    unet_forward(unet, xin, tdev, ctx_in, L, eout, nr, h, w, s);
    CDX_CHECK(!e.dry() || e.stat_dry - stat0 <= e.stat_cap,
              "edit_map: a %d-row U-Net call needs %zu GroupNorm statistics doubles, the pool holds %zu: lower rows_per_call", nr,
              e.stat_dry - stat0, e.stat_cap);
    edit_map_accum(e, eout, eout + chw, 2LL * chw, 2LL * B * chw, 2LL * p0 * chw, vscale, acc, B, C, hw, p0, p1, s);
  }
}

}  // namespace
}  // namespace cdx

using namespace cdx;

static inline cdx::Engine& engine_of(cdx_engine* h) { return h->e; }

extern "C" {

int cdx_abi_version(void) { return CDX_ABI_VERSION; }
const char* cdx_last_error(void) { return cdx::last_error().c_str(); }

int cdx_engine_create(int device, cdx_engine** out) {
  return guard([&] {
    CDX_CHECK(out != nullptr, "engine_create: null out");
    int count = 0;
    cudaError_t err = cudaGetDeviceCount(&count);
    if (err != cudaSuccess || count <= 0)
      throw Error(CDX_E_CUDA, std::string("no usable CUDA device (there is no CPU fallback): ") + cudaGetErrorString(err));
    CDX_CHECK(device >= 0 && device < count, "engine_create: device %d out of range (count %d)", device, count);
    CDX_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    CDX_CUDA(cudaGetDeviceProperties(&prop, device));
    cdx_engine* eng = new cdx_engine();
    eng->e.device = device;
    if (prop.major != 9 || prop.minor != 0)
      throw Error(CDX_E_CUDA, "libcdx is built for sm_90a (H100) only; device " + std::to_string(device) + " is sm_" +
                                  std::to_string(prop.major) + std::to_string(prop.minor));
    eng->e.num_sms = prop.multiProcessorCount;
    const char* persist = getenv("CDX_PERSIST");
    eng->e.persist = persist == nullptr || atoi(persist) != 0;
    *out = eng;
  });
}
void cdx_engine_destroy(cdx_engine* e) {
  if (!e) return;
  cudaSetDevice(e->e.device);
  cudaDeviceSynchronize();
  e->e.arena.destroy();
  if (e->e.done_ev) cudaEventDestroy(e->e.done_ev);
  if (e->e.side) cudaStreamDestroy(e->e.side);
  if (e->e.fork_ev) cudaEventDestroy(e->e.fork_ev);
  if (e->e.join_ev) cudaEventDestroy(e->e.join_ev);
  if (e->e.amax_pool) cudaFree(e->e.amax_pool);
  delete e;
}
size_t cdx_engine_workspace_bytes(const cdx_engine* e) { return e ? e->e.arena.cap : 0; }
uint64_t cdx_engine_launch_count(const cdx_engine* e) { return e ? e->e.launches : 0; }
int cdx_engine_set_mma_mode(cdx_engine* e, int mode) {
  return guard([&] {
    CDX_CHECK(e != nullptr && mode >= 0 && mode <= 5, "set_mma_mode: bad arguments");
    e->e.mma_mode = mode == 0 ? 0 : 1;       // 2 = tensor-core contractions but unfused attention (A/B comparisons)
    e->e.flash_attn = mode != 2 && mode != 0;
    e->e.tc_kind = mode == 3 ? 0 : mode >= 4 ? 2 : 1;    // 3 = 3xTF32 contractions, 4 / 5 = single-term fp16, else fp16 split
    e->e.attn_one = mode == 5;                            // 5 = as 4, plus one-term fused attention ("autocast")
  });
}

int cdx_engine_set_persist(cdx_engine* e, int enable, int max_ctas) {
  return guard([&] {
    CDX_CHECK(e != nullptr && max_ctas >= 0, "set_persist: bad arguments");
    e->e.persist = enable != 0;
    e->e.persist_grid = max_ctas;
  });
}

int cdx_engine_profile(cdx_engine* e, int enable) {
  return guard([&] {
    CDX_CHECK(e != nullptr, "profile: null engine");
    CDX_CUDA(cudaSetDevice(e->e.device));
    CDX_CUDA(cudaDeviceSynchronize());
    for (ProfRec& r : e->e.prof.recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    e->e.prof.recs.clear();
    e->e.prof.on = enable != 0;
  });
}
int cdx_engine_profile_read(cdx_engine* e, int tag, double* ms, double* flops, double* bytes, uint64_t* launches) {
  return guard([&] {
    CDX_CHECK(e && ms && flops && bytes && launches && tag >= 0 && tag < PROF_NTAGS, "profile_read: bad arguments");
    CDX_CUDA(cudaSetDevice(e->e.device));
    CDX_CUDA(cudaDeviceSynchronize());
    *ms = 0; *flops = 0; *bytes = 0; *launches = 0;
    const bool dump = getenv("CDX_PROF_DUMP") != nullptr;
    for (const ProfRec& r : e->e.prof.recs) {
      if (r.tag != tag) continue;
      float t = 0.f;
      CDX_CUDA(cudaEventElapsedTime(&t, r.a, r.b));
      if (dump) fprintf(stderr, "[cdx prof] tag %d  %8.3f ms  %8.1f GFLOP  %7.1f TF/s  %s\n", tag, t, r.flops * 1e-9, t > 0 ? r.flops / (t * 1e9) : 0.0, r.note);
      *ms += t; *flops += r.flops; *bytes += r.bytes; *launches += (uint64_t)r.launches;
    }
  });
}

// ---------------------------------------------------------------- networks
int cdx_unet_create(cdx_engine* e, const cdx_unet_config* cfg, cdx_net** out) {
  return guard([&] {
    CDX_CHECK(cfg && out, "unet_create: null argument");
    cdx_net* h = new cdx_net();
    h->owner = e;
    static Engine host_only;   // inventory-only nets (e == NULL) can be built without a GPU
    h->n = make_unet(e ? &e->e : &host_only, *cfg);
    *out = h;
  });
}
int cdx_vae_create(cdx_engine* e, const cdx_vae_config* cfg, cdx_net** out) {
  return guard([&] {
    CDX_CHECK(cfg && out, "vae_create: null argument");
    cdx_net* h = new cdx_net();
    h->owner = e;
    static Engine host_only;
    h->n = make_vae(e ? &e->e : &host_only, *cfg);
    *out = h;
  });
}
int cdx_text_create(cdx_engine* e, const cdx_text_config* cfg, cdx_net** out) {
  return guard([&] {
    CDX_CHECK(cfg && out, "text_create: null argument");
    cdx_net* h = new cdx_net();
    h->owner = e;
    static Engine host_only;
    h->n = make_text(e ? &e->e : &host_only, *cfg);
    *out = h;
  });
}
void cdx_net_destroy(cdx_net* n) {
  if (!n) return;
  destroy_net(n->n);
  delete n;
}
int cdx_net_num_params(const cdx_net* n) { return n ? (int)n->n->params.size() : 0; }
const char* cdx_net_param_name(const cdx_net* n, int i) {
  if (!n || i < 0 || i >= (int)n->n->params.size()) return nullptr;
  return n->n->params[i].name.c_str();
}
int cdx_net_param_shape(const cdx_net* n, int i, int64_t dims[4]) {
  if (!n || i < 0 || i >= (int)n->n->params.size()) return CDX_E_INVALID;
  const Param& p = n->n->params[i];
  for (int k = 0; k < 4; ++k) dims[k] = k < p.rank ? p.dims[k] : 1;
  return p.rank;
}
int cdx_net_load_param(cdx_net* n, const char* name, const float* data, int on_device, const int64_t* dims, int rank) {
  return guard([&] {
    CDX_CHECK(n && n->owner && name && data && dims, "load_param: null argument (nets created without an engine are inventory-only)");
    net_load_param(*n->n, name, data, on_device != 0, dims, rank);
  });
}
int cdx_net_finalize(cdx_net* n) {
  return guard([&] {
    CDX_CHECK(n && n->owner, "finalize: null / inventory-only net");
    net_finalize(*n->n);
  });
}
int cdx_net_weight_blob(cdx_net* n, void** dev_ptr, size_t* bytes) {
  return guard([&] {
    CDX_CHECK(n && n->owner && dev_ptr && bytes, "weight_blob: null argument");
    net_ensure_blob(*n->n);
    *dev_ptr = n->n->blob;
    *bytes = n->n->blob_floats * sizeof(float);
  });
}
int cdx_net_adopt_blob(cdx_net* n) {
  return guard([&] {
    CDX_CHECK(n && n->owner, "adopt_blob: null / inventory-only net");
    net_ensure_blob(*n->n);
    for (Param& p : n->n->params) p.loaded = true;
    // the blob contents changed under us: everything derived from it (operand planes, cached context K/V) is stale
    n->n->planes_valid = false;
    n->n->ctxkv.valid = false;
    n->n->finalized = false;
    net_finalize(*n->n);
  });
}
int cdx_unet_set_time_freqs(cdx_net* n, const float* freqs, int half) {
  return guard([&] {
    CDX_CHECK(n && freqs, "set_time_freqs: null argument");
    CDX_CHECK(n->n->kind != NET_VAE, "set_time_freqs on a VAE");
    CDX_CHECK(half == n->n->ucfg.model_channels / 2, "set_time_freqs: half=%d, expected %d", half, n->n->ucfg.model_channels / 2);
    n->n->freqs_host.assign(freqs, freqs + half);
    if (n->n->finalized) net_finalize(*n->n);
  });
}

int cdx_unet_set_prediction(cdx_net* n, int prediction, const float* sa_v, const float* s1_v, int T) {
  return guard([&] {
    CDX_CHECK(n && n->n, "set_prediction: null net");
    CDX_CHECK(n->n->kind == NET_UNET_OPENAI, "set_prediction: SD / LDM U-Nets only");
    CDX_CHECK(prediction == CDX_PRED_EPS || prediction == CDX_PRED_V, "set_prediction: prediction %d", prediction);
    if (prediction == CDX_PRED_EPS) {
      n->n->pred = 0; n->n->sa_v.clear(); n->n->s1_v.clear();
      return;
    }
    CDX_CHECK(sa_v && s1_v && T > 0, "set_prediction: v needs both tables");
    n->n->sa_v.assign(sa_v, sa_v + T);
    n->n->s1_v.assign(s1_v, s1_v + T);
    n->n->pred = 1;
  });
}

int cdx_unet_forward(cdx_net* n, const float* x, const float* t_dev, const float* ctx, int ctx_len, float* out, int B, int H, int W,
                     void* stream) {
  return guard([&] {
    CDX_CHECK(n && n->owner && x && t_dev && out && B > 0, "unet_forward: bad arguments");
    with_arena(n->owner->e, S(stream), [&] { unet_forward(*n->n, x, t_dev, ctx, ctx_len, out, B, H, W, S(stream)); });
  });
}
int cdx_vae_encode_hw(cdx_net* n, const float* img, float* moments, int B, int H, int W, void* stream) {
  return guard([&] {
    CDX_CHECK(n && n->owner && img && moments && B > 0, "vae_encode: bad arguments");
    with_arena(n->owner->e, S(stream), [&] { vae_encode(*n->n, img, moments, B, H, W, S(stream)); });
  });
}
int cdx_vae_encode(cdx_net* n, const float* img, float* moments, int B, int R, void* stream) {
  return cdx_vae_encode_hw(n, img, moments, B, R, R, stream);
}
int cdx_text_encode(cdx_net* n, const int* ids, int B, int L, float* out, void* stream) {
  return guard([&] {
    CDX_CHECK(n && n->owner && ids && out && B > 0, "text_encode: bad arguments");
    with_arena(n->owner->e, S(stream), [&] { text_encode(*n->n, ids, out, B, L, S(stream)); });
  });
}
#define ENG_CALL_(EH_, ...)                                \
  return guard([&] {                                       \
    CDX_CHECK((EH_) != nullptr, "null engine");            \
    CDX_CUDA(cudaSetDevice(engine_of(EH_).device));        \
    __VA_ARGS__;                                           \
  })
int cdx_text_features(cdx_net* n, const int* ids, int B, int L, float* out, void* stream) {
  return guard([&] {
    CDX_CHECK(n && n->owner && ids && out && B > 0, "text_features: bad arguments");
    with_arena(n->owner->e, S(stream), [&] { text_features(*n->n, ids, out, B, L, S(stream)); });
  });
}
int cdx_clip_image_features(cdx_net* n, const float* pixels, int B, float* out, void* stream) {
  return guard([&] {
    CDX_CHECK(n && n->owner && pixels && out && B > 0, "clip_image_features: bad arguments");
    with_arena(n->owner->e, S(stream), [&] { clip_image_features(*n->n, pixels, out, B, S(stream)); });
  });
}
int cdx_clip_preprocess(cdx_engine* e, const float* img, int B, int R, int size, float* out, void* s) {
  ENG_CALL_(e, CDX_CHECK(img && out && B > 0 && R > 0 && size > 0, "clip_preprocess: bad arguments"); clip_preprocess(e->e, img, B, R, size, out, S(s)));
}
int cdx_dclip_scores(cdx_engine* e, const float* img_f, const float* orig_f, const float* enc_f, const float* dec_f, int B, int D, float* clip_out,
                     float* dclip_out, void* s) {
  ENG_CALL_(e, CDX_CHECK(img_f && orig_f && enc_f && dec_f && clip_out && dclip_out && B > 0 && D > 0, "dclip_scores: bad arguments");
            dclip_scores(e->e, img_f, orig_f, enc_f, dec_f, B, D, clip_out, dclip_out, S(s)));
}
int cdx_image_metrics(cdx_engine* eh, const float* a, const float* b, int B, int H, int W, float* out, void* stream) {
  return guard([&] {
    CDX_CHECK(eh && a && b && out && B > 0, "image_metrics: bad arguments");
    with_arena(eh->e, S(stream), [&] { image_metrics(eh->e, a, b, B, H, W, out, S(stream)); });
  });
}
int cdx_vae_decode_hw(cdx_net* n, const float* z, float* img, int B, int h, int w, void* stream) {
  return guard([&] {
    CDX_CHECK(n && n->owner && z && img && B > 0, "vae_decode: bad arguments");
    with_arena(n->owner->e, S(stream), [&] { vae_decode(*n->n, z, img, B, h, w, S(stream)); });
  });
}
int cdx_vae_decode(cdx_net* n, const float* z, float* img, int B, int h, void* stream) {
  return cdx_vae_decode_hw(n, z, img, B, h, h, stream);
}

// ---------------------------------------------------------------- per-step kernels
#define ENG_CALL(EH_, ...)                                 \
  return guard([&] {                                       \
    CDX_CHECK((EH_) != nullptr, "null engine");            \
    CDX_CUDA(cudaSetDevice(engine_of(EH_).device));        \
    __VA_ARGS__;                                           \
  })

int cdx_affine(cdx_engine* e, const float* x, float a, float b, float* out, size_t n, void* s) { ENG_CALL(e, affine(e->e, x, a, b, out, n, S(s))); }
int cdx_shift_scale(cdx_engine* e, const float* x, float b, float a, float* out, size_t n, void* s) { ENG_CALL(e, shift_scale(e->e, x, b, a, out, n, S(s))); }
int cdx_q_sample(cdx_engine* e, const float* x0, const float* nz, float sa, float s1, float* out, size_t n, void* s) {
  ENG_CALL(e, q_sample(e->e, x0, nz, sa, s1, out, n, S(s)));
}
int cdx_vae_posterior(cdx_engine* e, const float* mom, const float* nz, float sf, float* out, int B, int C, int hw, void* s) {
  ENG_CALL(e, vae_posterior(e->e, mom, nz, sf, out, B, C, hw, S(s)));
}
int cdx_ddim_posterior_sample(cdx_engine* e, const float* x0, const float* xt, const float* nz, const cdx_ddim_coef* c, float* o, size_t n, void* s) {
  ENG_CALL(e, CDX_CHECK(c, "null coef"); ddim_posterior_sample(e->e, x0, xt, nz, *c, o, n, S(s)));
}
int cdx_ddim_compute_eps(cdx_engine* e, const float* xt, const float* xn, const float* e_c, const float* e_uc, float scale, const cdx_ddim_coef* c,
                         float* o, size_t n, void* s) {
  ENG_CALL(e, CDX_CHECK(c, "null coef"); ddim_compute_eps(e->e, xt, xn, e_c, e_uc, scale, *c, o, n, S(s)));
}
int cdx_ddim_step_with_eps(cdx_engine* e, const float* x, const float* e_c, const float* e_uc, float scale, const float* eps, const cdx_ddim_coef* c,
                           float* o, size_t n, void* s) {
  ENG_CALL(e, CDX_CHECK(c, "null coef"); ddim_step_with_eps(e->e, x, e_c, e_uc, scale, eps, *c, o, n, S(s)));
}
int cdx_pixel_posterior_sample(cdx_engine* e, const float* x0, const float* xt, const float* nz, const cdx_pixel_coef* c, float* o, size_t n, void* s) {
  ENG_CALL(e, CDX_CHECK(c, "null coef"); pixel_posterior_sample(e->e, x0, xt, nz, *c, o, n, S(s)));
}
int cdx_pixel_compute_eps(cdx_engine* e, const float* xt, const float* xn, const float* et, const cdx_pixel_coef* c, float* o, int B, int chw,
                          int net_chw, void* s) {
  ENG_CALL(e, CDX_CHECK(c, "null coef"); pixel_compute_eps(e->e, xt, xn, et, *c, o, B, chw, net_chw, S(s)));
}
int cdx_pixel_step_with_eps(cdx_engine* e, const float* xt, const float* et, const float* eps, const cdx_pixel_coef* c, float* o, int B, int chw,
                            int net_chw, void* s) {
  ENG_CALL(e, CDX_CHECK(c, "null coef"); pixel_step_with_eps(e->e, xt, et, eps, *c, o, B, chw, net_chw, S(s)));
}

// ---------------------------------------------------------------- loop drivers
int cdx_latent_encode(cdx_net* un, const float* x0, const float* c, const float* uc, int L, float scale, const cdx_ddim_coef* coef,
                      const float* t_host, int n_steps, int n_rec, const float* noise, float sqrt_a_T, float sqrt_1ma_T, float* z_out, int B,
                      int C, int h, int w, void* stream) {
  return guard([&] {
    CDX_CHECK(un && un->owner && x0 && (c || L == 0) && coef && t_host && noise && z_out, "latent_encode: null argument");
    CDX_CHECK(n_steps >= 1 && n_rec >= 0 && n_rec <= n_steps, "latent_encode: n_steps=%d n_rec=%d", n_steps, n_rec);
    for (int i = 0; i < n_rec; ++i) CDX_CHECK(coef[i].sigma > 0.f, "latent_encode: eta must be > 0 (sigma[%d] == 0), ddim.py:268", i);
    const std::vector<float> scales((size_t)std::max(B, 0), scale);
    ChainLoopArgs a;
    a.n_src = B; a.src = true;
    a.x0 = x0; a.c_src = c; a.uc = uc; a.L = L; a.s_scales = scales.data();
    a.coef = coef; a.t_host = t_host; a.n_steps = n_steps; a.n_rec = n_rec; a.noise = noise; a.sa = sqrt_a_T; a.s1 = sqrt_1ma_T;
    a.z_out = z_out; a.C = C; a.h = h; a.w = w;
    with_arena(un->owner->e, S(stream), [&] { run_latent_chains(*un->n, a, S(stream)); });
  });
}

int cdx_latent_decode(cdx_net* un, const float* z, int n_eps, const float* c, const float* uc, int L, float scale, const cdx_ddim_coef* coef,
                      const float* t_host, int n_steps, const float* extra_noise, float* x_out, int B, int C, int h, int w, void* stream) {
  return guard([&] {
    CDX_CHECK(un && un->owner && z && (c || L == 0) && coef && t_host && x_out, "latent_decode: null argument");
    CDX_CHECK(n_steps >= 1 && n_eps >= 0, "latent_decode: n_steps=%d n_eps=%d", n_steps, n_eps);
    CDX_CHECK(n_eps >= n_steps || extra_noise != nullptr, "latent_decode: %d steps but only %d recovered noises and no extra noise", n_steps, n_eps);
    const std::vector<float> scales((size_t)std::max(B, 0), scale);
    ChainLoopArgs a;
    a.n_src = B; a.K = 1;
    a.c_tgt = c; a.uc = uc; a.L = L; a.t_scales = scales.data();
    a.coef = coef; a.t_host = t_host; a.n_steps = n_steps;
    a.z_in = z; a.n_eps = n_eps; a.extra = extra_noise; a.x_out = x_out;
    a.C = C; a.h = h; a.w = w;
    with_arena(un->owner->e, S(stream), [&] { run_latent_chains(*un->n, a, S(stream)); });
  });
}

int cdx_cycle_lockstep(cdx_net* un, const float* x0, const float* c_src, const float* c_tgt, const float* uc, int L, float src_scale,
                       float tgt_scale, const cdx_ddim_coef* coef, const float* t_host, int n_steps, const float* noise, float sqrt_a_T,
                       float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w, void* stream) {
  return cdx_cycle_lockstep_masked(un, x0, c_src, c_tgt, uc, L, src_scale, tgt_scale, coef, t_host, n_steps, noise, sqrt_a_T, sqrt_1ma_T,
                                   x_out, z_out, B, C, h, w, stream, nullptr);
}

int cdx_cycle_lockstep_masked(cdx_net* un, const float* x0, const float* c_src, const float* c_tgt, const float* uc, int L, float src_scale,
                              float tgt_scale, const cdx_ddim_coef* coef, const float* t_host, int n_steps, const float* noise,
                              float sqrt_a_T, float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w, void* stream,
                              const float* mask) {
  return cdx_cycle_lockstep_ctl(un, x0, c_src, c_tgt, uc, L, src_scale, tgt_scale, coef, t_host, n_steps, noise, sqrt_a_T, sqrt_1ma_T,
                                x_out, z_out, B, C, h, w, stream, mask, nullptr);
}

int cdx_cycle_lockstep_ctl(cdx_net* un, const float* x0, const float* c_src, const float* c_tgt, const float* uc, int L, float src_scale,
                           float tgt_scale, const cdx_ddim_coef* coef, const float* t_host, int n_steps, const float* noise,
                           float sqrt_a_T, float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w, void* stream,
                           const float* mask, const cdx_attn_control* ctl) {
  return cdx_cycle_lockstep_refine(un, x0, c_src, c_tgt, uc, L, src_scale, tgt_scale, coef, t_host, n_steps, noise, sqrt_a_T, sqrt_1ma_T,
                                   x_out, z_out, B, C, h, w, stream, mask, ctl, nullptr);
}

// the single-image lock-step cycle under the controls of ChainLoopArgs (ctl, own_weight; mutual with start_step >= 0; pnp)
static int cycle_lockstep(cdx_net* un, const float* x0, const float* c_src, const float* c_tgt, const float* uc, int L, float src_scale,
                          float tgt_scale, const cdx_ddim_coef* coef, const float* t_host, int n_steps, const float* noise, float sqrt_a_T,
                          float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w, void* stream, const float* mask,
                          const cdx_attn_control* ctl, const float* own_weight, bool mutual, int start_step, int start_layer,
                          const PnpLoop* pnp = nullptr, const cdx_semantic_guidance* sega = nullptr, const float* c_edit = nullptr,
                          const cdx_semantic_attn_mask* sega_mask = nullptr, const cdx_sampler* sampler = nullptr,
                          const cdx_local_blend* blend = nullptr) {
  return guard([&] {
    CDX_CHECK(un && un->owner && x0 && c_src && c_tgt && coef && t_host && noise && x_out, "cycle_lockstep: null argument");
    CDX_CHECK(n_steps >= 1, "cycle_lockstep: n_steps=%d", n_steps);
    for (int i = 0; i < n_steps; ++i) CDX_CHECK(coef[i].sigma > 0.f, "cycle_lockstep: eta must be > 0 (sigma[%d] == 0), ddim.py:268", i);
    const std::vector<float> s_scales((size_t)std::max(B, 0), src_scale), t_scales((size_t)std::max(B, 0), tgt_scale);
    ChainLoopArgs a;
    a.n_src = B; a.K = 1; a.src = true;
    a.x0 = x0; a.c_src = c_src; a.c_tgt = c_tgt; a.uc = uc; a.L = L; a.s_scales = s_scales.data(); a.t_scales = t_scales.data();
    a.coef = coef; a.t_host = t_host; a.n_steps = n_steps; a.n_rec = n_steps; a.noise = noise; a.sa = sqrt_a_T; a.s1 = sqrt_1ma_T;
    a.z_out = z_out; a.x_out = x_out; a.mask = mask; a.ctl = ctl; a.own_weight = own_weight; a.C = C; a.h = h; a.w = w;
    a.mutual = mutual; a.start_step = start_step; a.start_layer = start_layer; a.pnp = pnp;
    a.sega = sega; a.c_edit = c_edit; a.sega_mask = sega_mask; a.sampler = sampler; a.blend = blend;
    with_arena(un->owner->e, S(stream), [&] { run_latent_chains(*un->n, a, S(stream)); });
  });
}

int cdx_cycle_lockstep_refine(cdx_net* un, const float* x0, const float* c_src, const float* c_tgt, const float* uc, int L, float src_scale,
                              float tgt_scale, const cdx_ddim_coef* coef, const float* t_host, int n_steps, const float* noise,
                              float sqrt_a_T, float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w, void* stream,
                              const float* mask, const cdx_attn_control* ctl, const float* own_weight) {
  return cycle_lockstep(un, x0, c_src, c_tgt, uc, L, src_scale, tgt_scale, coef, t_host, n_steps, noise, sqrt_a_T, sqrt_1ma_T, x_out, z_out,
                        B, C, h, w, stream, mask, ctl, own_weight, false, 0, 0);
}

int cdx_cycle_lockstep_mutual(cdx_net* un, const float* x0, const float* c_src, const float* c_tgt, const float* uc, int L, float src_scale,
                              float tgt_scale, const cdx_ddim_coef* coef, const float* t_host, int n_steps, const float* noise,
                              float sqrt_a_T, float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w, void* stream,
                              const float* mask, int start_step, int start_layer) {
  return cycle_lockstep(un, x0, c_src, c_tgt, uc, L, src_scale, tgt_scale, coef, t_host, n_steps, noise, sqrt_a_T, sqrt_1ma_T, x_out, z_out,
                        B, C, h, w, stream, mask, nullptr, nullptr, true, start_step, start_layer);
}

int cdx_cycle_lockstep_pnp(cdx_net* un, const float* x0, const float* c_src, const float* c_tgt, const float* uc, int L, float src_scale,
                           float tgt_scale, const cdx_ddim_coef* coef, const float* t_host, int n_steps, const float* noise,
                           float sqrt_a_T, float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w, void* stream,
                           const float* mask, int feature_steps, int attention_steps, int attention_start_layer, const int* feature_blocks,
                           int n_feature_blocks) {
  PnpLoop p;
  p.feature_steps = feature_steps; p.attention_steps = attention_steps; p.start_layer = attention_start_layer;
  p.blocks = feature_blocks; p.n_blocks = n_feature_blocks;
  return cycle_lockstep(un, x0, c_src, c_tgt, uc, L, src_scale, tgt_scale, coef, t_host, n_steps, noise, sqrt_a_T, sqrt_1ma_T, x_out, z_out,
                        B, C, h, w, stream, mask, nullptr, nullptr, false, 0, 0, &p);
}

int cdx_cycle_lockstep_semantic(cdx_net* un, const float* x0, const float* c_src, const float* c_tgt, const float* uc, int L, float src_scale,
                                float tgt_scale, const cdx_ddim_coef* coef, const float* t_host, int n_steps, const float* noise,
                                float sqrt_a_T, float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w, void* stream,
                                const float* mask, const float* c_edit, const cdx_semantic_guidance* sg) {
  if (!sg || !c_edit) return guard([] { throw Error(CDX_E_INVALID, "cycle_lockstep_semantic: null guidance or concept contexts"); });
  return cycle_lockstep(un, x0, c_src, c_tgt, uc, L, src_scale, tgt_scale, coef, t_host, n_steps, noise, sqrt_a_T, sqrt_1ma_T, x_out, z_out,
                        B, C, h, w, stream, mask, nullptr, nullptr, false, 0, 0, nullptr, sg, c_edit);
}

int cdx_cycle_lockstep_semantic_attn(cdx_net* un, const float* x0, const float* c_src, const float* c_tgt, const float* uc, int L,
                                     float src_scale, float tgt_scale, const cdx_ddim_coef* coef, const float* t_host, int n_steps,
                                     const float* noise, float sqrt_a_T, float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w,
                                     void* stream, const float* mask, const float* c_edit, const cdx_semantic_guidance* sg,
                                     const cdx_semantic_attn_mask* am) {
  if (!sg || !c_edit || !am)
    return guard([] { throw Error(CDX_E_INVALID, "cycle_lockstep_semantic_attn: null guidance, concept contexts or mask settings"); });
  return cycle_lockstep(un, x0, c_src, c_tgt, uc, L, src_scale, tgt_scale, coef, t_host, n_steps, noise, sqrt_a_T, sqrt_1ma_T, x_out, z_out,
                        B, C, h, w, stream, mask, nullptr, nullptr, false, 0, 0, nullptr, sg, c_edit, am);
}

int cdx_cycle_lockstep_sampler(cdx_net* un, const float* x0, const float* c_src, const float* c_tgt, const float* uc, int L, float src_scale,
                               float tgt_scale, const cdx_ddim_coef* coef, const float* t_host, int n_steps, const float* noise,
                               float sqrt_a_T, float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w, void* stream,
                               const cdx_sampler* sampler, const float* mask, const cdx_attn_control* ctl, const float* own_weight,
                               const cdx_mutual_control* mutual, const cdx_pnp_control* pnp, const float* c_edit,
                               const cdx_semantic_guidance* sg, const cdx_semantic_attn_mask* am) {
  if (!sampler) return guard([] { throw Error(CDX_E_INVALID, "cycle_lockstep_sampler: null sampler"); });
  PnpLoop p;
  if (pnp) {
    p.feature_steps = pnp->feature_steps; p.attention_steps = pnp->attention_steps; p.start_layer = pnp->attention_start_layer;
    p.blocks = pnp->feature_blocks; p.n_blocks = pnp->n_feature_blocks;
  }
  return cycle_lockstep(un, x0, c_src, c_tgt, uc, L, src_scale, tgt_scale, coef, t_host, n_steps, noise, sqrt_a_T, sqrt_1ma_T, x_out, z_out,
                        B, C, h, w, stream, mask, ctl, own_weight, mutual != nullptr, mutual ? mutual->start_step : 0,
                        mutual ? mutual->start_layer : 0, pnp ? &p : nullptr, sg, c_edit, am, sampler);
}

int cdx_cycle_lockstep_blend(cdx_net* un, const float* x0, const float* c_src, const float* c_tgt, const float* uc, int L, float src_scale,
                             float tgt_scale, const cdx_ddim_coef* coef, const float* t_host, int n_steps, const float* noise,
                             float sqrt_a_T, float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w, void* stream,
                             const cdx_sampler* sampler, const float* mask, const cdx_attn_control* ctl, const float* own_weight,
                             const cdx_mutual_control* mutual, const cdx_pnp_control* pnp, const float* c_edit,
                             const cdx_semantic_guidance* sg, const cdx_semantic_attn_mask* am, const cdx_local_blend* blend) {
  if (!blend) return guard([] { throw Error(CDX_E_INVALID, "cycle_lockstep_blend: null LocalBlend"); });
  if (mutual || pnp || c_edit || sg || am)
    return guard([] { throw Error(CDX_E_INVALID, "cycle_lockstep_blend: LocalBlend runs with Prompt-to-Prompt edits or none"); });
  return cycle_lockstep(un, x0, c_src, c_tgt, uc, L, src_scale, tgt_scale, coef, t_host, n_steps, noise, sqrt_a_T, sqrt_1ma_T, x_out, z_out,
                        B, C, h, w, stream, mask, ctl, own_weight, false, 0, 0, nullptr, nullptr, nullptr, nullptr, sampler, blend);
}

int cdx_latent_loop_ens(cdx_net* un, int mode, const float* x0, const float* c_src, const float* c_tgt, const float* uc, int L,
                        const float* src_scales, const float* tgt_scales, const cdx_ddim_coef* coef, const float* t_host, int n_steps, int n_rec,
                        const float* noise, float sqrt_a_T, float sqrt_1ma_T, const float* z_in, int n_eps, const float* extra_noise,
                        float* z_out, float* x_out, int B, int C, int h, int w, void* stream) {
  return guard([&] {
    CDX_CHECK(un && un->owner && coef && t_host && mode >= 1 && mode <= 3, "latent_loop_ens: bad arguments (mode %d)", mode);
    const bool enc = mode & 1, dec = mode & 2;            // 1 encode, 2 decode, 3 both in lock-step
    CDX_CHECK(n_steps >= 1, "latent_loop_ens: n_steps=%d", n_steps);
    ChainLoopArgs a;
    a.n_src = B; a.K = dec; a.src = enc; a.scales_on_device = true;
    a.uc = uc; a.L = L; a.coef = coef; a.t_host = t_host; a.n_steps = n_steps;
    a.C = C; a.h = h; a.w = w;
    if (enc) {
      CDX_CHECK(x0 && c_src && noise && src_scales && uc, "latent_loop_ens: the encode chain needs x0, c_src, uc, noise and per-sample scales");
      if (dec) n_rec = n_steps;
      CDX_CHECK(n_rec >= 0 && n_rec <= n_steps, "latent_loop_ens: n_rec=%d", n_rec);
      for (int i = 0; i < n_rec; ++i) CDX_CHECK(coef[i].sigma > 0.f, "latent_loop_ens: eta must be > 0 (sigma[%d] == 0), ddim.py:268", i);
      CDX_CHECK(dec || z_out, "latent_loop_ens: encode needs z_out");
      a.x0 = x0; a.c_src = c_src; a.s_scales = src_scales; a.n_rec = n_rec; a.noise = noise; a.sa = sqrt_a_T; a.s1 = sqrt_1ma_T; a.z_out = z_out;
    }
    if (dec) {
      CDX_CHECK(c_tgt && tgt_scales && uc && x_out, "latent_loop_ens: the decode chain needs c_tgt, uc, per-sample scales and x_out");
      a.c_tgt = c_tgt; a.t_scales = tgt_scales; a.x_out = x_out;
      if (!enc) {
        CDX_CHECK(z_in && n_eps >= 0 && (n_eps >= n_steps || extra_noise), "latent_loop_ens: decode needs z (%d noises for %d steps) or extra noise", n_eps, n_steps);
        a.z_in = z_in; a.n_eps = n_eps; a.extra = extra_noise;
      }
    }
    with_arena(un->owner->e, S(stream), [&] { run_latent_chains(*un->n, a, S(stream)); });
  });
}

int cdx_pixel_encode(cdx_net* un, const float* x0, const cdx_pixel_coef* coef, const float* t_host, int n_rec, const float* noise,
                     float sqrt_a_T, float sqrt_1ma_T, float* z_out, int B, int C, int R, void* stream) {
  return guard([&] {
    CDX_CHECK(un && un->owner && x0 && noise && z_out, "pixel_encode: null argument");
    CDX_CHECK(n_rec >= 0 && (n_rec == 0 || (coef && t_host)), "pixel_encode: n_rec=%d", n_rec);
    Engine& e = un->owner->e;
    Net& unet = *un->n;
    cudaStream_t s = S(stream);
    const int chw = C * R * R;
    const int net_chw = unet.ucfg.out_channels * R * R;
    const size_t n = (size_t)B * chw;
    with_arena(e, s, [&] {
      Scope sc(e.arena);
      float* xt = (float*)e.arena.alloc(n * sizeof(float));
      float* xn = (float*)e.arena.alloc(n * sizeof(float));
      float* eps = (float*)e.arena.alloc(n * sizeof(float));
      float* et = (float*)e.arena.alloc((size_t)B * net_chw * sizeof(float));
      float* tdev = (float*)e.arena.alloc((size_t)std::max(n_rec, 1) * B * sizeof(float));
      upload_timesteps(e, t_host, n_rec, B, tdev, s);
      q_sample(e, x0, noise, sqrt_a_T, sqrt_1ma_T, xt, n, s);                          // sample_xt, DW:310-314 (incl. the DW:483 index quirk)
      scatter_slot(e, xt, z_out, B, chw, n_rec + 1, 0, s);
      const int iters = e.dry() ? std::min(n_rec, 1) : n_rec;
      for (int i = 0; i < iters; ++i) {
        pixel_posterior_sample(e, x0, xt, noise + (size_t)(1 + i) * n, coef[i], xn, n, s);
        unet_forward(unet, xt, tdev + (size_t)i * B, nullptr, 0, et, B, R, R, s);
        pixel_compute_eps(e, xt, xn, et, coef[i], eps, B, chw, net_chw, s);
        scatter_slot(e, eps, z_out, B, chw, n_rec + 1, 1 + i, s);
        std::swap(xt, xn);
      }
    });
  });
}

int cdx_pixel_decode(cdx_net* un, const float* z, int n_eps, const cdx_pixel_coef* coef, const float* t_host, int n_steps,
                     const float* last_noise, float* x_out, int B, int C, int R, void* stream) {
  return guard([&] {
    CDX_CHECK(un && un->owner && z && coef && t_host && x_out, "pixel_decode: null argument");
    CDX_CHECK(n_steps >= 1 && n_eps >= 0 && n_eps <= n_steps, "pixel_decode: n_steps=%d n_eps=%d", n_steps, n_eps);
    Engine& e = un->owner->e;
    Net& unet = *un->n;
    cudaStream_t s = S(stream);
    const int chw = C * R * R;
    const int net_chw = unet.ucfg.out_channels * R * R;
    const size_t n = (size_t)B * chw;
    with_arena(e, s, [&] {
      Scope sc(e.arena);
      float* xa = (float*)e.arena.alloc(n * sizeof(float));
      float* xb = (float*)e.arena.alloc(n * sizeof(float));
      float* eps = (float*)e.arena.alloc(n * sizeof(float));
      float* et = (float*)e.arena.alloc((size_t)B * net_chw * sizeof(float));
      float* tdev = (float*)e.arena.alloc((size_t)n_steps * B * sizeof(float));
      upload_timesteps(e, t_host, n_steps, B, tdev, s);
      gather_slot(e, z, xa, B, chw, n_eps + 1, 0, s);
      const int iters = e.dry() ? 1 : n_steps;
      for (int i = 0; i < iters; ++i) {
        unet_forward(unet, xa, tdev + (size_t)i * B, nullptr, 0, et, B, R, R, s);
        const float* nz = nullptr;
        if (i < n_eps) { gather_slot(e, z, eps, B, chw, n_eps + 1, 1 + i, s); nz = eps; }
        else if (last_noise) nz = last_noise + (size_t)(i - n_eps) * n;
        float* dst = (i == n_steps - 1) ? x_out : xb;
        pixel_step_with_eps(e, xa, et, nz, coef[i], dst, B, chw, net_chw, s);
        std::swap(xa, xb);
      }
    });
  });
}

int cdx_pixel_cycle_lockstep(cdx_net* src, cdx_net* tgt, const float* x0, const cdx_pixel_coef* coef, const float* t_host, int i0, int i1,
                             const float* noise, float sqrt_a_T, float sqrt_1ma_T, float* state, int B, int C, int R, void* stream) {
  return guard([&] {
    CDX_CHECK(src && src->owner && tgt && tgt->owner && x0 && noise && state && B > 0, "pixel_cycle_lockstep: null argument");
    CDX_CHECK(i0 >= 0 && i1 >= i0 && (i1 == i0 || (coef && t_host)), "pixel_cycle_lockstep: steps [%d, %d)", i0, i1);
    Engine& es = src->owner->e;
    Engine& et = tgt->owner->e;
    cudaStream_t s = S(stream);
    const int chw = C * R * R, steps = i1 - i0;
    const int net_chw_s = src->n->ucfg.out_channels * R * R, net_chw_t = tgt->n->ucfg.out_channels * R * R;
    const size_t n = (size_t)B * chw;
    float* xs = state;
    float* ys = state + n;
    with_arena(es, s, [&] {
      Scope sc_s(es.arena), sc_t(et.arena);
      float* e_src = (float*)es.arena.alloc((size_t)B * net_chw_s * sizeof(float));
      float* e_tgt = (float*)et.arena.alloc((size_t)B * net_chw_t * sizeof(float));
      float* tdev = (float*)es.arena.alloc((size_t)std::max(steps, 1) * B * sizeof(float));
      if (steps) upload_timesteps(es, t_host + i0, steps, B, tdev, s);
      const float* nz = noise;
      if (i0 == 0) {                                                                      // sample_xt, DW:310-314 (incl. the DW:483 index quirk)
        q_sample(es, x0, nz, sqrt_a_T, sqrt_1ma_T, xs, n, s);
        copy_dd(es, xs, ys, n, s);
        nz += n;
      }
      PairStreams ps(es, et, s);
      const int iters = es.dry() ? std::min(steps, 1) : steps;
      for (int k = 0; k < iters; ++k) {
        ps.fork();
        unet_forward(*src->n, xs, tdev + (size_t)k * B, nullptr, 0, e_src, B, R, R, s);
        unet_forward(*tgt->n, ys, tdev + (size_t)k * B, nullptr, 0, e_tgt, B, R, R, ps.target_stream());
        ps.join();
        pixel_lockstep_step(es, x0, xs, ys, e_src, e_tgt, nz + (size_t)k * n, coef[i0 + k], B, chw, net_chw_s, net_chw_t, s);
      }
    }, &et);
  });
}

int cdx_latent_cycle_pair(cdx_net* src, cdx_net* tgt, const float* x0, const cdx_ddim_coef* coef, const float* t_host, int n_steps, int n_rec,
                          const float* noise, float sqrt_a_T, float sqrt_1ma_T, const float* extra_noise, float* x_out, int B, int C, int h,
                          int w, void* stream) {
  return guard([&] {
    CDX_CHECK(src && src->owner && tgt && tgt->owner && x0 && coef && t_host && noise && x_out, "latent_cycle_pair: null argument");
    CDX_CHECK(n_steps >= 1 && n_rec >= 0 && n_rec <= n_steps, "latent_cycle_pair: n_steps=%d n_rec=%d", n_steps, n_rec);
    CDX_CHECK(n_rec == n_steps || extra_noise, "latent_cycle_pair: %d steps, %d recovered noises and no extra noise", n_steps, n_rec);
    CDX_CHECK(src->n->ucfg.context_dim == 0 && tgt->n->ucfg.context_dim == 0, "latent_cycle_pair: unconditional U-Nets only");
    CDX_CHECK(!src->n->pred && !tgt->n->pred, "latent_cycle_pair: eps-prediction U-Nets only");
    for (int i = 0; i < n_rec; ++i) CDX_CHECK(coef[i].sigma > 0.f, "latent_cycle_pair: eta must be > 0 (sigma[%d] == 0), ddim.py:268", i);
    ChainLoopArgs a;
    a.n_src = B; a.K = 1; a.src = true;
    a.x0 = x0; a.coef = coef; a.t_host = t_host; a.n_steps = n_steps; a.n_rec = n_rec; a.noise = noise; a.sa = sqrt_a_T; a.s1 = sqrt_1ma_T;
    a.extra = extra_noise; a.x_out = x_out; a.C = C; a.h = h; a.w = w;
    with_arena(src->owner->e, S(stream), [&] { run_latent_chains(*src->n, a, S(stream), tgt->n); }, &tgt->owner->e);
  });
}

int cdx_latent_cycle_fan(cdx_net* un, int n_src, int K, const float* x0, const float* c_src, const float* c_tgt, const float* uc, int L,
                         const float* src_scales, const float* tgt_scales, const cdx_ddim_coef* coef, const float* t_host, int n_steps,
                         const float* noise, float sqrt_a_T, float sqrt_1ma_T, float* x_out, float* z_out, int C, int h, int w, void* stream) {
  return cdx_latent_cycle_fan_masked(un, n_src, K, x0, c_src, c_tgt, uc, L, src_scales, tgt_scales, coef, t_host, n_steps, noise, sqrt_a_T,
                                     sqrt_1ma_T, x_out, z_out, C, h, w, stream, nullptr);
}

int cdx_latent_cycle_fan_masked(cdx_net* un, int n_src, int K, const float* x0, const float* c_src, const float* c_tgt, const float* uc,
                                int L, const float* src_scales, const float* tgt_scales, const cdx_ddim_coef* coef, const float* t_host,
                                int n_steps, const float* noise, float sqrt_a_T, float sqrt_1ma_T, float* x_out, float* z_out, int C, int h,
                                int w, void* stream, const float* mask) {
  return guard([&] {
    CDX_CHECK(un && un->owner && x0 && c_src && c_tgt && uc && src_scales && tgt_scales && coef && t_host && noise && x_out,
              "latent_cycle_fan: null argument");
    CDX_CHECK(n_src >= 1 && K >= 1 && n_steps >= 1 && L >= 1 && C >= 1 && h >= 1 && w >= 1, "latent_cycle_fan: n_src=%d K=%d n_steps=%d L=%d",
              n_src, K, n_steps, L);
    CDX_CHECK(un->n->ucfg.context_dim > 0, "latent_cycle_fan: the U-Net takes no context");
    for (int i = 0; i < n_steps; ++i) CDX_CHECK(coef[i].sigma > 0.f, "latent_cycle_fan: eta must be > 0 (sigma[%d] == 0), ddim.py:268", i);
    ChainLoopArgs a;
    a.n_src = n_src; a.K = K; a.src = true; a.x0 = x0; a.c_src = c_src; a.c_tgt = c_tgt; a.uc = uc; a.L = L;
    a.s_scales = src_scales; a.t_scales = tgt_scales; a.coef = coef; a.t_host = t_host; a.n_steps = n_steps; a.n_rec = n_steps;
    a.noise = noise; a.sa = sqrt_a_T; a.s1 = sqrt_1ma_T; a.x_out = x_out; a.z_out = z_out; a.mask = mask; a.C = C; a.h = h; a.w = w;
    with_arena(un->owner->e, S(stream), [&] { run_latent_chains(*un->n, a, S(stream)); });
  });
}

int cdx_local_blend_mask(cdx_engine* e, const float* maps, int n_terms, int n_vec, float* run, const float* user_mask, float th_blend,
                         float th_sub, float* mask_out, int B, int h, int w, void* s) {
  ENG_CALL(e, local_blend_mask(e->e, maps, n_terms, n_vec, run, user_mask, th_blend, th_sub, mask_out, B, h, w, S(s)));
}
int cdx_mask_pool(cdx_engine* e, const float* mask, float* out, int B, int H, int W, int f, void* s) {
  ENG_CALL(e, CDX_CHECK(mask && out, "mask_pool: null argument"); mask_pool(e->e, mask, out, B, H, W, f, S(s)));
}
int cdx_mask_composite(cdx_engine* e, const float* dec, const float* image, const float* mask, float* out, int B, int C, int H, int W, void* s) {
  ENG_CALL(e, CDX_CHECK(dec && image && mask && out, "mask_composite: null argument"); mask_composite(e->e, dec, image, mask, out, B, C, H, W, S(s)));
}

int cdx_edit_map(cdx_net* un, const float* x0, const float* c_src, const float* c_tgt, int L, float t, float sqrt_a, float sqrt_1ma,
                 const float* noise, int n_maps, int rows_per_call, float* acc_out, int B, int C, int h, int w, void* stream) {
  return guard([&] {
    CDX_CHECK(un && un->owner && x0 && c_src && c_tgt && noise && acc_out, "edit_map: null argument");
    CDX_CHECK(n_maps >= 1 && B >= 1 && C >= 1 && h >= 1 && w >= 1, "edit_map: n_maps=%d B=%d C=%d %dx%d", n_maps, B, C, h, w);
    CDX_CHECK(rows_per_call >= 2, "edit_map: rows_per_call=%d, a (map, image) pair takes 2 rows", rows_per_call);
    CDX_CHECK(un->n->ucfg.context_dim > 0 && L > 0, "edit_map: needs a text-conditioned U-Net and its context");
    with_arena(un->owner->e, S(stream), [&] {
      run_edit_map(*un->n, x0, c_src, c_tgt, L, t, sqrt_a, sqrt_1ma, noise, n_maps, rows_per_call, acc_out, B, C, h, w, S(stream));
    });
  });
}
int cdx_edit_map_from_eps(cdx_engine* e, const float* e_src, const float* e_tgt, float vscale, int n_maps, int maps_per_launch,
                          float* acc_out, int B, int C, int h, int w, void* s) {
  ENG_CALL(e, CDX_CHECK(e_src && e_tgt && acc_out, "edit_map_from_eps: null argument");
           CDX_CHECK(n_maps >= 1 && maps_per_launch >= 1 && B >= 1 && C >= 1 && h >= 1 && w >= 1,
                     "edit_map_from_eps: n_maps=%d maps_per_launch=%d B=%d C=%d %dx%d", n_maps, maps_per_launch, B, C, h, w);
           const long long chw = (long long)C * h * w;
           CDX_CUDA(cudaMemsetAsync(acc_out, 0, (size_t)B * h * w * sizeof(float), S(s)));
           for (int k0 = 0; k0 < n_maps; k0 += maps_per_launch)
             edit_map_accum(e->e, e_src, e_tgt, n_maps * chw, chw, 0, vscale, acc_out, B, C, h * w, k0 * B,
                            std::min(k0 + maps_per_launch, n_maps) * B, S(s)));
}
int cdx_edit_mask(cdx_engine* e, const float* acc, int n_maps, float ratio, float* map_out, float* mask_out, float* mask_img_out, int f, int B,
                  int C, int h, int w, void* s) {
  ENG_CALL(e, CDX_CHECK(acc && map_out && mask_out, "edit_mask: null argument");
           CDX_CHECK(ratio > 0.f && ratio < INFINITY, "edit_mask: ratio %g", ratio);
           edit_mask(e->e, acc, n_maps, ratio, map_out, mask_out, mask_img_out, f, B, C, h, w, S(s)));
}

int cdx_ensemble_select(cdx_engine* eh, int n, const float* scores, const int64_t* cand_idx, const int* sample_idx, const float* images,
                        float* best_score, int64_t* best_idx, float* best_img, float* score_mat, int B, int n_total, int H, int W, void* stream) {
  ENG_CALL(eh, CDX_CHECK(n >= 0 && B >= 1 && n_total >= 1 && H >= 1 && W >= 1, "ensemble_select: n=%d B=%d n_total=%d %dx%d", n, B, n_total, H, W);
           CDX_CHECK(n == 0 || (scores && cand_idx && sample_idx && images), "ensemble_select: null candidate array");
           CDX_CHECK(best_score && best_idx && best_img && score_mat, "ensemble_select: null state");
           ensemble_select(eh->e, n, scores, reinterpret_cast<const long long*>(cand_idx), sample_idx, images, best_score,
                           reinterpret_cast<long long*>(best_idx), best_img, score_mat, B, n_total, (size_t)3 * H * W, S(stream)));
}

// ---------------------------------------------------------------- unit-test hooks
int cdx_op_conv3x3(cdx_engine* eh, const float* x, const float* w_oihw, const float* bias, float* y, int B, int H, int W, int Cin, int Cout,
                   int stride, int pad_lo, int upsample, void* stream) {
  return guard([&] {
    CDX_CHECK(eh && x && w_oihw && y, "op_conv3x3: null argument");
    Engine& e = eh->e;
    cudaStream_t s = S(stream);
    with_arena(e, s, [&] {
      Scope sc(e.arena);
      e.pools_reset(s);
      float* wr = (float*)e.arena.alloc((size_t)Cout * Cin * 9 * sizeof(float));
      repack_conv3x3(e, w_oihw, wr, Cout, Cin, s);
      const int Hl = H * upsample, Wl = W * upsample;
      GemmArgs g;
      g.mode = 1;
      g.Hout = stride == 1 ? Hl : Hl / 2;
      g.Wout = stride == 1 ? Wl : Wl / 2;
      g.M = B * g.Hout * g.Wout; g.N = Cout; g.K = 9 * Cin;
      g.A = x; g.lda = Cin; g.C1 = Cin;
      g.Hin = H; g.Win = W; g.stride = stride; g.pad = pad_lo; g.up = upsample;
      g.Bw = wr; g.ldb = 9 * Cin;
      g.Cout = y; g.ldc = Cout;
      g.bias = bias;
      hook_weight_planes(e, wr, (size_t)Cout * Cin * 9, g, s);
      gemm(e, g, s);
    });
  });
}
int cdx_op_linear(cdx_engine* eh, const float* x, const float* w, const float* bias, float* y, int M, int K, int N, void* stream) {
  return guard([&] {
    CDX_CHECK(eh && x && w && y, "op_linear: null argument");
    Engine& e = eh->e;
    with_arena(e, S(stream), [&] {
      Scope sc(e.arena);
      e.pools_reset(S(stream));
      GemmArgs g;
      g.M = M; g.N = N; g.K = K;
      g.A = x; g.lda = K; g.C1 = K;
      g.Bw = w; g.ldb = K;
      g.Cout = y; g.ldc = N;
      g.bias = bias;
      hook_weight_planes(e, w, (size_t)N * K, g, S(stream));
      gemm(e, g, S(stream));
    });
  });
}
int cdx_op_groupnorm(cdx_engine* eh, const float* x, const float* gamma, const float* beta, float eps, int silu_, float* y, int B, int HW, int C,
                     void* stream) {
  return guard([&] {
    CDX_CHECK(eh && x && gamma && beta && y, "op_groupnorm: null argument");
    with_arena(eh->e, S(stream), [&] { eh->e.pools_reset(S(stream)); groupnorm(eh->e, x, C, nullptr, 0, gamma, beta, eps, silu_ != 0, nullptr, nullptr, 0, y, B, HW, S(stream)); });
  });
}
int cdx_op_layernorm(cdx_engine* eh, const float* x, const float* gamma, const float* beta, float* y, int M, int C, void* stream) {
  ENG_CALL(eh, layernorm(eh->e, x, gamma, beta, y, M, C, S(stream)));
}
// cdx_op_attention with the fused kernel's options: a Q / K row table (qk_rows, host [B]), a K / V row table (kv_rows, host [B]) or
// the accumulating launch over a row list (acc_rows, host [n_acc]); each needs the fused kernel
static int op_attention(cdx_engine* eh, const float* q, const float* k, const float* v, float* out, int B, int Nq, int Nk, int heads, int d,
                        float scale, const int* qk_rows, const int* acc_rows, int n_acc, void* stream, const int* kv_rows = nullptr) {
  return guard([&] {
    CDX_CHECK(eh && q && k && v && out, "op_attention: null argument");
    CDX_CHECK(!qk_rows || !kv_rows, "op_attention: qk_rows and kv_rows in one launch");
    if (qk_rows) for (int b = 0; b < B; ++b) CDX_CHECK(qk_rows[b] >= 0 && qk_rows[b] < B, "op_attention: qk_rows[%d] = %d outside [0, %d)", b, qk_rows[b], B);
    if (kv_rows) for (int b = 0; b < B; ++b) CDX_CHECK(kv_rows[b] >= 0 && kv_rows[b] < B, "op_attention: kv_rows[%d] = %d outside [0, %d)", b, kv_rows[b], B);
    if (acc_rows) for (int r = 0; r < n_acc; ++r) CDX_CHECK(acc_rows[r] >= 0 && acc_rows[r] < B, "op_attention: acc_rows[%d] = %d outside [0, %d)", r, acc_rows[r], B);
    const int C = heads * d;
    Engine& e = eh->e;
    cudaStream_t s = S(stream);
    with_arena(e, s, [&] {
      Scope sc(e.arena);
      bool done = false;
      const bool fused = flash_eligible(e, Nq, Nk, d, C);
      CDX_CHECK((!qk_rows && !kv_rows && !acc_rows) || fused, "op_attention: a row table needs the fused kernel (mode %d, d=%d)", e.mma_mode, d);
      int *rows_dev = nullptr, *kv_dev = nullptr;
      if (qk_rows || kv_rows) {
        int*& dev = qk_rows ? rows_dev : kv_dev;
        dev = (int*)e.arena.alloc((size_t)B * sizeof(int));
        if (!e.dry()) CDX_CUDA(cudaMemcpyAsync(dev, qk_rows ? qk_rows : kv_rows, (size_t)B * sizeof(int), cudaMemcpyHostToDevice, s));
      }
      int* acc_dev = nullptr;
      if (acc_rows) {
        acc_dev = (int*)e.arena.alloc((size_t)n_acc * sizeof(int));
        if (!e.dry()) CDX_CUDA(cudaMemcpyAsync(acc_dev, acc_rows, (size_t)n_acc * sizeof(int), cudaMemcpyHostToDevice, s));
      }
      if (fused && e.tc_kind >= 1) {
        // the SpatialTransformer's fp16-split path on loose q / k / v: ranges measured here, keys padded to a multiple of 8 per image
        e.pools_reset(s);
        const int Nks = (Nk + 7) & ~7, M = B * Nq, Mk = B * Nks;
        float *qa = e.amax_slot(), *ka = e.amax_slot(), *va = e.amax_slot();
        amax_rows(e, q, M, C, C, qa, s);
        amax_rows(e, k, (long long)B * Nk, C, C, ka, s);
        amax_rows(e, v, (long long)B * Nk, C, C, va, s);
        const float *kp = k, *vp = v;
        if (Nks != Nk) {
          float* kb = (float*)e.arena.alloc((size_t)Mk * C * sizeof(float));
          float* vb = (float*)e.arena.alloc((size_t)Mk * C * sizeof(float));
          if (!e.dry()) {
            CDX_CUDA(cudaMemsetAsync(kb, 0, (size_t)Mk * C * 4, s));
            CDX_CUDA(cudaMemsetAsync(vb, 0, (size_t)Mk * C * 4, s));
            CDX_CUDA(cudaMemcpy2DAsync(kb, (size_t)Nks * C * 4, k, (size_t)Nk * C * 4, (size_t)Nk * C * 4, B, cudaMemcpyDeviceToDevice, s));
            CDX_CUDA(cudaMemcpy2DAsync(vb, (size_t)Nks * C * 4, v, (size_t)Nk * C * 4, (size_t)Nk * C * 4, B, cudaMemcpyDeviceToDevice, s));
          }
          kp = kb; vp = vb;
        }
        const bool lo = !e.attn_one;                 // mode 5: hi planes only
        void* qh = e.arena.alloc((size_t)M * C * 2);
        void* ql = lo ? e.arena.alloc((size_t)M * C * 2) : nullptr;
        void* kh = e.arena.alloc((size_t)Mk * C * 2);
        void* kl = lo ? e.arena.alloc((size_t)Mk * C * 2) : nullptr;
        void* vh = e.arena.alloc((size_t)Mk * C * 2);
        void* vl = lo ? e.arena.alloc((size_t)Mk * C * 2) : nullptr;
        split_rows_h16(e, q, M, C, C, qh, ql, C, qa, s);
        split_rows_h16(e, kp, Mk, C, C, kh, kl, C, ka, s);
        split_transpose_h16(e, vp, Mk, C, C, vh, vl, va, s);
        const AttnPlanes pl{AttnPlanes::H16, qh, ql, C, kh, kl, C, vh, vl, qa, ka, va};
        done = flash_attention(e, pl, out, C, B, Nq, Nk, Nks, Nks, heads, d, scale, s, rows_dev, acc_dev, n_acc, kv_dev);
      }
      if (!done && e.mma_mode == 1 && Nq == Nk && (Nq % 32) == 0 && Nq >= 128 && (d % 4) == 0) {
        // same operand preparation as the SpatialTransformer: q|k side by side, V transposed, TF32 planes
        const int M = B * Nq;
        float* qk = (float*)e.arena.alloc((size_t)M * 2 * C * sizeof(float));
        float* vt = (float*)e.arena.alloc((size_t)C * M * sizeof(float));
        if (!e.dry()) {
          CDX_CUDA(cudaMemcpy2DAsync(qk, (size_t)2 * C * 4, q, (size_t)C * 4, (size_t)C * 4, M, cudaMemcpyDeviceToDevice, s));
          CDX_CUDA(cudaMemcpy2DAsync(qk + C, (size_t)2 * C * 4, k, (size_t)C * 4, (size_t)C * 4, M, cudaMemcpyDeviceToDevice, s));
        }
        nhwc_to_nchw(e, v, vt, 1, C, M, s);
        if (fused) {
          float* qh = (float*)e.arena.alloc((size_t)M * 2 * C * sizeof(float));
          float* ql = (float*)e.arena.alloc((size_t)M * 2 * C * sizeof(float));
          float* vh = (float*)e.arena.alloc((size_t)C * M * sizeof(float));
          float* vl = (float*)e.arena.alloc((size_t)C * M * sizeof(float));
          split_planes(e, qk, qh, ql, (size_t)M * 2 * C, s);
          split_planes(e, vt, vh, vl, (size_t)C * M, s);
          const AttnPlanes pl{AttnPlanes::TF32, qh, ql, 2 * C, qh + C, ql + C, 2 * C, vh, vl};
          done = flash_attention(e, pl, out, C, B, Nq, Nq, Nq, Nq, heads, d, scale, s, rows_dev, acc_dev, n_acc, kv_dev);
        }
        CDX_CHECK(done || (!rows_dev && !kv_dev && !acc_dev), "op_attention: the fused kernel rejected a row-table shape");
        if (!done) done = attention_tc(e, qk, 2 * C, qk + C, 2 * C, d, vt, out, C, B, Nq, Nk, heads, d, scale, s);
      }
      if (!done && fused) {
        // cross-attention shape, or a key count off the TMA granule: keys padded to a multiple of 4 per image, masked inside the kernel
        const int Nks = (Nk + 3) & ~3, M = B * Nq, Mk = B * Nks;
        float* kp = (float*)e.arena.alloc((size_t)Mk * C * sizeof(float));
        float* vp = (float*)e.arena.alloc((size_t)Mk * C * sizeof(float));
        float* vt = (float*)e.arena.alloc((size_t)C * Mk * sizeof(float));
        float* qh = (float*)e.arena.alloc((size_t)M * C * sizeof(float));
        float* ql = (float*)e.arena.alloc((size_t)M * C * sizeof(float));
        float* kh = (float*)e.arena.alloc((size_t)Mk * C * sizeof(float));
        float* kl = (float*)e.arena.alloc((size_t)Mk * C * sizeof(float));
        float* vh = (float*)e.arena.alloc((size_t)C * Mk * sizeof(float));
        float* vl = (float*)e.arena.alloc((size_t)C * Mk * sizeof(float));
        if (!e.dry()) {
          CDX_CUDA(cudaMemsetAsync(kp, 0, (size_t)Mk * C * 4, s));
          CDX_CUDA(cudaMemsetAsync(vp, 0, (size_t)Mk * C * 4, s));
          CDX_CUDA(cudaMemcpy2DAsync(kp, (size_t)Nks * C * 4, k, (size_t)Nk * C * 4, (size_t)Nk * C * 4, B, cudaMemcpyDeviceToDevice, s));
          CDX_CUDA(cudaMemcpy2DAsync(vp, (size_t)Nks * C * 4, v, (size_t)Nk * C * 4, (size_t)Nk * C * 4, B, cudaMemcpyDeviceToDevice, s));
        }
        nhwc_to_nchw(e, vp, vt, 1, C, Mk, s);
        split_planes(e, q, qh, ql, (size_t)M * C, s);
        split_planes(e, kp, kh, kl, (size_t)Mk * C, s);
        split_planes(e, vt, vh, vl, (size_t)C * Mk, s);
        const AttnPlanes pl{AttnPlanes::TF32, qh, ql, C, kh, kl, C, vh, vl};
        done = flash_attention(e, pl, out, C, B, Nq, Nk, Nks, Nks, heads, d, scale, s, rows_dev, acc_dev, n_acc, kv_dev);
      }
      CDX_CHECK(done || (!rows_dev && !kv_dev && !acc_dev), "op_attention: the fused kernel rejected a row-table shape");
      if (!done) attention(e, q, C, k, C, v, C, out, C, B, Nq, Nk, heads, d, d, scale, s);
    });
  });
}
int cdx_op_attention(cdx_engine* eh, const float* q, const float* k, const float* v, float* out, int B, int Nq, int Nk, int heads, int d, float scale,
                     void* stream) {
  return cdx_op_attention_rows(eh, q, k, v, out, B, Nq, Nk, heads, d, scale, nullptr, stream);
}
int cdx_op_attention_rows(cdx_engine* eh, const float* q, const float* k, const float* v, float* out, int B, int Nq, int Nk, int heads, int d,
                          float scale, const int* qk_rows, void* stream) {
  return op_attention(eh, q, k, v, out, B, Nq, Nk, heads, d, scale, qk_rows, nullptr, 0, stream);
}
int cdx_op_attention_kv_rows(cdx_engine* eh, const float* q, const float* k, const float* v, float* out, int B, int Nq, int Nk, int heads, int d,
                             float scale, const int* kv_rows, void* stream) {
  return op_attention(eh, q, k, v, out, B, Nq, Nk, heads, d, scale, nullptr, nullptr, 0, stream, kv_rows);
}
int cdx_op_attention_accum(cdx_engine* eh, const float* q, const float* k, const float* v, float* out, int B, int Nq, int Nk, int heads, int d,
                           float scale, const int* acc_rows, int n_acc, void* stream) {
  if (!acc_rows || n_acc < 1) return guard([&] { CDX_CHECK(false, "op_attention_accum: an empty row list"); });
  return op_attention(eh, q, k, v, out, B, Nq, Nk, heads, d, scale, nullptr, acc_rows, n_acc, stream);
}
static int op_attention_net(cdx_engine* eh, const cdx_attention_net_desc* d, const float* probe_weights, int* plan_out, void* stream) {
  return guard([&] {
    CDX_CHECK(eh && d && d->out && d->kind >= 0 && d->kind <= 2, "op_attention_net: null argument or bad kind");
    const int kind = d->kind, B = d->B, N = d->N, heads = d->heads, dh = d->d, C = heads * dh;
    const int L = kind == 0 ? N : d->L;
    CDX_CHECK(B > 0 && N > 0 && L > 0 && heads > 0 && dh > 0, "op_attention_net: B=%d N=%d L=%d heads=%d d=%d", B, N, L, heads, dh);
    CDX_CHECK(kind != 0 || d->qkv, "op_attention_net: self-attention needs qkv");
    CDX_CHECK(kind != 1 || (d->q && d->kv && d->ctx_lp >= L), "op_attention_net: cross-attention needs q and kv of ctx_lp >= L rows per image");
    CDX_CHECK(kind != 2 || (d->q && d->k && d->v), "op_attention_net: generic attention needs q, k and v");
    CDX_CHECK(!d->causal || kind == 2, "op_attention_net: the causal mask is the generic route's");
    CDX_CHECK(!d->qk_rows || !d->kv_rows, "op_attention_net: qk_rows and kv_rows in one launch");
    CDX_CHECK(!d->acc_rows || d->n_acc >= 1, "op_attention_net: an empty acc_rows list");
    for (const int* t : {d->qk_rows, d->kv_rows})
      if (t) for (int b = 0; b < B; ++b) CDX_CHECK(t[b] >= 0 && t[b] < B, "op_attention_net: row table entry %d = %d outside [0, %d)", b, t[b], B);
    if (d->acc_rows) for (int r = 0; r < d->n_acc; ++r) CDX_CHECK(d->acc_rows[r] >= 0 && d->acc_rows[r] < B, "op_attention_net: acc_rows[%d] outside [0, %d)", r, B);
    const bool tables = d->qk_rows || d->kv_rows || d->acc_rows;
    const bool probing = d->n_probe > 0;
    if (probing) {
      CDX_CHECK(kind == 1 && d->probe_rows && (probe_weights ? !d->probe_spans : d->probe_spans != nullptr) && d->probe_map && L >= 3,
                "op_attention_net: the probe needs kind 1, L >= 3, rows, spans or weights and a map");
      for (int i = 0; i < d->n_probe; ++i)
        CDX_CHECK(d->probe_rows[i] >= 0 && d->probe_rows[i] < B && (probe_weights || (d->probe_spans[i] >= 1 && d->probe_spans[i] <= L - 2)),
                  "op_attention_net: probe row %d = %d of %d, span %d outside 1..%d", i, d->probe_rows[i], B,
                  probe_weights ? 0 : d->probe_spans[i], L - 2);
      if (probe_weights)
        for (size_t i = 0; i < (size_t)d->n_probe * L; ++i)
          CDX_CHECK(std::isfinite(probe_weights[i]), "op_attention_net: probe weight %zu is not finite", i);
    }
    Engine& e = eh->e;
    cudaStream_t s = S(stream);
    int plan[7] = {};
    with_arena(e, s, [&] {
      Scope sc(e.arena);
      e.pools_reset(s);
      auto stage = [&](const int* host, int n) -> const int* {
        if (!host) return nullptr;
        int* dev = (int*)e.arena.alloc((size_t)n * sizeof(int));
        if (!e.dry()) CDX_CUDA(cudaMemcpyAsync(dev, host, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
        return dev;
      };
      const int *qk_dev = stage(d->qk_rows, B), *kv_dev = stage(d->kv_rows, B), *acc_dev = stage(d->acc_rows, d->n_acc);
      const int *probe_dev = probing ? stage(d->probe_rows, d->n_probe) : nullptr;
      const int* span_dev = probing && !probe_weights ? stage(d->probe_spans, d->n_probe) : nullptr;
      float* wts_dev = nullptr;
      if (probing && probe_weights) {
        wts_dev = (float*)e.arena.alloc((size_t)d->n_probe * L * sizeof(float));
        if (!e.dry()) CDX_CUDA(cudaMemcpyAsync(wts_dev, probe_weights, (size_t)d->n_probe * L * sizeof(float), cudaMemcpyHostToDevice, s));
      }
      ProbeOperands po;
      // a range slot as the network's producer leaves it: max |x| over the tensor, or the caller's (conservative) value
      auto slot_of = [&](float value, const float* x, long long rows, int cols) {
        float* slot = e.amax_slot();
        if (value > 0.f) {
          if (!e.dry()) CDX_CUDA(cudaMemcpyAsync(slot, &value, sizeof(float), cudaMemcpyHostToDevice, s));
        } else {
          amax_rows(e, x, rows, cols, cols, slot, s);
        }
        return slot;
      };
      // TF32 planes of `cols` columns of x (row stride ld) as a projection epilogue writes them: hi = rn_tf32(x), lo = rn_tf32(x - hi)
      auto tf32_planes = [&](const float* x, long long rows, int cols, long long ld, float*& hi, float*& lo) {
        const size_t n = (size_t)rows * cols;
        float* c = (float*)e.arena.alloc(n * sizeof(float));
        hi = (float*)e.arena.alloc(n * sizeof(float));
        lo = (float*)e.arena.alloc(n * sizeof(float));
        if (!e.dry()) CDX_CUDA(cudaMemcpy2DAsync(c, (size_t)cols * 4, x, (size_t)ld * 4, (size_t)cols * 4, rows, cudaMemcpyDeviceToDevice, s));
        split_planes(e, c, hi, lo, n, s);
        return c;
      };
      auto fused_plan = [&](int route, bool h16, int Nq, int Nks, int Nvs) {
        const FlashPlan f = flash_plan(dh, h16, e.attn_one, Nq);
        plan[0] = route; plan[1] = f.qrows; plan[2] = f.rag; plan[3] = f.ksplit; plan[4] = f.ring; plan[5] = Nks; plan[6] = Nvs;
      };
      const long long M = (long long)B * N;
      bool done = false;
      if (kind == 0) {
        const float* slot = slot_of(d->slot, d->qkv, M, 3 * C);
        const bool flash_ok = flash_eligible(e, N, N, dh, C);
        CDX_CHECK(!tables || flash_ok, "op_attention_net: a row table needs the fused kernel (mode %d, d=%d)", e.mma_mode, dh);
        if (flash_ok && e.tc_kind >= 1) {
          int Nvs = 0;
          done = self_attention_h16(e, d->qkv, slot, d->out, B, N, C, heads, dh, d->scale, !e.attn_one, s, qk_dev, kv_dev, acc_dev, d->n_acc, &Nvs);
          fused_plan(e.attn_one ? 4 : 2, true, N, N, Nvs);
        } else if (flash_ok) {
          float *qk_hi, *qk_lo, *vt_hi, *vt_lo;
          tf32_planes(d->qkv, M, 2 * C, 3 * C, qk_hi, qk_lo);
          int Nvs = N;
          if (N % 4) {
            float* vr = (float*)e.arena.alloc((size_t)M * C * sizeof(float));
            if (!e.dry()) CDX_CUDA(cudaMemcpy2DAsync(vr, (size_t)C * 4, d->qkv + 2 * C, (size_t)3 * C * 4, (size_t)C * 4, M, cudaMemcpyDeviceToDevice, s));
            done = self_attention_tf32_padded(e, qk_hi, qk_lo, vr, d->out, B, N, C, heads, dh, d->scale, s, qk_dev, kv_dev, acc_dev, d->n_acc, &Nvs);
          } else {
            float* vr = (float*)e.arena.alloc((size_t)M * C * sizeof(float));
            float* vt = (float*)e.arena.alloc((size_t)M * C * sizeof(float));
            if (!e.dry()) CDX_CUDA(cudaMemcpy2DAsync(vr, (size_t)C * 4, d->qkv + 2 * C, (size_t)3 * C * 4, (size_t)C * 4, M, cudaMemcpyDeviceToDevice, s));
            nhwc_to_nchw(e, vr, vt, 1, C, (int)M, s);
            tf32_planes(vt, 1, (int)(M * C), M * C, vt_hi, vt_lo);
            const AttnPlanes pl{AttnPlanes::TF32, qk_hi, qk_lo, 2 * C, qk_hi + C, qk_lo + C, 2 * C, vt_hi, vt_lo};
            done = flash_attention(e, pl, d->out, C, B, N, N, N, N, heads, dh, d->scale, s, qk_dev, acc_dev, d->n_acc, kv_dev);
          }
          fused_plan(3, false, N, N, Nvs);
        } else if (e.mma_mode >= 1 && (N % 32) == 0 && N >= 128 && (dh % 4) == 0) {
          float* qk = (float*)e.arena.alloc((size_t)M * 2 * C * sizeof(float));
          float* vr = (float*)e.arena.alloc((size_t)M * C * sizeof(float));
          float* vt = (float*)e.arena.alloc((size_t)M * C * sizeof(float));
          if (!e.dry()) {
            CDX_CUDA(cudaMemcpy2DAsync(qk, (size_t)2 * C * 4, d->qkv, (size_t)3 * C * 4, (size_t)2 * C * 4, M, cudaMemcpyDeviceToDevice, s));
            CDX_CUDA(cudaMemcpy2DAsync(vr, (size_t)C * 4, d->qkv + 2 * C, (size_t)3 * C * 4, (size_t)C * 4, M, cudaMemcpyDeviceToDevice, s));
          }
          nhwc_to_nchw(e, vr, vt, 1, C, (int)M, s);
          done = attention_tc(e, qk, 2 * C, qk + C, 2 * C, dh, vt, d->out, C, B, N, N, heads, dh, d->scale, s);
          plan[0] = 1;
        }
        if (!done) {
          attention(e, d->qkv, 3 * C, d->qkv + C, 3 * C, d->qkv + 2 * C, 3 * C, d->out, C, B, N, N, heads, dh, dh, d->scale, s);
          plan[0] = 0;
        }
      } else if (kind == 1) {
        const int Lp = d->ctx_lp;
        const long long Mk = (long long)B * Lp;
        const bool flash_ok = flash_eligible(e, N, L, dh, C);
        CDX_CHECK(!tables || flash_ok, "op_attention_net: a row table needs the fused kernel (mode %d, d=%d)", e.mma_mode, dh);
        if (flash_ok) {
          const bool h16 = e.tc_kind >= 1, lo = !e.attn_one;
          AttnPlanes pl{h16 ? AttnPlanes::H16 : AttnPlanes::TF32, nullptr, nullptr, C, nullptr, nullptr, C, nullptr, nullptr};
          if (h16) {
            const float* kv_slot = slot_of(d->slot, d->kv, Mk, 2 * C);
            const float* q_slot = slot_of(d->q_slot, d->q, M, C);
            void* q_hi = e.arena.alloc((size_t)M * C * 2);
            void* q_lo = lo ? e.arena.alloc((size_t)M * C * 2) : nullptr;
            void* k_hi = e.arena.alloc((size_t)Mk * C * 2);
            void* k_lo = lo ? e.arena.alloc((size_t)Mk * C * 2) : nullptr;
            void* vt_hi = e.arena.alloc((size_t)Mk * C * 2);
            void* vt_lo = lo ? e.arena.alloc((size_t)Mk * C * 2) : nullptr;
            split_rows_h16(e, d->q, M, C, C, q_hi, q_lo, C, q_slot, s);
            context_split_h16(e, d->kv, (int)Mk, C, kv_slot, k_hi, k_lo, vt_hi, vt_lo, s);
            pl.q_hi = q_hi; pl.q_lo = q_lo; pl.k_hi = k_hi; pl.k_lo = k_lo; pl.vt_hi = vt_hi; pl.vt_lo = vt_lo;
            pl.q_amax = q_slot; pl.k_amax = kv_slot; pl.v_amax = kv_slot;
            po.fmt = ProbeOperands::H16; po.q = d->q; po.k = k_hi; po.k_lo = k_lo; po.k_amax = kv_slot;
          } else {
            float *q_hi, *q_lo, *k_hi, *k_lo, *vt_hi, *vt_lo;
            tf32_planes(d->q, M, C, C, q_hi, q_lo);
            tf32_planes(d->kv, Mk, C, 2 * C, k_hi, k_lo);
            float* vr = (float*)e.arena.alloc((size_t)Mk * C * sizeof(float));
            float* vt = (float*)e.arena.alloc((size_t)Mk * C * sizeof(float));
            if (!e.dry()) CDX_CUDA(cudaMemcpy2DAsync(vr, (size_t)C * 4, d->kv + C, (size_t)2 * C * 4, (size_t)C * 4, Mk, cudaMemcpyDeviceToDevice, s));
            nhwc_to_nchw(e, vr, vt, 1, C, (int)Mk, s);
            tf32_planes(vt, 1, (int)(Mk * C), Mk * C, vt_hi, vt_lo);
            pl.q_hi = q_hi; pl.q_lo = q_lo; pl.k_hi = k_hi; pl.k_lo = k_lo; pl.vt_hi = vt_hi; pl.vt_lo = vt_lo;
            po.fmt = ProbeOperands::TF32; po.q = q_hi; po.q_lo = q_lo; po.k = k_hi; po.k_lo = k_lo;
          }
          po.ldq = C; po.ldk = C; po.Lk = Lp;
          done = flash_attention(e, pl, d->out, C, B, N, L, Lp, Lp, heads, dh, d->scale, s, qk_dev, acc_dev, d->n_acc, kv_dev);
          fused_plan(h16 ? (e.attn_one ? 4 : 2) : 3, h16, N, Lp, Lp);
        }
        if (!done) {
          // the unfused route reads the context unpadded, L rows per image
          float* kv = (float*)e.arena.alloc((size_t)B * L * 2 * C * sizeof(float));
          if (!e.dry())
            CDX_CUDA(cudaMemcpy2DAsync(kv, (size_t)L * 2 * C * 4, d->kv, (size_t)Lp * 2 * C * 4, (size_t)L * 2 * C * 4, B, cudaMemcpyDeviceToDevice, s));
          attention(e, d->q, C, kv, 2 * C, kv + C, 2 * C, d->out, C, B, N, L, heads, dh, dh, d->scale, s);
          plan[0] = 0;
          po.fmt = ProbeOperands::F32; po.q = d->q; po.q_lo = nullptr; po.ldq = C; po.k = kv; po.k_lo = nullptr; po.ldk = 2 * C; po.Lk = L;
        }
        if (probing) attn_probe(e, po, probe_dev, span_dev, wts_dev, d->n_probe, d->probe_map, N, L, heads, dh, d->scale, false, s);
      } else {
        CDX_CHECK(!tables, "op_attention_net: row tables need a fused route");
        attention(e, d->q, C, d->k, C, d->v, C, d->out, C, B, N, L, heads, dh, dh, d->scale, s, d->causal != 0);
      }
      CDX_CHECK(done || !tables, "op_attention_net: the fused kernel rejected a row-table shape");
    });
    if (plan_out) for (int i = 0; i < 7; ++i) plan_out[i] = plan[i];
  });
}
int cdx_op_attention_net(cdx_engine* eh, const cdx_attention_net_desc* d, int* plan_out, void* stream) {
  return op_attention_net(eh, d, nullptr, plan_out, stream);
}
int cdx_op_attention_net_weighted(cdx_engine* eh, const cdx_attention_net_desc* d, const float* probe_weights, int* plan_out, void* stream) {
  if (!probe_weights) return guard([] { throw Error(CDX_E_INVALID, "op_attention_net_weighted: null probe weights"); });
  return op_attention_net(eh, d, probe_weights, plan_out, stream);
}
int cdx_op_nchw_to_nhwc(cdx_engine* eh, const float* x, float* y, int B, int C, int HW, void* stream) { ENG_CALL(eh, nchw_to_nhwc(eh->e, x, y, B, C, HW, S(stream))); }
int cdx_op_nhwc_to_nchw(cdx_engine* eh, const float* x, float* y, int B, int C, int HW, void* stream) { ENG_CALL(eh, nhwc_to_nchw(eh->e, x, y, B, C, HW, S(stream))); }

int cdx_op_groupnorm_ex(cdx_engine* eh, const float* x1, int C1, const float* x2, int C2, const float* gamma, const float* beta, float eps,
                        int silu_, const float* scale, const float* shift, int ld_ss, float* y, float* amax_out, float* ab_out, int B, int HW,
                        void* stream) {
  return guard([&] {
    CDX_CHECK(eh && x1 && gamma && beta && y && B > 0 && HW > 0 && C1 > 0 && C2 >= 0 && (C2 == 0) == (x2 == nullptr),
              "op_groupnorm_ex: bad arguments");
    CDX_CHECK(!scale == !shift && (!scale || ld_ss >= C1 + C2), "op_groupnorm_ex: scale and shift go together, with ld_ss >= C");
    CDX_CHECK(((uintptr_t)ab_out & 7) == 0, "op_groupnorm_ex: ab_out must be 8-byte aligned");
    Engine& e = eh->e;
    cudaStream_t s = S(stream);
    with_arena(e, s, [&] {
      Scope sc(e.arena);
      e.pools_reset(s);
      // the statistics of sources whose producer did not fuse them (one pass each)
      const double* st1 = gn_channel_stats(e, x1, C1, B, HW, s);
      const double* st2 = x2 ? gn_channel_stats(e, x2, C2, B, HW, s) : nullptr;
      float* slot = e.amax_slot();
      groupnorm(e, x1, C1, x2, C2, gamma, beta, eps, silu_ != 0, scale, shift, ld_ss, y, B, HW, s, st1, st2, slot,
                reinterpret_cast<float2*>(ab_out));
      if (e.dry()) return;
      if (amax_out) CDX_CUDA(cudaMemcpyAsync(amax_out, slot, sizeof(float), cudaMemcpyDeviceToDevice, s));
    });
  });
}
int cdx_op_groupnorm_rows(cdx_engine* eh, const float* x1, int C1, const float* x2, int C2, const float* gamma, const float* beta, float eps,
                          int silu_, const float* scale, const float* shift, int ld_ss, const int* src_rows, float* y, float* amax_out,
                          float* y_rows, float* amax_rows_out, int B, int HW, void* stream) {
  return guard([&] {
    CDX_CHECK(eh && x1 && gamma && beta && y && y_rows && src_rows && B > 0 && HW > 0 && C1 > 0 && C2 >= 0 && (C2 == 0) == (x2 == nullptr),
              "op_groupnorm_rows: bad arguments");
    CDX_CHECK(!scale == !shift && (!scale || ld_ss >= C1 + C2), "op_groupnorm_rows: scale and shift go together, with ld_ss >= C");
    for (int b = 0; b < B; ++b) CDX_CHECK(src_rows[b] >= 0 && src_rows[b] < B, "op_groupnorm_rows: src_rows[%d] = %d outside [0, %d)", b, src_rows[b], B);
    Engine& e = eh->e;
    cudaStream_t s = S(stream);
    with_arena(e, s, [&] {
      Scope sc(e.arena);
      e.pools_reset(s);
      // one set of statistics for both norms (the statistics pass accumulates with atomics: two passes need not agree in the last bit)
      const double* st1 = gn_channel_stats(e, x1, C1, B, HW, s);
      const double* st2 = x2 ? gn_channel_stats(e, x2, C2, B, HW, s) : nullptr;
      int* rows_dev = (int*)e.arena.alloc((size_t)B * sizeof(int));
      if (!e.dry()) CDX_CUDA(cudaMemcpyAsync(rows_dev, src_rows, (size_t)B * sizeof(int), cudaMemcpyHostToDevice, s));   // (pageable: staged)
      float* slot = e.amax_slot();
      float* slot_rows = e.amax_slot();
      groupnorm(e, x1, C1, x2, C2, gamma, beta, eps, silu_ != 0, scale, shift, ld_ss, y, B, HW, s, st1, st2, slot);
      groupnorm(e, x1, C1, x2, C2, gamma, beta, eps, silu_ != 0, scale, shift, ld_ss, y_rows, B, HW, s, st1, st2, slot_rows, nullptr, rows_dev);
      if (e.dry()) return;
      if (amax_out) CDX_CUDA(cudaMemcpyAsync(amax_out, slot, sizeof(float), cudaMemcpyDeviceToDevice, s));
      if (amax_rows_out) CDX_CUDA(cudaMemcpyAsync(amax_rows_out, slot_rows, sizeof(float), cudaMemcpyDeviceToDevice, s));
    });
  });
}
int cdx_op_layernorm_ex(cdx_engine* eh, const float* x, const float* gamma, const float* beta, float* y, float* amax_out, int M, int C,
                        void* stream) {
  return guard([&] {
    CDX_CHECK(eh && x && gamma && beta && y && M > 0, "op_layernorm_ex: bad arguments");
    Engine& e = eh->e;
    cudaStream_t s = S(stream);
    with_arena(e, s, [&] {
      e.pools_reset(s);
      float* slot = e.amax_slot();
      layernorm(e, x, gamma, beta, y, M, C, s, slot);
      if (!e.dry() && amax_out) CDX_CUDA(cudaMemcpyAsync(amax_out, slot, sizeof(float), cudaMemcpyDeviceToDevice, s));
    });
  });
}
int cdx_op_softmax_rows(cdx_engine* eh, float* x, int64_t rows, int L, int ld, int causal_nq, void* stream) {
  ENG_CALL(eh, CDX_CHECK(x && rows > 0 && L > 0 && ld >= L && causal_nq >= 0, "op_softmax_rows: bad arguments");
           softmax_rows(eh->e, x, (long long)rows, L, ld, S(stream), causal_nq));
}
int cdx_op_produce_norm(cdx_engine* eh, const float* x, const float* w, const float* bias, int conv, int B, int H, int W, int Cin, int Cout,
                        const float* gamma, const float* beta, float eps, float* y, float* amax_out, double* stats_out, float* yn, int* path_out,
                        void* stream) {
  return guard([&] {
    CDX_CHECK(eh && x && w && gamma && beta && y && amax_out && stats_out && yn && path_out, "op_produce_norm: null argument");
    CDX_CHECK((conv == 0 || conv == 1) && B > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && Cout % 4 == 0,
              "op_produce_norm: conv=%d B=%d %dx%d Cin=%d Cout=%d", conv, B, H, W, Cin, Cout);
    Engine& e = eh->e;
    cudaStream_t s = S(stream);
    with_arena(e, s, [&] {
      Scope sc(e.arena);
      e.pools_reset(s);
      const int K = conv ? 9 * Cin : Cin;
      const float* wk = w;
      if (conv) {
        float* wr = (float*)e.arena.alloc((size_t)Cout * K * sizeof(float));
        repack_conv3x3(e, w, wr, Cout, Cin, s);
        wk = wr;
      }
      GemmArgs g;
      g.mode = conv;
      g.M = B * H * W; g.N = Cout; g.K = K;
      g.A = x; g.lda = Cin; g.C1 = Cin;
      if (conv) { g.Hin = H; g.Win = W; g.Hout = H; g.Wout = W; g.stride = 1; g.pad = 1; g.up = 1; }
      g.Bw = wk; g.ldb = K;
      g.Cout = y; g.ldc = Cout;
      g.bias = bias;
      hook_weight_planes(e, wk, (size_t)Cout * K, g, s);
      Tensor t;
      t.p = y; t.B = B; t.H = H; t.W = W; t.C = Cout;
      track_outputs(e, t, g, true);
      int route = 0;
      gemm(e, g, s, &route);          // statistics the epilogue could not fuse come from the standalone pass inside
      *path_out = (route & 2) ? 1 : (route & 4) ? 3 : (route & 8) ? 2 : 0;
      groupnorm(e, y, Cout, nullptr, 0, gamma, beta, eps, false, nullptr, nullptr, 0, yn, B, H * W, s, t.stats, nullptr, e.amax_slot());
      if (e.dry()) return;
      CDX_CUDA(cudaMemcpyAsync(amax_out, t.amax, sizeof(float), cudaMemcpyDeviceToDevice, s));
      CDX_CUDA(cudaMemcpyAsync(stats_out, t.stats, (size_t)B * Cout * 2 * sizeof(double), cudaMemcpyDeviceToDevice, s));
    });
  });
}
int cdx_op_gemm(cdx_engine* eh, const cdx_gemm_desc* d, int* plan_out, void* stream) {
  return guard([&] {
    CDX_CHECK(eh && d && d->A && d->w && d->C, "op_gemm: null argument");
    CDX_CHECK((d->mode == 0 || d->mode == 1) && d->M > 0 && d->N > 0 && d->K > 0 && d->C1 > 0 && d->C2 >= 0 && (d->C2 == 0) == !d->A2,
              "op_gemm: mode=%d M=%d N=%d K=%d C1=%d C2=%d", d->mode, d->M, d->N, d->K, d->C1, d->C2);
    CDX_CHECK(d->batch >= 0 && d->heads >= 0 && d->rows_per_batch >= 0 && (d->out_nchw ? d->rows_per_img > 0 : d->rows_per_img >= 0),
              "op_gemm: bad batch / image counts");
    const int batch = d->batch > 0 ? d->batch : 1, heads = d->heads > 0 ? d->heads : 1;
    CDX_CHECK(d->mode == 0 || (!d->b_kn && batch * heads == 1), "op_gemm: a conv3x3 is one unbatched [N][K] product");
    const int up = d->up > 0 ? d->up : 1;
    CDX_CHECK(up == 1 || (up == 2 && d->mode == 1), "op_gemm: up=%d (mode %d): a conv3x3 folds a nearest-2x upsample only", d->up, d->mode);
    Engine& e = eh->e;
    cudaStream_t s = S(stream);
    int route = 0;
    with_arena(e, s, [&] {
      Scope sc(e.arena);
      e.pools_reset(s);
      GemmArgs g;
      g.mode = d->mode;
      g.M = d->M; g.N = d->N; g.K = d->K;
      g.A = d->A; g.lda = d->lda; g.C1 = d->C1;
      g.A2 = d->A2; g.lda2 = d->lda2; g.C2 = d->C2;
      g.Hin = d->Hin; g.Win = d->Win; g.Hout = d->Hout; g.Wout = d->Wout; g.stride = d->stride; g.pad = d->pad; g.up = up;
      const float* wk = d->w;
      size_t wn;                                   // weight elements the planes cover (element index = float index)
      if (d->mode == 1) {
        float* wr = (float*)e.arena.alloc((size_t)d->N * d->K * sizeof(float));
        repack_conv3x3(e, d->w, wr, d->N, d->C1, s);
        wk = wr;
        g.ldb = d->K;
        wn = (size_t)d->N * d->K;
      } else {
        g.ldb = d->ldb;
        wn = d->b_kn ? (size_t)(d->K - 1) * d->ldb + d->N : (size_t)(d->N - 1) * d->ldb + d->K;
      }
      g.Bw = wk; g.b_kn = d->b_kn;
      if (!d->b_kn && batch * heads == 1) hook_weight_planes(e, wk, wn, g, s, d->w_range);
      g.a_amax = d->a_amax; g.a2_amax = d->a2_amax;
      g.c_amax = d->c_amax; g.c_stats = d->c_stats;
      g.Cout = d->C; g.ldc = d->ldc; g.Cout_lo = d->C_lo;
      g.Ct_hi = d->Ct_hi; g.Ct_lo = d->Ct_lo; g.t_col0 = d->t_col0; g.ldt = d->ldt;
      g.bias = d->bias;
      g.rowvec = d->rowvec; g.ld_rowvec = d->ld_rowvec; g.rows_per_batch = d->rows_per_batch > 0 ? d->rows_per_batch : 1;
      g.residual = d->residual; g.ldr = d->ldr;
      g.alpha = d->alpha;
      g.geglu = d->geglu;
      g.out_nchw = d->out_nchw; g.rows_per_img = d->rows_per_img;
      g.batch = batch; g.heads = heads;
      g.sA_b = d->sA_b; g.sA_h = d->sA_h; g.sB_b = d->sB_b; g.sB_h = d->sB_h; g.sC_b = d->sC_b; g.sC_h = d->sC_h;
      gemm(e, g, s, &route);
    });
    if (plan_out) *plan_out = route;
  });
}
int cdx_op_latent_chains(cdx_engine* eh, const cdx_latent_chains_desc* d, int stage, void* stream) {
  return guard([&] {
    CDX_CHECK(eh && d && d->chains, "op_latent_chains: null argument");
    CDX_CHECK(stage >= 0 && stage <= 2, "op_latent_chains: stage %d", stage);
    CDX_CHECK(d->chw > 0 && d->n_src > 0 && d->K >= 0 && d->rows >= 0 && (d->src == 0 || d->src == 1) && (d->pred == 0 || d->pred == 1),
              "op_latent_chains: chw=%d n_src=%d K=%d rows=%d src=%d pred=%d", d->chw, d->n_src, d->K, d->rows, d->src, d->pred);
    CDX_CHECK(d->next >= 0 && d->next <= 3 && (d->src || d->next == 0), "op_latent_chains: next=%d without a source chain", d->next);
    CDX_CHECK(d->solver >= 0 && d->solver <= 2 && (d->solver ? d->next != 1 : d->next != 3), "op_latent_chains: next=%d under solver %d",
              d->next, d->solver);
    const size_t n_chains = (size_t)d->n_src * (1 + d->K);
    // every row a launch writes or reads: the source chains' when they run, always the target chains'
    for (size_t k = d->src ? 0 : d->n_src; k < n_chains; ++k) {
      const cdx_latent_chain& c = d->chains[k];
      CDX_CHECK(c.row >= 0 && c.row < d->rows && c.row2 >= -1 && c.row2 < d->rows && c.row2 != c.row,
                "op_latent_chains: chain %zu on rows %d, %d of %d", k, c.row, c.row2, d->rows);
    }
    const bool targets = d->K > 0, reads_x0 = d->src && (stage == 0 || d->next > 0);
    if (stage != 2) {                      // the threshold stage reads eout and the tables only
      CDX_CHECK((!d->src && !targets) || d->xin, "op_latent_chains: null xin");
      CDX_CHECK(!reads_x0 || d->x0, "op_latent_chains: null x0");
      CDX_CHECK(!(d->src && (d->next == 1 || d->next == 3)) || d->noise_next, "op_latent_chains: next == %d without noise_next", d->next);
      CDX_CHECK(!d->z_out || d->z_stride >= d->chw, "op_latent_chains: z_stride %lld < chw %d", (long long)d->z_stride, d->chw);
      CDX_CHECK(d->src || !targets || (d->eps_in && d->eps_stride >= d->chw), "op_latent_chains: no source chain and no eps_in (stride %lld)",
                (long long)d->eps_stride);
    }
    if (stage == 0) {
      CDX_CHECK(!d->src || (d->noise0 && d->xt && (d->next == 0 || d->xn)), "op_latent_chains: init: null noise0 / xt / xn");
      CDX_CHECK(!targets || d->yt, "op_latent_chains: init: null yt");
    } else if (stage == 1) {
      CDX_CHECK((!d->src && !targets) || d->eout, "op_latent_chains: step: null eout");
      CDX_CHECK(!d->src || (d->xt && d->xn && (d->next == 0 || d->xn2)), "op_latent_chains: step: null xt / xn / xn2");
      CDX_CHECK(!targets || (d->yt && d->y_out), "op_latent_chains: step: null yt / y_out");
      CDX_CHECK(!d->mask || (d->src && d->hw > 0 && d->hw <= d->chw), "op_latent_chains: a mask needs a source chain and 0 < hw (%d) <= chw",
                d->hw);
      if (d->solver == 2)
        CDX_CHECK((!d->src || d->d_src) && (!targets || d->d_tgt) && (d->dc.order == 1 || d->dc.order == 2),
                  "op_latent_chains: solver 2 needs d_src / d_tgt and order 1 or 2 (order %d)", d->dc.order);
    }
    CDX_CHECK(d->sg_m >= 0 && d->sg_m <= SEMANTIC_MAX_CONCEPTS && (stage != 2 || d->sg_m > 0), "op_latent_chains: sg_m=%d at stage %d", d->sg_m,
              stage);
    const size_t n_sg = (size_t)d->n_src * d->K * d->sg_m;
    if (d->sg_m) {
      CDX_CHECK(targets && d->sg_rows && d->hw > 0 && d->chw % d->hw == 0, "op_latent_chains: concepts need target chains, sg_rows and hw (%d) "
                "dividing chw", d->hw);
      CDX_CHECK(stage == 0 || (d->eout && d->sg_thr), "op_latent_chains: concepts: null eout / sg_thr");
      CDX_CHECK(stage != 1 || d->sg_nu, "op_latent_chains: concepts: null sg_nu");
      for (size_t k = 0; k < n_sg; ++k)
        CDX_CHECK(d->sg_rows[k] >= 0 && d->sg_rows[k] < d->rows, "op_latent_chains: concept row %d of %d", d->sg_rows[k], d->rows);
      for (int q = 0; q < d->sg_m; ++q)
        CDX_CHECK(d->sg_lambda[q] >= 0.0f && d->sg_lambda[q] < 1.0f, "op_latent_chains: sg_lambda[%d]=%g outside [0, 1)", q, d->sg_lambda[q]);
    }
    CDX_CHECK(d->sg_mask >= 0 && d->sg_mask <= 2 && (!d->sg_mask || d->sg_m), "op_latent_chains: sg_mask=%d with sg_m=%d", d->sg_mask, d->sg_m);
    if (d->sg_mask && stage != 0)
      CDX_CHECK(d->sg_map && d->sg_gh >= 2 && d->sg_gw >= 2 && d->w == 4 * d->sg_gw && d->hw == 16 * d->sg_gh * d->sg_gw,
                "op_latent_chains: sg_mask needs sg_map on an sg_gh x sg_gw >= 2x2 grid of the (4 sg_gh) x (4 sg_gw) latent (w=%d hw=%d, %dx%d)",
                d->w, d->hw, d->sg_gh, d->sg_gw);
    Engine& e = eh->e;
    cudaStream_t s = S(stream);
    std::vector<Chain> ch(n_chains);
    for (size_t k = 0; k < n_chains; ++k) ch[k] = Chain{d->chains[k].row, d->chains[k].row2, d->chains[k].scale};
    with_arena(e, s, [&] {
      Scope sc(e.arena);
      Chain* chd = (Chain*)e.arena.alloc(ch.size() * sizeof(Chain));
      int* sg_rows = n_sg ? (int*)e.arena.alloc(n_sg * sizeof(int)) : nullptr;
      if (!e.dry()) CDX_CUDA(cudaMemcpyAsync(chd, ch.data(), ch.size() * sizeof(Chain), cudaMemcpyHostToDevice, s));   // (pageable: staged)
      if (!e.dry() && n_sg) CDX_CUDA(cudaMemcpyAsync(sg_rows, d->sg_rows, n_sg * sizeof(int), cudaMemcpyHostToDevice, s));
      LatentChains a;
      a.n = (size_t)d->n_src * d->chw; a.chw = d->chw; a.n_src = d->n_src; a.K = d->K;
      a.chains = chd; a.src = d->src;
      a.x0 = d->x0; a.eout = d->eout; a.c = d->c;
      a.noise0 = d->noise0; a.sa = d->sa; a.s1 = d->s1;
      a.xt = d->xt; a.xn = d->xn;
      a.next = d->next; a.noise_next = d->noise_next; a.cnext = d->cnext;
      a.xn2 = d->xn2;
      a.z_out = d->z_out; a.z_stride = d->z_stride;
      a.eps_in = d->eps_in; a.eps_stride = d->eps_stride;
      a.yt = d->yt; a.y_out = d->y_out; a.xin = d->xin;
      a.pred = d->pred; a.vsa = d->vsa; a.vs1 = d->vs1;
      a.mask = d->mask; a.hw = d->hw;
      a.sg_m = d->sg_m; a.sg_rows = sg_rows; a.sg_thr = d->sg_thr; a.sg_nu = d->sg_nu;
      for (int q = 0; q < d->sg_m; ++q) { a.sg_scale[q] = d->sg_scale[q]; a.sg_lambda[q] = d->sg_lambda[q]; }
      a.sg_active = d->sg_active; a.sg_apply = d->sg_apply; a.sg_mu = d->sg_mu; a.sg_beta = d->sg_beta; a.sg_beta1 = d->sg_beta1;
      a.sg_mask = d->sg_mask; a.sg_map = d->sg_map; a.sg_gh = d->sg_gh; a.sg_gw = d->sg_gw; a.w = d->w;
      a.solver = d->solver; a.dc = d->dc; a.d_src = d->d_src; a.d_tgt = d->d_tgt; a.qa = d->qa; a.q1 = d->q1;
      if (stage == 0) latent_chains_init(e, a, s);
      else if (stage == 2) semantic_thresholds(e, a, s);
      else latent_chains_step(e, a, s);
    });
  });
}
int cdx_op_pixel_lockstep(cdx_engine* e, const float* x0, float* xs, float* ys, const float* et_src, const float* et_tgt, const float* noise,
                          const cdx_pixel_coef* c, int B, int chw, int net_chw_src, int net_chw_tgt, void* s) {
  ENG_CALL(e, CDX_CHECK(x0 && xs && ys && et_src && et_tgt && noise && c, "op_pixel_lockstep: null argument");
           CDX_CHECK(B > 0 && chw > 0 && net_chw_src >= chw && net_chw_tgt >= chw, "op_pixel_lockstep: B=%d chw=%d net_chw %d / %d", B, chw,
                     net_chw_src, net_chw_tgt);
           pixel_lockstep_step(e->e, x0, xs, ys, et_src, et_tgt, noise, *c, B, chw, net_chw_src, net_chw_tgt, S(s)));
}

}  // extern "C"
