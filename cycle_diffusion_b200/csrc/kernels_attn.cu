// kernels_attn.cu -- fused self- / cross-attention on sm_90a wgmma (flash-style, fp32-faithful three-term products).
//
//   out[b, q, h*d + c] = sum_j softmax_j( scale * <Q[b,q,h,:], K[b,j,h,:]> ) * V[b,j,h,c]
// replaces CrossAttention.forward's two einsums + softmax (ldm/modules/attention.py:178-192), which materialise a
// [B*heads, N, N] fp32 score matrix (4.3 GB per layer at N=4096, B=8) -- here scores never leave the SM.
//
// Inputs are hi / lo planes of q, k [rows, ld] and of the transposed values V^T [C, B*N] (see nets.cu), so every operand tile arrives
// by TMA ready for the tensor core.  Default (F16): fp16 planes of x * 2^e, e from the tensor's tracked range (split_rows_h16 /
// split_transpose_h16 at the end of this file), three wgmma .f16 per 16-wide K step; F16 = false: TF32 planes (rn_tf32(x),
// rn_tf32(x - hi)) written by the projection's epilogue, three wgmma .tf32 per 8-wide step (--mma 3).  ONE (mma mode 5,
// "autocast"): fp16 hi planes only and a single wgmma .f16 per step (S = Q_hi K_hi^T, O_j = P_hi V_hi): fp16 inputs with fp32
// accumulation, the precision of torch.autocast's matmuls, at a third of the tensor-pipe time and half the K / V bytes.
//
// One CTA = 128 queries of one (batch, head); keys are walked in blocks of 64.  384 threads = 3 warpgroups:
//   warpgroup 0     TMA producer (one thread): Q planes once, then K and V^T hi+lo tiles into KS / VS deep rings.
//   warpgroups 1-2  64 query rows each: S_j = Q K_j^T (lo*hi + hi*lo + hi*hi, both operands from smem, m64n64) -> online max / exp2 /
//                   row sum in registers -> P split into hi / lo in registers (the accumulator layout of S is the A-fragment layout
//                   of the next wgmma; F16: fp16(p * 2^10)) -> O_j = P_j V_j (m64nNV, V^T tiles from smem) written fresh per block ->
//                   O_total = O_total * corr + O_j with round-to-nearest fp32 adds (the tensor core's accumulation truncates, see
//                   kernels_tc.cu; accumulating per block in registers also makes the online-softmax rescale free).  Final O / l -> global.
// Any token count: ceil(N / 128) query tiles (TMA zero-fills Q rows >= N; RAG instantiations, chosen on the host by N % 128, store no
// row >= N) and keys >= Nk in the last block masked.  d = 160 (fp16 variants): 64 queries per CTA, the two consumer warpgroups take
// alternate key blocks and merge their softmax states at the end (KSPLIT), and O_j is formed in two n80 halves (PVH) so that O_total,
// O_j, S and the P fragments fit the 232-register budget; see ACfg.
// Accumulating launch (AttnParams::acc_rows): CTAs only for the listed images, and the epilogue adds O / l into out instead of
// storing it -- a second attention term on a few rows (Prompt-to-Prompt's refine) with every variant above as it is.
// Row tables (AttnParams::qk_row, kv_row): the producer loads image b's Q and K tiles from image qk_row[b] (Prompt-to-Prompt: the
// source row's probabilities), or its K and V^T tiles from image kv_row[b] (MasaCtrl: the row's own queries over the source row's
// keys and values) -- a change of TMA coordinates only.
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace cdx {
namespace {

using namespace tc;

constexpr int AQ = 128;        // queries per CTA
constexpr int AKV = 64;        // keys per block
constexpr int ATHREADS = 384;
// queries per CTA: d = 160 takes 64 (its two Q planes are 48 KB per 64 rows; at 128 the K / V ring would be one stage deep)
constexpr int flash_qrows(int d) { return d > 80 ? 64 : AQ; }

// F16: operands are fp16 hi / lo planes (x * 2^e split as in kernels_tc.cu's KIND_H16) and the three product terms run as
// wgmma .f16 (K = 16 per instruction): half the tensor-pipe time and half the operand bytes of the TF32 planes.  P is split as
// fp16(p * 2^10): the scale keeps the lo term out of fp16's subnormal range and cancels in O / l.
// ONE (F16 only): hi planes alone, one product term; P rounded once as fp16(p * 2^10) (the scale keeps small probabilities out of
// the subnormals).  The stages are half the size, so the ring is as deep as shared memory allows (up to 4; the three-term
// variants keep depth 2).
// d = 160 (fp16 only): QROWS = 64 queries shared by both consumer warpgroups, which walk alternate key blocks with their own online
// softmax state (KSPLIT) and merge it through shared memory at the end; P.V as two m64n80 halves (PVH = 2), each added into O_total
// before the next, so a thread holds O_total (80) + one half of O_j (40) + S (32) + the P fragments (32) instead of 80 + 80 + 64.
template <int D, bool F16, bool ONE = false>
struct ACfg {
  static_assert(!ONE || F16, "the one-term variant is fp16 only");
  static constexpr int QROWS = flash_qrows(D);
  static constexpr bool KSPLIT = QROWS < AQ;
  static constexpr int PVH = D > 80 ? 2 : 1;
  static constexpr int NPL = ONE ? 1 : 2;                   // operand planes per tensor (hi, or hi + lo)
  static constexpr int KD = F16 ? (D + 15) / 16 * 16 : D;    // head dim as the QK products see it (F16: zero-padded to K = 16 steps by the TMA fill)
  static constexpr int KW = F16 ? 64 : 32;                  // elements per 128-byte k-block row
  static constexpr int KB2 = (D + KW - 1) / KW;             // 128-byte k-blocks covering the head dim
  static constexpr int NG = F16 ? KD / 16 : D / 8;          // K steps of Q.K^T (4 per 128-byte k-block)
  static constexpr int NV = (D + 15) / 16 * 16;             // PV N (rows of the V^T tile)
  static constexpr int KTILE = AKV * 128;                   // one k-block tile of K: 64 rows x 128 B
  static constexpr int K_STAGE = NPL * KB2 * KTILE;         // hi (+ lo)
  static constexpr int VTILE = NV * 128;                    // one 128-byte block of V^T (32 keys; F16: 64 keys): NV rows x 128 B
  static constexpr int V_STAGE = (F16 ? 1 : 2) * NPL * VTILE; // (key sub-blocks) x (hi (+ lo))
  static constexpr int Q_PLANE = KB2 * QROWS * 128;         // one plane of Q
  // ring depth: the deepest up to RING_MAX that fits (TF32 at d = 80 has room for one K and one V stage only)
  static constexpr int RING_MAX = ONE ? 4 : 2;
  static constexpr int RING_FIT = (232448 - 2048 - NPL * Q_PLANE) / (K_STAGE + V_STAGE);
  static constexpr int RING = RING_FIT < 1 ? 1 : RING_FIT < RING_MAX ? RING_FIT : RING_MAX;
  static constexpr int KS = RING, VS = RING;
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = NPL * Q_PLANE;
  static constexpr int OFF_V = OFF_K + KS * K_STAGE;
  static constexpr int OFF_BAR = OFF_V + VS * V_STAGE;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;   // 1 KB slack: the tiles are placed at the next 1024-byte boundary
  static_assert(D % 8 == 0 && D >= 16 && (D <= 80 || (F16 && D == 160)), "head dim must be a multiple of 8 in [16, 80], or 160 (fp16)");
  static_assert(SMEM_BYTES <= 232448, "smem overflow");
  static_assert(8 + 32 * RING <= 256, "barrier area");
  static_assert(NV % 16 == 0 && (NV / PVH) % 16 == 0, "NV");
  // key split: each warpgroup owns the stages of its key-block parity (an even ring); the merge reuses the K / V rings
  static_assert(!KSPLIT || (RING >= 2 && RING % 2 == 0), "key-split ring");
  static_assert(!KSPLIT || (NV / 2 + 4) * 128 * 4 <= KS * K_STAGE + VS * V_STAGE, "merge buffer");
};

struct AttnParams {
  int N, Nk, heads, d, B;   // N queries, Nk keys (cross-attention: Nk != N; keys >= Nk in the last block are masked); B: CTAs along z
  float scale_log2e;      // scale * log2(e): scores are kept in the log2 domain
  float* out; int ldo;
  const float *q_amax, *k_amax, *v_amax;   // F16: tracked max |q|, |k|, |v| (the planes hold x * 2^h16_exp_of(amax))
  // optional [B]: image qk_row[b] supplies the Q and K tiles of image b (attention control: a target row attends with its source
  // row's probabilities); V^T and the output stay image b's.  Null: every image its own
  const int* qk_row;
  // optional [B]: image kv_row[b] supplies the K and V^T tiles of image b (mutual self-attention: a target row's own queries
  // attend over its source row's keys and values); Q and the output stay image b's.  Exclusive with qk_row.  Null: every image its own
  const int* kv_row;
  // optional [gridDim.z]: the accumulating launch.  CTA z serves image acc_rows[z] and adds its result into out (out += O / l)
  // instead of storing it; images not listed get no CTA and are not touched (refine's second term over the controlled rows)
  const int* acc_rows;
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ void split_h16_pair(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 hh = __floats2half2_rn(x0, x1);          // .x (low half) = even key
  const float2 hf2 = __half22float2(hh);
  const __half2 ll = __floats2half2_rn(x0 - hf2.x, x1 - hf2.y);
  hi = *reinterpret_cast<const uint32_t*>(&hh);
  lo = *reinterpret_cast<const uint32_t*>(&ll);
}

template <int D, bool F16, bool ONE, bool RAG>
__global__ void __launch_bounds__(ATHREADS, 1)
flash_attn_kernel(const __grid_constant__ CUtensorMap mapQh, const __grid_constant__ CUtensorMap mapQl,
                  const __grid_constant__ CUtensorMap mapKh, const __grid_constant__ CUtensorMap mapKl,
                  const __grid_constant__ CUtensorMap mapVh, const __grid_constant__ CUtensorMap mapVl, const AttnParams p) {
  using C = ACfg<D, F16, ONE>;
  constexpr int KB2 = C::KB2, NV = C::NV, KW = C::KW, KS = C::KS, VS = C::VS, QR = C::QROWS;
  constexpr bool KSPLIT = C::KSPLIT;
  constexpr int NO = NV / 2;                       // O accumulators per thread (m64nNV)
  pdl_trigger();
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bars = base + C::OFF_BAR;
  const uint32_t bar_q_full = bars;
  auto bar_k_full = [&](int s) { return bars + 8u + 8u * s; };
  auto bar_k_empty = [&](int s) { return bars + 8u + 8u * (KS + s); };
  auto bar_v_full = [&](int s) { return bars + 8u + 8u * (2 * KS + s); };
  auto bar_v_empty = [&](int s) { return bars + 8u + 8u * (2 * KS + VS + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * QR, h = blockIdx.y;
  const int nb = (p.Nk + AKV - 1) / AKV;

  if (threadIdx.x == 0) {
    mbar_init(bar_q_full, 1);
    for (int s = 0; s < KS; ++s) { mbar_init(bar_k_full(s), 1); mbar_init(bar_k_empty(s), KSPLIT ? 4 : 8); }
    for (int s = 0; s < VS; ++s) { mbar_init(bar_v_full(s), 1); mbar_init(bar_v_empty(s), KSPLIT ? 4 : 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();                     // everything above touched shared memory only
  // (row list and, below, out of an accumulating launch: coherent reads after the dependent-launch wait, so they see everything
  // the previous launch on the stream wrote)
  const int b = p.acc_rows ? __ldcg(p.acc_rows + blockIdx.z) : (int)blockIdx.z;

  if (warp < 4) {
    // =========================================================================== TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      // the images Q, K and V^T come from (coherent reads after the dependent-launch wait; qk_row and kv_row are exclusive)
      const int bq = p.qk_row ? __ldcg(p.qk_row + b) : b;
      const int bv = p.kv_row ? __ldcg(p.kv_row + b) : b;
      const int bk = p.qk_row ? bq : bv;
      const uint32_t sq = base + C::OFF_Q;
      mbar_expect_tx(bar_q_full, C::NPL * C::Q_PLANE);
      for (int kb = 0; kb < KB2; ++kb) {
        tma_load_4d(sq + kb * QR * 128, &mapQh, kb * KW, h, q0, bq, bar_q_full);
        if (!ONE) tma_load_4d(sq + C::Q_PLANE + kb * QR * 128, &mapQl, kb * KW, h, q0, bq, bar_q_full);
      }
      for (int j = 0; j < nb; ++j) {
        // K block j: [64 keys x d] hi + lo
        const int s = j % KS;
        mbar_wait(bar_k_empty(s), ((j / KS) & 1) ^ 1);
        const uint32_t sk = base + C::OFF_K + s * C::K_STAGE;
        mbar_expect_tx(bar_k_full(s), C::K_STAGE);
        for (int kb = 0; kb < KB2; ++kb) {
          tma_load_4d(sk + kb * C::KTILE, &mapKh, kb * KW, h, j * AKV, bk, bar_k_full(s));
          if (!ONE) tma_load_4d(sk + (KB2 + kb) * C::KTILE, &mapKl, kb * KW, h, j * AKV, bk, bar_k_full(s));
        }
        // V^T block j: [NV channel rows x 64 keys] (TF32: two 32-key tiles), hi + lo
        const int sv_ = j % VS;
        mbar_wait(bar_v_empty(sv_), ((j / VS) & 1) ^ 1);
        const uint32_t sv = base + C::OFF_V + sv_ * C::V_STAGE;
        mbar_expect_tx(bar_v_full(sv_), C::V_STAGE);
        if (F16) {
          tma_load_4d(sv, &mapVh, j * AKV, bv, h * p.d, 0, bar_v_full(sv_));
          if (!ONE) tma_load_4d(sv + C::VTILE, &mapVl, j * AKV, bv, h * p.d, 0, bar_v_full(sv_));
        } else {
          for (int kk = 0; kk < 2; ++kk) {
            tma_load_4d(sv + kk * C::VTILE, &mapVh, j * AKV + kk * 32, bv, h * p.d, 0, bar_v_full(sv_));
            tma_load_4d(sv + (2 + kk) * C::VTILE, &mapVl, j * AKV + kk * 32, bv, h * p.d, 0, bar_v_full(sv_));
          }
        }
      }
    }
    return;
  }

  // ============================================================================= consumer warpgroups
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wg = (warp >> 2) - 1;                  // rows [64 wg, 64 wg + 64) of the CTA's queries (KSPLIT: key blocks j = wg mod 2)
  const int wi = warp & 3, g = lane >> 2, qd = lane & 3;
  // F16: the planes carry 2^eq q, 2^ek k, 2^ev v -> scores rescaled by the exact 2^-(eq+ek), output by 2^-ev; P is handed to the
  // tensor core as p * 2^10 (folded into the exponent; the row sum carries the same factor, so O / l is unchanged)
  float scale_l2 = p.scale_log2e, oscale = 1.f;
  if (F16) {
    scale_l2 = scale_l2 * exp2i(-h16_exp_of(*p.q_amax)) * exp2i(-h16_exp_of(*p.k_amax));
    // q and k both far below fp32's range (exponents near the +100 clamp) take the product under 2^-126, and a zero scale would turn
    // the masked scores' -inf into NaN.  Every score is then below 2^-88 in the log2 domain (|raw| < 2^38), 0 to fp32 either way
    scale_l2 = fmaxf(scale_l2, exp2i(-126));
    oscale = exp2i(-h16_exp_of(*p.v_amax));
  }
  constexpr float PEXP = F16 ? 10.f : 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // l_run: this thread's share of the row sum
  float o[NO], ob[NO], sc[32];
#pragma unroll
  for (int c = 0; c < NO; ++c) o[c] = 0.f;
  const uint32_t qh_base = base + C::OFF_Q + (KSPLIT ? 0u : (uint32_t)wg * 64u * 128u), ql_base = qh_base + C::Q_PLANE;
  mbar_wait(bar_q_full, 0);

#pragma unroll 1
  for (int j = KSPLIT ? wg : 0; j < nb; j += KSPLIT ? 2 : 1) {
    // ---- S = Q K_j^T
    const int ks = j % KS;
    mbar_wait(bar_k_full(ks), (j / KS) & 1);
    const uint32_t sk = base + C::OFF_K + ks * C::K_STAGE;
#pragma unroll
    for (int c = 0; c < 32; ++c) sc[c] = 0.f;
    wgmma_pin(sc);
    wgmma_fence();
#pragma unroll
    for (int c = 0; c < C::NG; ++c) {
      const int kb = c >> 2;
      const uint64_t adv = (uint64_t)((c & 3) * 2);
      const uint64_t q_hi = make_desc(qh_base + kb * QR * 128) + adv, q_lo = make_desc(ql_base + kb * QR * 128) + adv;
      const uint64_t k_hi = make_desc(sk + kb * C::KTILE) + adv, k_lo = make_desc(sk + (KB2 + kb) * C::KTILE) + adv;
      if (ONE) {
        Wgmma<64>::f16_ss(sc, q_hi, k_hi);
      } else if (F16) {
        Wgmma<64>::f16_ss(sc, q_lo, k_hi);
        Wgmma<64>::f16_ss(sc, q_hi, k_lo);
        Wgmma<64>::f16_ss(sc, q_hi, k_hi);
      } else {
        Wgmma<64>::tf32_ss(sc, q_lo, k_hi);
        Wgmma<64>::tf32_ss(sc, q_hi, k_lo);
        Wgmma<64>::tf32_ss(sc, q_hi, k_hi);
      }
    }
    wgmma_commit();
    wgmma_wait0();
    wgmma_pin(sc);
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_k_empty(ks));
    // element j8*4 + i*2 + c: query row 16 wi + g + 8 i, key j*64 + 8 j8 + 2 qd + c
    if (j == nb - 1 && nb * AKV != p.Nk) {           // ragged last key block (TMA zero-filled the missing keys): mask
#pragma unroll
      for (int c = 0; c < 32; ++c)
        if (j * AKV + 8 * (c >> 2) + 2 * qd + (c & 1) >= p.Nk) sc[c] = -INFINITY;
    }
    // ---- online softmax (rows g, g + 8: the four lanes of a quad share a row)
    float corr[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int j8 = 0; j8 < 8; ++j8) mx = fmaxf(mx, fmaxf(sc[j8 * 4 + i * 2], sc[j8 * 4 + i * 2 + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      mx *= scale_l2;                                // (raw scores; the positive scale commutes with max)
      const float m_new = fmaxf(m_run[i], mx);
      corr[i] = ex2_approx(m_run[i] - m_new);        // 0 on the first block (m_run = -inf)
      const float nm = PEXP - m_new;
      float psum = 0.f;
#pragma unroll
      for (int j8 = 0; j8 < 8; ++j8)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          float& x = sc[j8 * 4 + i * 2 + c];
          x = ex2_approx(fmaf(x, scale_l2, nm));
          psum += x;
        }
      l_run[i] = l_run[i] * corr[i] + psum;
      m_run[i] = m_new;
    }
    // ---- O_j = P V_j, P hi / lo as register A fragments
    const int vs = j % VS;
    mbar_wait(bar_v_full(vs), (j / VS) & 1);
    const uint32_t sv = base + C::OFF_V + vs * C::V_STAGE;
    if constexpr (C::PVH == 2) {
      // channels [0, NV/2) then [NV/2, NV): rows NV/2.. of the V^T tile start on a 1024-byte swizzle atom
      constexpr int NH = NV / 2, NOH = NO / 2;
      uint32_t ph[4][4], pl[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int e = (2 * kk + (r >> 1)) * 4 + (r & 1) * 2;
          if (ONE) {
            const __half2 hh = __floats2half2_rn(sc[e], sc[e + 1]);
            ph[kk][r] = *reinterpret_cast<const uint32_t*>(&hh);
          } else {
            split_h16_pair(sc[e], sc[e + 1], ph[kk][r], pl[kk][r]);
          }
        }
#pragma unroll
      for (int hv = 0; hv < 2; ++hv) {
        float oh[NOH];
#pragma unroll
        for (int c = 0; c < NOH; ++c) oh[c] = 0.f;
        wgmma_pin(oh);
        wgmma_fence();
        const uint32_t svh = sv + hv * NH * 128;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const uint64_t adv = (uint64_t)(kk * 2);
          const uint64_t v_hi = make_desc(svh) + adv;
          if (ONE) {
            Wgmma<NH>::f16_rs(oh, ph[kk], v_hi);
          } else {
            const uint64_t v_lo = make_desc(svh + C::VTILE) + adv;
            Wgmma<NH>::f16_rs(oh, pl[kk], v_hi);
            Wgmma<NH>::f16_rs(oh, ph[kk], v_lo);
            Wgmma<NH>::f16_rs(oh, ph[kk], v_hi);
          }
        }
        wgmma_commit();
        wgmma_wait0();
        wgmma_pin(oh);
#pragma unroll
        for (int c = 0; c < NOH; ++c) o[hv * NOH + c] = o[hv * NOH + c] * corr[(c >> 1) & 1] + oh[c];
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_v_empty(vs));
    } else {
#pragma unroll
      for (int c = 0; c < NO; ++c) ob[c] = 0.f;
      if (ONE) {
        uint32_t ph[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const int e = (2 * kk + (r >> 1)) * 4 + (r & 1) * 2;
            const __half2 hh = __floats2half2_rn(sc[e], sc[e + 1]);
            ph[kk][r] = *reinterpret_cast<const uint32_t*>(&hh);
          }
        wgmma_pin(ob);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) Wgmma<NV>::f16_rs(ob, ph[kk], make_desc(sv) + (uint64_t)(kk * 2));
      } else if (F16) {
        uint32_t ph[4][4], pl[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)               // keys 16 kk .. 16 kk + 15: accumulator groups 2 kk, 2 kk + 1
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const int e = (2 * kk + (r >> 1)) * 4 + (r & 1) * 2;
            split_h16_pair(sc[e], sc[e + 1], ph[kk][r], pl[kk][r]);
          }
        wgmma_pin(ob);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const uint64_t adv = (uint64_t)(kk * 2);
          const uint64_t v_hi = make_desc(sv) + adv, v_lo = make_desc(sv + C::VTILE) + adv;
          Wgmma<NV>::f16_rs(ob, pl[kk], v_hi);
          Wgmma<NV>::f16_rs(ob, ph[kk], v_lo);
          Wgmma<NV>::f16_rs(ob, ph[kk], v_hi);
        }
      } else {
        // TF32 A fragment of keys 8 kk .. 8 kk + 7: (row, key qd) and (row, key qd + 4); this thread holds keys 2 qd, 2 qd + 1
        uint32_t ph[8][4], pl[8][4];
        const int src1 = (lane & ~3) | (qd >> 1), src2 = src1 + 2;
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const float a0 = __shfl_sync(0xffffffffu, sc[kk * 4 + i * 2], src1), a1 = __shfl_sync(0xffffffffu, sc[kk * 4 + i * 2 + 1], src1);
            const float b0 = __shfl_sync(0xffffffffu, sc[kk * 4 + i * 2], src2), b1 = __shfl_sync(0xffffffffu, sc[kk * 4 + i * 2 + 1], src2);
            const float xa = (qd & 1) ? a1 : a0, xb = (qd & 1) ? b1 : b0;
            ph[kk][i] = rn_tf32(__float_as_uint(xa));
            pl[kk][i] = __float_as_uint(xa - __uint_as_float(ph[kk][i]));   // lo left to the tensor core's own truncation
            ph[kk][2 + i] = rn_tf32(__float_as_uint(xb));
            pl[kk][2 + i] = __float_as_uint(xb - __uint_as_float(ph[kk][2 + i]));
          }
        wgmma_pin(ob);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
          const uint64_t adv = (uint64_t)((kk & 3) * 2);
          const uint64_t v_hi = make_desc(sv + (kk >> 2) * C::VTILE) + adv, v_lo = make_desc(sv + (2 + (kk >> 2)) * C::VTILE) + adv;
          Wgmma<NV>::tf32_rs(ob, pl[kk], v_hi);
          Wgmma<NV>::tf32_rs(ob, ph[kk], v_lo);
          Wgmma<NV>::tf32_rs(ob, ph[kk], v_hi);
        }
      }
      wgmma_commit();
      wgmma_wait0();
      wgmma_pin(ob);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_v_empty(vs));
#pragma unroll
      for (int c = 0; c < NO; ++c) o[c] = o[c] * corr[(c >> 1) & 1] + ob[c];
    }
  }

  if constexpr (KSPLIT) {
    // warpgroup 1 hands (m, l, O) of its key blocks to warpgroup 0.  Once both have left the loop every K / V stage has been
    // consumed, so the rings hold the exchange.  O = O_0 2^(m_0 - m) + O_1 2^(m_1 - m): the online-softmax rescale, fp32 adds
    float* xch = reinterpret_cast<float*>(smem_raw + (base - smem_u32(smem_raw)) + C::OFF_K);
    const int tl = threadIdx.x & 127;
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (wg == 1) {
#pragma unroll
      for (int i = 0; i < 2; ++i) { xch[i * 128 + tl] = m_run[i]; xch[(2 + i) * 128 + tl] = l_run[i]; }
#pragma unroll
      for (int c = 0; c < NO; ++c) xch[(4 + c) * 128 + tl] = o[c];
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    if (wg == 1) return;
    float c0[2], c1[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float m1 = xch[i * 128 + tl], l1 = xch[(2 + i) * 128 + tl];
      const float m = fmaxf(m_run[i], m1);                 // finite: block 0 (warpgroup 0's) holds key 0
      c0[i] = ex2_approx(m_run[i] - m);
      c1[i] = ex2_approx(m1 - m);                          // 0 when warpgroup 1 had no key block (m1 = -inf)
      l_run[i] = l_run[i] * c0[i] + l1 * c1[i];
    }
#pragma unroll
    for (int c = 0; c < NO; ++c) o[c] = o[c] * c0[(c >> 1) & 1] + xch[(4 + c) * 128 + tl] * c1[(c >> 1) & 1];
  }

  // total row sums over the quad, fixed order: every thread of the row gets the same sum
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float l0 = __shfl_sync(0xffffffffu, l_run[i], lane & ~3), l1 = __shfl_sync(0xffffffffu, l_run[i], (lane & ~3) | 1);
    const float l2 = __shfl_sync(0xffffffffu, l_run[i], (lane & ~3) | 2), l3 = __shfl_sync(0xffffffffu, l_run[i], (lane & ~3) | 3);
    const float inv_l = oscale / (((l0 + l1) + l2) + l3);
    const int row = (KSPLIT ? 0 : wg * 64) + wi * 16 + g + 8 * i;
    if (RAG && q0 + row >= p.N) continue;          // ragged last query tile: rows >= N belong to the next image
    float* dst = p.out + ((long long)b * p.N + q0 + row) * p.ldo + h * p.d;
#pragma unroll
    for (int j8 = 0; j8 < NV / 8; ++j8) {
      const int col = 8 * j8 + 2 * qd;
      if (col < D) {
        float2 r = make_float2(o[j8 * 4 + i * 2] * inv_l, o[j8 * 4 + i * 2 + 1] * inv_l);
        if (p.acc_rows) {                            // out + O / l: the product rounded first, never fused into an FMA
          const float2 prev = __ldcg(reinterpret_cast<const float2*>(dst + col));
          r = make_float2(__fadd_rn(prev.x, r.x), __fadd_rn(prev.y, r.y));
        }
        *reinterpret_cast<float2*>(dst + col) = r;
      }
    }
  }
}

template <int D, bool F16, bool ONE, bool RAG>
void launch_flash_k(const CUtensorMap& qh, const CUtensorMap& ql, const CUtensorMap& kh, const CUtensorMap& kl, const CUtensorMap& vh,
                    const CUtensorMap& vl, const AttnParams& p, cudaStream_t s) {
  using C = ACfg<D, F16, ONE>;
  static bool attr[64] = {};          // per device (cudaFuncSetAttribute is device state); engines are single-threaded per device
  int dev = 0;
  CDX_CUDA(cudaGetDevice(&dev));
  if (!attr[dev & 63]) {
    CDX_CUDA(cudaFuncSetAttribute(flash_attn_kernel<D, F16, ONE, RAG>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    attr[dev & 63] = true;
  }
  launch_ex(flash_attn_kernel<D, F16, ONE, RAG>, dim3((p.N + C::QROWS - 1) / C::QROWS, p.heads, p.B), dim3(ATHREADS), C::SMEM_BYTES, s, 1, qh, ql,
            kh, kl, vh, vl, p);
}

// N a multiple of the query tile: the instantiation without the row guard
template <int D, bool F16, bool ONE = false>
void launch_flash(const CUtensorMap& qh, const CUtensorMap& ql, const CUtensorMap& kh, const CUtensorMap& kl, const CUtensorMap& vh,
                  const CUtensorMap& vl, const AttnParams& p, cudaStream_t s) {
  if (p.N % ACfg<D, F16, ONE>::QROWS) launch_flash_k<D, F16, ONE, true>(qh, ql, kh, kl, vh, vl, p, s);
  else launch_flash_k<D, F16, ONE, false>(qh, ql, kh, kl, vh, vl, p, s);
}

// the instantiation for head width d (160: fp16 planes only); false for a width without one
template <bool F16, bool ONE>
bool launch_flash_d(int d, const CUtensorMap& qh, const CUtensorMap& ql, const CUtensorMap& kh, const CUtensorMap& kl, const CUtensorMap& vh,
                    const CUtensorMap& vl, const AttnParams& p, cudaStream_t s) {
  switch (d) {
    case 16: launch_flash<16, F16, ONE>(qh, ql, kh, kl, vh, vl, p, s); return true;
    case 32: launch_flash<32, F16, ONE>(qh, ql, kh, kl, vh, vl, p, s); return true;
    case 40: launch_flash<40, F16, ONE>(qh, ql, kh, kl, vh, vl, p, s); return true;
    case 64: launch_flash<64, F16, ONE>(qh, ql, kh, kl, vh, vl, p, s); return true;
    case 80: launch_flash<80, F16, ONE>(qh, ql, kh, kl, vh, vl, p, s); return true;
    case 160:
      if constexpr (F16) { launch_flash<160, F16, ONE>(qh, ql, kh, kl, vh, vl, p, s); return true; }
      return false;
    default: return false;
  }
}

// x * 2^e -> fp16 hi / lo planes, e = h16_exp_of(*amax) (the exponent the attention kernel derives from the same slot).
// src [rows, ld] (cols % 4 == 0) -> hi / lo [rows, ldh].  LO = false: the hi plane only (one-term attention)
template <bool LO>
__global__ void split_rows_h16_kernel(const float* src, long long rows, int cols, long long ld, __half* hi,
                                      __half* lo, long long ldh, const float* amax) {
  pdl_trigger();
  pdl_wait();
  const float sc = exp2i(h16_exp_of(*amax));
  const int c4n = cols >> 2;
  const long long total = rows * (long long)c4n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / c4n;
    const int c = (int)(i - r * c4n) * 4;
    float4 v = *reinterpret_cast<const float4*>(src + r * ld + c);
    v.x *= sc; v.y *= sc; v.z *= sc; v.w *= sc;
    const __half2 h0 = __floats2half2_rn(v.x, v.y), h1 = __floats2half2_rn(v.z, v.w);
    uint2 ph;
    ph.x = *reinterpret_cast<const uint32_t*>(&h0); ph.y = *reinterpret_cast<const uint32_t*>(&h1);
    *reinterpret_cast<uint2*>(hi + r * ldh + c) = ph;
    if (LO) {
      const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
      const __half2 l0 = __floats2half2_rn(v.x - f0.x, v.y - f0.y), l1 = __floats2half2_rn(v.z - f1.x, v.w - f1.y);
      uint2 pl;
      pl.x = *reinterpret_cast<const uint32_t*>(&l0); pl.y = *reinterpret_cast<const uint32_t*>(&l1);
      *reinterpret_cast<uint2*>(lo + r * ldh + c) = pl;
    }
  }
}

// the same split, transposed: src [R, ld] columns 0..C-1 -> hi / lo [C, R] (V^T: both P.V operands K-major for wgmma).
// Per image (blockIdx.z of gridDim.z): its Ri source rows -> output columns [z Rp, z Rp + Rp), columns Ri..Rp-1 zero (a key stride
// padded to the TMA granule).  64 (rows) x 32 (columns) tiles through shared memory; Rp % 2 == 0
template <bool LO>
__global__ void __launch_bounds__(256) split_transpose_h16_kernel(const float* src, int Ri, int Rp, int Cc, long long ld, __half* hi,
                                                                   __half* lo, const float* amax) {
  __shared__ float tile[64][33];
  pdl_trigger();
  pdl_wait();
  const float sc = exp2i(h16_exp_of(*amax));
  const int r0 = blockIdx.x * 64, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 32 x 8
  const long long R = (long long)gridDim.z * Rp;               // output row length
  src += (long long)blockIdx.z * Ri * ld;
  const long long o0 = (long long)blockIdx.z * Rp;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int r = r0 + ty + 8 * k, c = c0 + tx;
    tile[ty + 8 * k][tx] = (r < Ri && c < Cc) ? src[(long long)r * ld + c] * sc : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = c0 + ty + 8 * k, r = r0 + 2 * tx;            // one warp: 64 consecutive rows of one output row = 128 B
    if (c < Cc && r < Rp) {
      const float x0 = tile[2 * tx][ty + 8 * k], x1 = tile[2 * tx + 1][ty + 8 * k];
      const __half2 h = __floats2half2_rn(x0, x1);
      *reinterpret_cast<__half2*>(hi + (long long)c * R + o0 + r) = h;
      if (LO) {
        const float2 f = __half22float2(h);
        *reinterpret_cast<__half2*>(lo + (long long)c * R + o0 + r) = __floats2half2_rn(x0 - f.x, x1 - f.y);
      }
    }
  }
}

}  // namespace

// The fused kernels' shape rule, in one place: every caller routes by it.  Any N >= 1 queries and Nk >= 1 keys (callers lay K and V^T
// out at a per-image key stride padded to 8 (fp16) / 4 (TF32) keys); head widths with an instantiation: 16, 32, 40, 64, 80, and 160
// for the fp16 planes (tc_kind >= 1; mma mode 3's TF32 planes at d = 160 keep the unfused route).  Mode 0 (FFMA) and mode 2 (unfused
// attention) never take it.
bool flash_eligible(const Engine& e, int N, int Nk, int d, int C) {
  if (e.mma_mode != 1 || !e.flash_attn || N < 1 || Nk < 1) return false;
  const bool h16 = e.tc_kind >= 1;
  if (!(d == 16 || d == 32 || d == 40 || d == 64 || d == 80 || (h16 && d == 160))) return false;
  return C % (h16 ? 8 : 4) == 0;
}

bool flash_attention(Engine& e, const AttnPlanes& a, float* out, int ldo, int B, int N, int Nk, int Nks, int Nvs, int heads, int d, float scale,
                     cudaStream_t s, const int* qk_row, const int* acc_rows, int n_acc, const int* kv_row) {
  CDX_CHECK(!qk_row || !kv_row, "flash_attention: a Q / K row table and a K / V row table in one launch");
  const bool h16 = a.fmt == AttnPlanes::H16;
  const int gm = h16 ? 7 : 3;            // strides in whole 16-byte granules (TMA)
  if (N < 1 || (a.ldq & gm) || (a.ldk & gm) || (ldo & 3) || (Nvs & gm) || Nk < 1 || Nk > Nks || Nk > Nvs) return false;
  if (!(d == 16 || d == 32 || d == 40 || d == 64 || d == 80 || (h16 && d == 160))) return false;
  const bool one = h16 && !a.q_lo;
  if (h16 && (one ? (a.k_lo || a.vt_lo) : (!a.k_lo || !a.vt_lo))) return false;
  if (!a16(a.q_hi) || !a16(a.k_hi) || !a16(a.vt_hi) || !a16(out)) return false;
  if (!one && (!a16(a.q_lo) || !a16(a.k_lo) || !a16(a.vt_lo))) return false;
  if (acc_rows && n_acc < 1) return false;
  if (e.dry()) return true;
  const int es = h16 ? 2 : 4;            // element bytes; every box row is 128 bytes
  const uint32_t bw = 128 / es;
  const int NV = (d + 15) / 16 * 16;
  uint64_t dq[4] = {(uint64_t)d, (uint64_t)heads, (uint64_t)N, (uint64_t)B};
  uint64_t sq[3] = {(uint64_t)d * es, (uint64_t)a.ldq * es, (uint64_t)N * a.ldq * es};
  uint64_t dk[4] = {(uint64_t)d, (uint64_t)heads, (uint64_t)Nks, (uint64_t)B};
  uint64_t sk[3] = {(uint64_t)d * es, (uint64_t)a.ldk * es, (uint64_t)Nks * a.ldk * es};
  uint32_t bq[4] = {bw, 1, (uint32_t)flash_qrows(d), 1}, bk[4] = {bw, 1, AKV, 1};
  uint64_t dv[4] = {(uint64_t)Nvs, (uint64_t)B, (uint64_t)heads * d, 1};
  uint64_t sv[3] = {(uint64_t)Nvs * es, (uint64_t)B * Nvs * es, (uint64_t)B * Nvs * es * heads * d};
  uint32_t bv[4] = {bw, 1, (uint32_t)NV, 1};
  const CUtensorMap& qh = get_map(a.q_hi, 4, dq, sq, bq, nullptr, es);
  const CUtensorMap& kh = get_map(a.k_hi, 4, dk, sk, bk, nullptr, es);
  const CUtensorMap& vh = get_map(a.vt_hi, 4, dv, sv, bv, nullptr, es);
  // (one-term: the lo maps are never read; the hi maps stand in for them)
  const CUtensorMap& ql = one ? qh : get_map(a.q_lo, 4, dq, sq, bq, nullptr, es);
  const CUtensorMap& kl = one ? kh : get_map(a.k_lo, 4, dk, sk, bk, nullptr, es);
  const CUtensorMap& vl = one ? vh : get_map(a.vt_lo, 4, dv, sv, bv, nullptr, es);
  AttnParams p;
  p.N = N; p.Nk = Nk; p.heads = heads; p.d = d;
  p.B = acc_rows ? n_acc : B;           // CTAs along z: the images served
  p.scale_log2e = scale * 1.4426950408889634f;
  p.out = out; p.ldo = ldo;
  p.q_amax = a.q_amax; p.k_amax = a.k_amax; p.v_amax = a.v_amax;
  p.qk_row = qk_row;
  p.kv_row = kv_row;
  p.acc_rows = acc_rows;
  const double bytes = h16 ? (one ? 1.0 : 2.0) * p.B * heads * (2.0 * N * d + 2.0 * (double)Nk * d) + (acc_rows ? 8.0 : 4.0) * p.B * heads * (double)N * d
                           : 4.0 * p.B * heads * (2.0 * N * d + 2.0 * (double)Nk * d) + (acc_rows ? 4.0 * p.B * (double)N * d * heads : 0.0);
  ProfScope ps(e, s, PROF_BATCHED_TC, 4.0 * N * (double)Nk * d * p.B * heads, bytes, 1);
  const bool ok = one ? launch_flash_d<true, true>(d, qh, ql, kh, kl, vh, vl, p, s)
                      : h16 ? launch_flash_d<true, false>(d, qh, ql, kh, kl, vh, vl, p, s)
                            : launch_flash_d<false, false>(d, qh, ql, kh, kl, vh, vl, p, s);
  if (!ok) return false;
  CDX_CUDA(cudaGetLastError());
  e.launches++;
  return true;
}

void split_rows_h16(Engine& e, const float* src, long long rows, int cols, long long ld, void* hi, void* lo, long long ldh, const float* amax,
                    cudaStream_t s) {
  CDX_CHECK((cols & 3) == 0 && (ld & 3) == 0 && (ldh & 3) == 0 && a16(src) && a16(hi) && (!lo || a16(lo)),
            "split_rows_h16: cols / strides must be multiples of 4");
  if (e.dry()) return;
  const long long total = rows * (long long)(cols >> 2);
  const int blocks = (int)std::min<long long>((total + 255) / 256, (long long)e.num_sms * 16);
  launch_ex(lo ? split_rows_h16_kernel<true> : split_rows_h16_kernel<false>, dim3((unsigned)(blocks > 0 ? blocks : 1)), dim3(256), 0, s, 1, src, rows,
            cols, ld, (__half*)hi, (__half*)lo, ldh, amax);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}

void split_transpose_h16(Engine& e, const float* src, int R, int Cc, long long ld, void* hi, void* lo, const float* amax, cudaStream_t s, int images,
                         int Rp) {
  CDX_CHECK(images >= 1 && R % images == 0, "split_transpose_h16: rows not a whole number of images");
  int Ri = R / images;
  if (Rp <= 0 || Rp == Ri) { Rp = Ri = R; images = 1; }      // no padding: one image of all R rows
  CDX_CHECK((Rp & 1) == 0 && Rp >= Ri && a16(hi) && (!lo || a16(lo)), "split_transpose_h16: even row count");
  if (e.dry()) return;
  launch_ex(lo ? split_transpose_h16_kernel<true> : split_transpose_h16_kernel<false>,
            dim3((unsigned)((Rp + 63) / 64), (unsigned)((Cc + 31) / 32), (unsigned)images), dim3(256), 0, s, 1, src, Ri, Rp, Cc, ld, (__half*)hi,
            (__half*)lo, amax);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}

namespace {
template <int D, bool F16, bool ONE>
FlashPlan plan_of(int N) {
  using C = ACfg<D, F16, ONE>;
  return {C::QROWS, N % C::QROWS != 0, C::KSPLIT, C::RING};
}
template <bool F16, bool ONE>
FlashPlan plan_d(int d, int N) {
  switch (d) {
    case 16: return plan_of<16, F16, ONE>(N);
    case 32: return plan_of<32, F16, ONE>(N);
    case 40: return plan_of<40, F16, ONE>(N);
    case 64: return plan_of<64, F16, ONE>(N);
    case 80: return plan_of<80, F16, ONE>(N);
    case 160: if constexpr (F16) return plan_of<160, F16, ONE>(N); else return {};
    default: return {};
  }
}
}  // namespace

FlashPlan flash_plan(int d, bool h16, bool one, int N) {
  return one ? plan_d<true, true>(d, N) : h16 ? plan_d<true, false>(d, N) : plan_d<false, false>(d, N);
}

bool self_attention_h16(Engine& e, const float* qkv, const float* slot, float* out, int B, int HW, int C, int heads, int d, float scale, bool lo,
                        cudaStream_t s, const int* qk_row, const int* kv_row, const int* acc_rows, int n_acc, int* Nvs_out) {
  const int M = B * HW, Nvs = (HW + 7) & ~7;
  void* qk_hi = e.arena.alloc((size_t)M * 2 * C * 2);
  void* qk_lo = lo ? e.arena.alloc((size_t)M * 2 * C * 2) : nullptr;
  void* vt_hi = e.arena.alloc((size_t)C * B * Nvs * 2);
  void* vt_lo = lo ? e.arena.alloc((size_t)C * B * Nvs * 2) : nullptr;
  split_rows_h16(e, qkv, M, 2 * C, 3 * C, qk_hi, qk_lo, 2 * C, slot, s);
  split_transpose_h16(e, qkv + 2 * C, M, C, 3 * C, vt_hi, vt_lo, slot, s, B, Nvs);
  const AttnPlanes pl{AttnPlanes::H16, qk_hi, qk_lo, 2 * C, (const char*)qk_hi + (size_t)C * 2, lo ? (const char*)qk_lo + (size_t)C * 2 : nullptr,
                      2 * C, vt_hi, vt_lo, slot, slot, slot};
  if (Nvs_out) *Nvs_out = Nvs;
  return flash_attention(e, pl, out, C, B, HW, HW, HW, Nvs, heads, d, scale, s, qk_row, acc_rows, n_acc, kv_row);
}

bool self_attention_tf32_padded(Engine& e, const float* qk_hi, const float* qk_lo, const float* vr, float* out, int B, int HW, int C, int heads,
                                int d, float scale, cudaStream_t s, const int* qk_row, const int* kv_row, const int* acc_rows, int n_acc,
                                int* Nvs_out) {
  const int Nvs = (HW + 3) & ~3;
  const size_t nvt = (size_t)C * B * Nvs;
  float* vp = (float*)e.arena.alloc(nvt * sizeof(float));
  float* vt = (float*)e.arena.alloc(nvt * sizeof(float));
  float* vt_hi = (float*)e.arena.alloc(nvt * sizeof(float));
  float* vt_lo = (float*)e.arena.alloc(nvt * sizeof(float));
  if (!e.dry()) {
    CDX_CUDA(cudaMemsetAsync(vp, 0, nvt * sizeof(float), s));
    CDX_CUDA(cudaMemcpy2DAsync(vp, (size_t)Nvs * C * 4, vr, (size_t)HW * C * 4, (size_t)HW * C * 4, B, cudaMemcpyDeviceToDevice, s));
  }
  nhwc_to_nchw(e, vp, vt, 1, C, B * Nvs, s);
  split_planes(e, vt, vt_hi, vt_lo, nvt, s);
  const AttnPlanes pl{AttnPlanes::TF32, qk_hi, qk_lo, 2 * C, qk_hi + C, qk_lo + C, 2 * C, vt_hi, vt_lo};
  if (Nvs_out) *Nvs_out = Nvs;
  return flash_attention(e, pl, out, C, B, HW, HW, HW, Nvs, heads, d, scale, s, qk_row, acc_rows, n_acc, kv_row);
}

void context_split_h16(Engine& e, const float* kv, int Mk, int C, const float* slot, void* k_hi, void* k_lo, void* vt_hi, void* vt_lo,
                       cudaStream_t s) {
  if (k_hi) split_rows_h16(e, kv, Mk, C, 2 * C, k_hi, k_lo, C, slot, s);
  split_transpose_h16(e, kv + C, Mk, C, 2 * C, vt_hi, vt_lo, slot, s);
}

// ------------------------------------------------------------------------------------------------ cross-attention probe (LEDITS++)
namespace {
constexpr int PROBE_WARPS = 8, PROBE_QPW = 2;          // 8 warps x 2 queries per CTA
template <int FMT>
__device__ __forceinline__ float probe_key(const ProbeOperands& o, size_t i, float kscale) {
  if constexpr (FMT == ProbeOperands::H16) {
    const float hi = __half2float(reinterpret_cast<const __half*>(o.k)[i]);
    const float lo = o.k_lo ? __half2float(reinterpret_cast<const __half*>(o.k_lo)[i]) : 0.f;
    return (hi + lo) * kscale;
  } else if constexpr (FMT == ProbeOperands::TF32) {
    return reinterpret_cast<const float*>(o.k)[i] + reinterpret_cast<const float*>(o.k_lo)[i];
  } else {
    return reinterpret_cast<const float*>(o.k)[i];
  }
}
// CTA (x, i): row i's queries [16x, 16x + 16); per head the head's L keys are staged in shared memory as fp32 (row stride d + 1: lane
// j reads key j's channel c without bank conflicts), each warp stages its query and lane j forms the logits of keys j, j + 32, ...
template <int FMT>
__global__ void __launch_bounds__(PROBE_WARPS * 32) attn_probe_kernel(const ProbeOperands o, const int* rows, const int* span, float* map, int N,
                                                                       int L, int heads, int d, float scale, int accumulate) {
  extern __shared__ float sm[];
  const int dp = d + 1, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* sk = sm;                                  // [L][d + 1]
  float* sq = sk + (size_t)L * dp + warp * d;      // [PROBE_WARPS][d]
  float* ss = sk + (size_t)L * dp + PROBE_WARPS * d + warp * L;   // [PROBE_WARPS][L] logits
  const int i = blockIdx.y, b = rows[i], n = span[i];
  const int p0 = (blockIdx.x * PROBE_WARPS + warp) * PROBE_QPW;
  const float kscale = FMT == ProbeOperands::H16 ? exp2i(-h16_exp_of(*o.k_amax)) : 1.f;
  float acc[PROBE_QPW] = {};
  for (int h = 0; h < heads; ++h) {
    __syncthreads();
    for (int x = threadIdx.x; x < L * d; x += blockDim.x) {
      const int j = x / d, c = x - j * d;
      sk[j * dp + c] = probe_key<FMT>(o, ((size_t)b * o.Lk + j) * o.ldk + (size_t)h * d + c, kscale);
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < PROBE_QPW; ++u) {
      const int p = p0 + u;
      if (p >= N) continue;                      // (warp-uniform; no break, so acc stays in registers)
      const size_t qi = ((size_t)b * N + p) * o.ldq + (size_t)h * d;
      for (int c = lane; c < d; c += 32) sq[c] = FMT == ProbeOperands::TF32 ? o.q[qi + c] + o.q_lo[qi + c] : o.q[qi + c];
      __syncwarp();
      float mx = -INFINITY;
      for (int j = lane; j < L; j += 32) {
        const float* kr = sk + j * dp;
        float dot = 0.f;
        for (int c = 0; c < d; ++c) dot = fmaf(sq[c], kr[c], dot);
        const float sj = __fmul_rn(scale, dot);
        ss[j] = sj;
        mx = fmaxf(mx, sj);
      }
      for (int m = 16; m; m >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, m));
      float tot = 0.f, sp = 0.f;
      for (int j = lane; j < L; j += 32) {
        const float ej = expf(__fsub_rn(ss[j], mx));
        tot = __fadd_rn(tot, ej);
        if (j >= 1 && j <= n) sp = __fadd_rn(sp, ej);
      }
      // butterfly: every lane adds the same two partial sums at each level, so all lanes hold the same total
      for (int m = 16; m; m >>= 1) {
        tot = __fadd_rn(tot, __shfl_xor_sync(0xffffffffu, tot, m));
        sp = __fadd_rn(sp, __shfl_xor_sync(0xffffffffu, sp, m));
      }
      const float ph = __fdiv_rn(sp, tot);
      acc[u] = h ? __fadd_rn(acc[u], ph) : ph;
      __syncwarp();
    }
  }
  if (lane == 0)
#pragma unroll
    for (int u = 0; u < PROBE_QPW; ++u) {
      const int p = p0 + u;
      if (p >= N) continue;
      float* o_ = map + (size_t)i * N + p;
      *o_ = accumulate ? __fadd_rn(*o_, acc[u]) : acc[u];
    }
}
// LocalBlend's weighted form of attn_probe_kernel, the same code with the span test replaced by the weights: entry i's softmax sum is
// sum_j w[i, j] e_j, one fmaf per key in the same lane order (w_j in {0, 1} adds exactly what the span form adds).  A kernel of its
// own, so that the span form's code is the one LEDITS++ measured and tested.
template <int FMT>
__global__ void __launch_bounds__(PROBE_WARPS * 32) attn_probe_weighted_kernel(const ProbeOperands o, const int* rows, const float* wts,
                                                                                float* map, int N, int L, int heads, int d, float scale,
                                                                                int accumulate) {
  extern __shared__ float sm[];
  const int dp = d + 1, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* sk = sm;                                  // [L][d + 1]
  float* sq = sk + (size_t)L * dp + warp * d;      // [PROBE_WARPS][d]
  float* ss = sk + (size_t)L * dp + PROBE_WARPS * d + warp * L;   // [PROBE_WARPS][L] logits
  const int i = blockIdx.y, b = rows[i];
  const float* wv = wts + (size_t)i * L;
  const int p0 = (blockIdx.x * PROBE_WARPS + warp) * PROBE_QPW;
  const float kscale = FMT == ProbeOperands::H16 ? exp2i(-h16_exp_of(*o.k_amax)) : 1.f;
  float acc[PROBE_QPW] = {};
  for (int h = 0; h < heads; ++h) {
    __syncthreads();
    for (int x = threadIdx.x; x < L * d; x += blockDim.x) {
      const int j = x / d, c = x - j * d;
      sk[j * dp + c] = probe_key<FMT>(o, ((size_t)b * o.Lk + j) * o.ldk + (size_t)h * d + c, kscale);
    }
    __syncthreads();
#pragma unroll
    for (int u = 0; u < PROBE_QPW; ++u) {
      const int p = p0 + u;
      if (p >= N) continue;                      // (warp-uniform; no break, so acc stays in registers)
      const size_t qi = ((size_t)b * N + p) * o.ldq + (size_t)h * d;
      for (int c = lane; c < d; c += 32) sq[c] = FMT == ProbeOperands::TF32 ? o.q[qi + c] + o.q_lo[qi + c] : o.q[qi + c];
      __syncwarp();
      float mx = -INFINITY;
      for (int j = lane; j < L; j += 32) {
        const float* kr = sk + j * dp;
        float dot = 0.f;
        for (int c = 0; c < d; ++c) dot = fmaf(sq[c], kr[c], dot);
        const float sj = __fmul_rn(scale, dot);
        ss[j] = sj;
        mx = fmaxf(mx, sj);
      }
      for (int m = 16; m; m >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, m));
      float tot = 0.f, sp = 0.f;
      for (int j = lane; j < L; j += 32) {
        const float ej = expf(__fsub_rn(ss[j], mx));
        tot = __fadd_rn(tot, ej);
        sp = fmaf(wv[j], ej, sp);
      }
      // butterfly: every lane adds the same two partial sums at each level, so all lanes hold the same total
      for (int m = 16; m; m >>= 1) {
        tot = __fadd_rn(tot, __shfl_xor_sync(0xffffffffu, tot, m));
        sp = __fadd_rn(sp, __shfl_xor_sync(0xffffffffu, sp, m));
      }
      const float ph = __fdiv_rn(sp, tot);
      acc[u] = h ? __fadd_rn(acc[u], ph) : ph;
      __syncwarp();
    }
  }
  if (lane == 0)
#pragma unroll
    for (int u = 0; u < PROBE_QPW; ++u) {
      const int p = p0 + u;
      if (p >= N) continue;
      float* o_ = map + (size_t)i * N + p;
      *o_ = accumulate ? __fadd_rn(*o_, acc[u]) : acc[u];
    }
}
}  // namespace

void attn_probe(Engine& e, const ProbeOperands& o, const int* rows, const int* span, const float* weights, int n_rows, float* map, int N, int L,
                int heads, int d, float scale, bool accumulate, cudaStream_t s) {
  CDX_CHECK(!span != !weights, "attn_probe: give spans or weights");
  CDX_CHECK(rows && map && n_rows >= 1 && N >= 1 && L >= 1 && heads >= 1 && d >= 1 && o.q && o.k && o.Lk >= L,
            "attn_probe: %d rows, N=%d L=%d Lk=%d heads=%d d=%d", n_rows, N, L, o.Lk, heads, d);
  CDX_CHECK(o.fmt != ProbeOperands::H16 || o.k_amax, "attn_probe: fp16 K planes need their range slot");
  CDX_CHECK(o.fmt != ProbeOperands::TF32 || (o.q_lo && o.k_lo), "attn_probe: TF32 planes need both terms");
  const size_t smem = ((size_t)L * (d + 1) + (size_t)PROBE_WARPS * (d + L)) * sizeof(float);
  CDX_CHECK(smem <= 227 * 1024, "attn_probe: %d keys of width %d need %zu bytes of shared memory", L, d, smem);
  if (e.dry()) return;
  const dim3 grid((unsigned)((N + PROBE_WARPS * PROBE_QPW - 1) / (PROBE_WARPS * PROBE_QPW)), (unsigned)n_rows);
  auto launch = [&](auto kernel, const auto* sel) {
    if (smem > 48 * 1024) CDX_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<grid, PROBE_WARPS * 32, smem, s>>>(o, rows, sel, map, N, L, heads, d, scale, accumulate ? 1 : 0);
  };
  ProfScope ps(e, s, PROF_SOFTMAX, 2.0 * n_rows * (double)N * L * heads * d, 4.0 * n_rows * ((double)N * heads * d + (double)L * heads * d), 1);
  ps.note("attention probe %d %s x %d queries x %d keys, %d heads x %d", n_rows, weights ? "weighted rows" : "rows", N, L, heads, d);
  if (weights)
    launch(o.fmt == ProbeOperands::H16 ? attn_probe_weighted_kernel<ProbeOperands::H16>
           : o.fmt == ProbeOperands::TF32 ? attn_probe_weighted_kernel<ProbeOperands::TF32> : attn_probe_weighted_kernel<ProbeOperands::F32>, weights);
  else
    launch(o.fmt == ProbeOperands::H16 ? attn_probe_kernel<ProbeOperands::H16>
           : o.fmt == ProbeOperands::TF32 ? attn_probe_kernel<ProbeOperands::TF32> : attn_probe_kernel<ProbeOperands::F32>, span);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}

}  // namespace cdx
