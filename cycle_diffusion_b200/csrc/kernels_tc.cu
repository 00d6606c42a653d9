// kernels_tc.cu -- sm_90a wgmma / TMA back end for the dense contractions (conv3x3, conv1x1 / Linear, batched attention products):
// fp32-faithful products from three tensor-core terms.
//
// Why three terms: the path's acceptance bar is parity with the reference's fp32 CPU path (|d pixel| <= 1e-3 through 50-250 sequential
// U-Net calls with a 1/sigma_t amplification), which plain TF32/BF16/FP16 tensor-core math cannot hold (SURVEY.md section 7; the
// single-term fast path ends at 6e-3).  Every fp32 operand is split into hi + lo and the product is accumulated as
// lo*hi + hi*lo + hi*hi in fp32 (the dropped lo*lo term is < 2^-22 relative):
//   KIND_H16 (default)  x' = x * 2^e (e from the tensor's tracked range), hi = fp16(x'), lo = fp16(x' - hi): three
//                       wgmma .f16 per 16-wide K step, exact power-of-two rescale in the epilogue;
//   KIND_TS / KIND_SS   hi = rn_tf32(x), lo = rn_tf32(x - hi): three wgmma .tf32 per 8-wide K step (--mma 3, and the
//                       activation x activation products, where neither operand has pre-split planes: KIND_SS splits B in smem).
//
// Tensor-core accumulation truncates (the error of one long accumulation grows linearly with K), so the K loop is cut into chunks of
// 256 elements (one chunk if the work item has K <= 512): each chunk accumulates in its own register set, which is added into the
// fp32 total with round-to-nearest adds when the chunk ends.
//
// One CTA per work item (tile, K split) of 128 rows x BN (64 or 128) columns -- or, for unsplit dense fp16-split work, one
// persistent CTA per SM walking the work items (PERSIST, below); 384 threads = 3 warpgroups:
//   warpgroup 0   TMA producer (one thread): A is a 2D [M,K] row matrix (dense / 1x1 conv / Linear, optionally two
//                 channel-concatenated sources), or for conv3x3 a 4D box of the NHWC activation -- per (tap, 32-channel block) {32 ch, bw,
//                 bh, bn} shifted by (dy-1, dx-1): TMA's out-of-bounds zero fill *is* the conv's zero padding, im2col is never
//                 materialised; or (batched mode) 4D maps over (k, head, row, batch) for the attention contractions.  B: pre-split
//                 weight planes (fp16 or TF32), or raw fp32 (KIND_SS).  One ring of 32-K stages in shared memory, as deep as
//                 227 KB allows (Cfg: 7 stages at BN 128 and 9 at BN 64 for the fp16 split, whose B rows are 64 B with the 64B
//                 swizzle; 4 / 7 for TF32, 128B swizzle), so the producer runs up to STAGES - 2 stages ahead of the consumers.
//   warpgroups 1-2  64 rows each: raw fp32 A from smem -> hi / lo split in registers (the wgmma A fragment layout) -> three wgmmas
//                 per K step against the B tiles in smem -> chunk accumulator -> total, software-pipelined (the next stage's A
//                 is split into a second fragment set while the current stage's wgmmas run, one batch per stage); then the
//                 epilogue from registers: alpha / rescale, +bias, +per-sample row vector (timestep embedding), GEGLU, +residual, range / GroupNorm side outputs.
// Staged epilogue (every fp32 row output of a dense or conv3x3 work item that is not split along K): once the producer has issued
// the last K stage it claims the ring slots that follow it and, with a residual, TMA-loads the residual tile there as 32-column
// boxes (the A box's shape) while the last stages' wgmmas run; the consumers add it from shared memory, write the result back in
// place (or into the claimed slots), and one thread stores the tile by TMA, which clips rows and columns outside C.  Split-K partials,
// the NCHW store, TF32 / transposed planes and batched products store per element from registers.
#include <algorithm>

#include <mutex>
#include <array>
#include <map>
#include <unordered_map>
#include <vector>
#include <cstdlib>
#include <cmath>
#include <type_traits>

#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace cdx {
namespace {

using namespace tc;

constexpr int TBM = 128, TBN = 128, TBK = 32;
constexpr int TILE_BYTES = TBM * TBK * 4;          // 16 KB: one 32-float A block of 128 rows
constexpr int TC_THREADS = 384;                     // producer warpgroup + two consumer warpgroups (setmaxnreg is per warpgroup)
constexpr int SMEM_MAX = 232448;                    // sm_90 opt-in dynamic shared memory per block
constexpr int BAR_BYTES = 256, ALIGN_SLACK = 1024;  // the ring's mbarriers; slack to align the ring base to 1024 B

// KIND_H16_FAST: the separately reported reduced-precision path (hi*hi term only), a compile-time variant of KIND_H16 so that no
// runtime branch sits inside a batch of wgmmas
enum { KIND_SS = 0, KIND_TS = 1, KIND_H16 = 2, KIND_H16_FAST = 3 };

// One ring stage = 32 K elements: the fp32 A block (128 rows x 128 B, 128B swizzle) + two B planes (hi / lo; KIND_SS: raw fp32
// and its in-place lo), BN rows each: 32 fp16 = 64 B (64B swizzle) or 32 fp32 = 128 B (128B swizzle).  The ring is as deep as the
// shared memory allows: the deeper it is, the more operand bytes the producer keeps in flight ahead of the consumers
// (H16: 7 stages at BN 128, 9 at BN 64; TS / SS: 4 at BN 128, 7 at BN 64).
//
// PERSIST (fp16 split, unsplit dense work items with the staged store): the epilogue has a buffer of its own after the ring, one
// 32-column box per 32 output columns (64 KB at BN 128, 32 KB at BN 64), and the ring shrinks to fit (5 / 8 stages).
template <int KIND, int BN, bool PERSIST = false>
struct Cfg {
  static constexpr bool H16 = KIND == KIND_H16 || KIND == KIND_H16_FAST;
  static constexpr int BK = TBK;                     // K elements per pipeline stage
  static constexpr int KSTEPS = H16 ? 2 : 4;         // wgmma K steps per stage: k16 (fp16) or k8 (tf32)
  static constexpr int KCHUNK = 256 / BK;            // stages per accumulation chunk (256 K elements)
  static constexpr int A_BYTES = TILE_BYTES;
  static constexpr int B_ROW = H16 ? 64 : 128;       // bytes of one B row of a stage
  static constexpr int B_PLANE = BN * B_ROW;
  static constexpr int STAGE_BYTES = A_BYTES + 2 * B_PLANE;
  static constexpr int EPI_BOX = TBM * TBK * 4;
  static constexpr int EPI_BYTES = PERSIST ? BN / TBK * EPI_BOX : 0;     // the persistent epilogue's own buffer
  static constexpr int STAGES = (SMEM_MAX - BAR_BYTES - ALIGN_SLACK - EPI_BYTES) / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + EPI_BYTES + BAR_BYTES + ALIGN_SLACK;
  // Staged epilogue: the output tile (and the residual tile, loaded by TMA) as 32-column fp32 boxes of 128 rows (the A box's shape,
  // 128B swizzle), EPI_PER_SLOT to a ring slot, in the slots of ring stages nst, nst + 1, ... after the work item's nst stages.  The
  // producer claims each through its empty barrier, which frees the slot of stage nst + k - STAGES; the last stage's slot is never
  // handed back, so every claimed slot must have held a stage before nst - 1, and for the residual to land while the last wgmmas
  // run, before nst - 2: STAGES >= 2 + EPI_SLOTS.  (PERSIST: the boxes live in the epilogue's buffer instead.)
  static constexpr int EPI_PER_SLOT = STAGE_BYTES / EPI_BOX;
  static constexpr int EPI_SLOTS = (BN / TBK + EPI_PER_SLOT - 1) / EPI_PER_SLOT;
  static_assert(PERSIST || STAGES >= 2 + EPI_SLOTS, "the epilogue's slots never include the last stages' slots");
  static_assert(!PERSIST || (H16 && STAGES == (BN == 128 ? 5 : 8)), "persistent ring: 5 stages at BN 128, 8 at BN 64 beside the epilogue buffer");
  static_assert(EPI_BYTES % 1024 == 0, "the barriers after the epilogue buffer stay aligned");
  static_assert(STAGES >= 3 && (2 * STAGES + 2) * 8 <= BAR_BYTES, "barrier area holds a full and an empty barrier per stage, bar_res and bar_out");
  static_assert(STAGE_BYTES % 1024 == 0 && B_PLANE % 1024 == 0, "stage and plane bases stay 1024-byte aligned (swizzle atoms)");
  static_assert(SMEM_BYTES <= SMEM_MAX, "smem overflow");
};

struct TcParams {
  int M, N, K;
  int mode;                 // 0 dense, 1 conv3x3, 2 batched dense
  int C1, C2;               // channels of source 1 / 2 (dense: k-blocks never straddle, C1 % 32 == 0 when C2 > 0; conv: one
                            // source, C1 = input channels, a multiple of 32)
  int H, W, B;              // conv: spatial size of the output and batch
  int bw, bh, bn;           // conv: pixel box of one M tile (bw*bh*bn == 128)
  int tiles_x, tiles_y;     // conv: tiles per row / column (cdiv: a tile may overhang the map; its outside rows are masked)
  int cstride, cpad;        // conv: stride (1 or 2: TMA element traversal stride) and low-side padding
  float* C; int ldc;
  float* C_lo;              // optional: C <- rn_tf32(result), C_lo <- rn_tf32(result - hi)
  float* Ct_hi; float* Ct_lo; int t_col0; long long ldt;   // optional transposed plane output for columns >= t_col0
  const float* bias;
  const float* rowvec; int ld_rowvec; int rows_per_batch;
  const float* residual; int ldr;
  float alpha;
  int geglu;                    // N tiles hold [32 value | 32 gate] column blocks: store value * gelu(gate) to [M, N/2]
  int out_nchw, rows_per_img;   // store C as [B, N, rows_per_img] (final conv of a network, reference NCHW layout)
  // mode 2 (z = zb*heads + zh): 4D maps, coordinate recipe per operand
  int heads;
  int a_code[4], b_code[4];   // per map dim: 0 -> k0, 1 -> row0, 2 -> zh, 3 -> zb, 4 -> 0
  int a_rowoff_h, b_rowoff_h; // row0 += zh * rowoff (heads packed along the row dimension)
  long long sC_b, sC_h;       // output offsets per zb / zh
  // work item t (= blockIdx.x) -> (split = t % splits, tm, tn, z): see tile_coord
  int tiles_m, tiles_n, total_tiles;
  int tn_w;                 // tile width along N (== the kernel's BN)
  // split-K (small-M layers that cannot fill the GPU): split s covers k-blocks [s*kb_per_split, min(num_kb, (s+1)*kb_per_split)) and
  // writes its raw partial tile to ws[s][M][N]; splitk_reduce_kernel then sums the partials in fixed order and applies the epilogue
  int splits, kb_per_split;
  float* ws;
  // KIND_H16: tracked max |A| (device scalars written by the producers of A / A2), exponent of the pre-scaled fp16 weight planes
  const float* a_amax; const float* a2_amax;
  int b_exp;
  float* c_amax;            // optional: atomic max of |C| over everything this launch stores (operand range for the consumer GEMM)
  double* c_stats;          // optional: per-(image, channel) fp64 {sum, sum sq} of C, for the GroupNorm that consumes it; requires
                            // every 32-row quadrant of a tile to lie inside one image (checked on the host)
};

// Result tiles staged in shared memory and stored by TMA (mapC; the residual tile arrives by TMA through mapR): every fp32 row
// output of a dense or conv3x3 work item.  Split-K partials, the NCHW store, TF32 / transposed planes and batched products keep the
// per-element stores.
__host__ __device__ __forceinline__ bool staged_store(const TcParams& p) {
  return p.mode != 2 && p.splits == 1 && !p.out_nchw && !p.Ct_hi && !p.C_lo;
}

__device__ __forceinline__ int h16_a_exp(const TcParams& p) {
  float m = p.a_amax ? *p.a_amax : 0.f;
  if (p.a2_amax) m = fmaxf(m, *p.a2_amax);
  return h16_exp_of(m);
}

struct TileCoord { int n0, nend, m0, x0, y0, b0, zb, zh, kb0, kb1, split; };

// Raster of the tiles of one z: bands of RASTER_M tiles along M, walked band by band; inside a band M varies fastest, then N.  A wave
// of CTAs then covers a few M tiles x many N tiles instead of ~num_sms M tiles x one N tile, so every A row band is fetched from HBM
// about once per launch rather than once per N tile (an A tile and a B tile of a k-block are both 32 KB: the wave's footprint is
// smallest when it spans similar numbers of M and N tiles).
constexpr int RASTER_M = 8;

__device__ __forceinline__ TileCoord tile_coord(const TcParams& p, int t, int num_kb) {
  TileCoord c;
  c.split = t % p.splits;
  t /= p.splits;
  c.kb0 = c.split * p.kb_per_split;
  c.kb1 = min(num_kb, c.kb0 + p.kb_per_split);
  const int per_z = p.tiles_m * p.tiles_n;
  const int z = t / per_z;
  int u = t - z * per_z;
  const int m_lo = u / (RASTER_M * p.tiles_n) * RASTER_M;       // first M tile of the band
  const int bm = min(RASTER_M, p.tiles_m - m_lo);                 // M tiles of the band (the last one may be short)
  u -= m_lo * p.tiles_n;
  const int tm = m_lo + u % bm, tn = u / bm;
  c.n0 = tn * p.tn_w;
  c.nend = min(p.N, c.n0 + p.tn_w);
  c.m0 = 0; c.x0 = 0; c.y0 = 0; c.b0 = 0; c.zb = 0; c.zh = 0;
  if (p.mode == 1) {
    int u = tm;
    const int tx = u % p.tiles_x; u /= p.tiles_x;
    const int ty = u % p.tiles_y; u /= p.tiles_y;
    c.x0 = tx * p.bw; c.y0 = ty * p.bh; c.b0 = u * p.bn;
  } else {
    c.m0 = tm * TBM;
    c.zb = z / p.heads;
    c.zh = z - c.zb * p.heads;
  }
  return c;
}

__device__ __forceinline__ uint32_t tf32_lo(float x, uint32_t hi) { return rn_tf32(__float_as_uint(x - __uint_as_float(hi))); }

// Timeline probe, compiled in only with -DCDX_GEMM_TIMELINE (tools/gemm_timeline.py builds that variant into a directory of its own):
// %globaltimer stamps per CTA into a device buffer, TL_SLOTS per CTA at [blockIdx.x * TL_SLOTS]: 0 entry, 1 after pdl_wait, 2 the
// first stage has landed, 3 the last stage has retired, 4 bar_res passed, 5 the TMA store issued, 6 bulk_wait0 returned.  A
// persistent CTA stamps 2 at its first work item and 3 - 6 at its last.
#ifdef CDX_GEMM_TIMELINE
constexpr int TL_SLOTS = 8;
__device__ unsigned long long* g_gemm_timeline = nullptr;
__device__ __forceinline__ void tl_stamp(int k) {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t) :: "memory");
  if (g_gemm_timeline) g_gemm_timeline[(size_t)blockIdx.x * TL_SLOTS + k] = t;
}
#define TL_STAMP(k) tl_stamp(k)
#else
#define TL_STAMP(k) ((void)0)
#endif

// PERSIST (KIND_H16 / KIND_H16_FAST, unsplit dense work items with the staged store; gemm_tc decides): a grid of at most one CTA
// per SM, CTA c walking work items t = c, c + gridDim.x, ... of the same raster.  The ring's stage counter and phases run on across
// the items, so the producer fills item t + gridDim.x's stages as soon as item t's last stage is issued.  The epilogue has its own
// buffer after the ring: thread 32 (warpgroup 0) stores item j's boxes from it by TMA once the consumers have written them (bar_out),
// waits only until the store has read the buffer, then TMA-loads item j + 1's residual boxes into it (bar_res: the buffer is free
// and the residual has landed).  Full completion of the stores is awaited once, after the CTA's last item.  Each output tile is
// computed by the same stages, wgmmas and epilogue arithmetic as without PERSIST.
template <int KIND, int BN, bool PERSIST = false>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapA2,
               const __grid_constant__ CUtensorMap mapB, const __grid_constant__ CUtensorMap mapBlo,
               const __grid_constant__ CUtensorMap mapR, const __grid_constant__ CUtensorMap mapC, const TcParams p) {
  using CF = Cfg<KIND, BN, PERSIST>;
  constexpr bool H16 = CF::H16, FAST = KIND == KIND_H16_FAST;
  constexpr int BK = CF::BK, KSTEPS = CF::KSTEPS, A_BYTES = CF::A_BYTES, B_PLANE = CF::B_PLANE, STAGE_BYTES = CF::STAGE_BYTES;
  constexpr int STAGES = CF::STAGES, EPI_BOX = CF::EPI_BOX, EPI_PER_SLOT = CF::EPI_PER_SLOT, EPI_SLOTS = CF::EPI_SLOTS;
  constexpr int NACC = BN / 2;                     // fp32 accumulators per thread of an m64nBN tile
  if (threadIdx.x == 0) TL_STAMP(0);
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;     // 1024-byte aligned (swizzle atoms)
  const uint32_t epi = base + STAGES * STAGE_BYTES;                // PERSIST: the epilogue's buffer
  const uint32_t bars = epi + CF::EPI_BYTES;
  auto bar_full = [&](int s) { return bars + 8u * s; };
  auto bar_empty = [&](int s) { return bars + 8u * (STAGES + s); };
  const uint32_t bar_res = bars + 16u * STAGES;    // the epilogue's slots are claimed (and the residual tile has landed)
  const uint32_t bar_out = bar_res + 8u;           // PERSIST: the consumers have written a work item's output boxes

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = (p.K + BK - 1) / BK;
  TileCoord tc_ = tile_coord(p, blockIdx.x, num_kb);
  int nst = tc_.kb1 - tc_.kb0;                     // stages of this work item (>= 1; K % 32 == 0: every stage is full)
  const bool staged = PERSIST || staged_store(p);
  // shared address of 32-column box k of the staged output / residual tile
  auto epi_box = [&](int k) {
    return PERSIST ? epi + k * EPI_BOX : base + ((nst + k / EPI_PER_SLOT) % STAGES) * STAGE_BYTES + (k % EPI_PER_SLOT) * EPI_BOX;
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(bar_full(s), 1);
      mbar_init(bar_empty(s), 8);                 // one arrival per consumer warp
    }
    mbar_init(bar_res, 1);
    if (PERSIST) mbar_init(bar_out, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();                     // everything above touched shared memory only
  if (threadIdx.x == 0) TL_STAMP(1);

  if (PERSIST && warp < 4) {
    // =========================================================================== TMA producer and epilogue store, persistent
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int it = 0;                                  // ring stage counter, across the CTA's work items
      for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
        const TileCoord c = tile_coord(p, t, num_kb);
        for (int kb = c.kb0; kb < c.kb1; ++kb, ++it) {
          const int s = it % STAGES;
          mbar_wait(bar_empty(s), ((it / STAGES) & 1) ^ 1);
          const uint32_t st = base + s * STAGE_BYTES;
          const int k0 = kb * BK;
          mbar_expect_tx(bar_full(s), TILE_BYTES + 2 * B_PLANE);
          if (k0 < p.C1) tma_load_2d(st, &mapA, k0, c.m0, bar_full(s));
          else tma_load_2d(st, &mapA2, k0 - p.C1, c.m0, bar_full(s));
          tma_load_2d(st + A_BYTES, &mapB, k0, c.n0, bar_full(s));
          tma_load_2d(st + A_BYTES + B_PLANE, &mapBlo, k0, c.n0, bar_full(s));
        }
      }
    } else if (threadIdx.x == 32) {
      const int c0_div = p.geglu ? 2 : 1, ncols = p.geglu ? p.N / 2 : p.N, nbox = p.geglu ? BN / 64 : BN / TBK;
      auto store = [&](const TileCoord& c) {
        const int c0 = c.n0 / c0_div;
        for (int b = 0; b < nbox && c0 + b * TBK < ncols; ++b) tma_store_2d(epi_box(b), &mapC, c0 + b * TBK, c.m0);
        bulk_commit();
      };
      int j = 0;
      TileCoord prev;
      for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x, ++j) {
        const TileCoord c = tile_coord(p, t, num_kb);
        if (j > 0) {
          mbar_wait(bar_out, (j - 1) & 1);
          store(prev);
          bulk_wait_read0();                       // the buffer has been read: it may take item j's residual and output
        }
        if (p.residual) {
          mbar_expect_tx(bar_res, BN * TBM * 4);
          for (int b = 0; b < BN / TBK; ++b) tma_load_2d(epi_box(b), &mapR, c.n0 + b * TBK, c.m0, bar_res);
        } else {
          mbar_arrive(bar_res);
        }
        prev = c;
      }
      if (j > 0) {
        mbar_wait(bar_out, (j - 1) & 1);
        store(prev);
        TL_STAMP(5);
        bulk_wait0();                              // written, not only read: a dependent launch reads C after its griddepcontrol.wait
        TL_STAMP(6);
      }
    }
    return;
  }

  if (warp < 4) {
    // =========================================================================== TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      const int cblocks = p.mode == 1 ? p.C1 / TBK : 0;
      int it = 0;
      for (int kb = tc_.kb0; kb < tc_.kb1; ++kb, ++it) {
        const int s = it % STAGES;
        mbar_wait(bar_empty(s), ((it / STAGES) & 1) ^ 1);
        const uint32_t st = base + s * STAGE_BYTES;
        const uint32_t sb = st + A_BYTES;
        const int k0 = kb * BK;
        if (p.mode == 2) {
          mbar_expect_tx(bar_full(s), TILE_BYTES + BN * 128);
          int ca[4], cb4[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int ac = p.a_code[i], bc = p.b_code[i];
            ca[i] = ac == 0 ? k0 : ac == 1 ? tc_.m0 + tc_.zh * p.a_rowoff_h : ac == 2 ? tc_.zh : ac == 3 ? tc_.zb : 0;
            cb4[i] = bc == 0 ? k0 : bc == 1 ? tc_.n0 + tc_.zh * p.b_rowoff_h : bc == 2 ? tc_.zh : bc == 3 ? tc_.zb : 0;
          }
          tma_load_4d(st, &mapA, ca[0], ca[1], ca[2], ca[3], bar_full(s));
          tma_load_4d(sb, &mapB, cb4[0], cb4[1], cb4[2], cb4[3], bar_full(s));
          continue;
        }
        mbar_expect_tx(bar_full(s), TILE_BYTES + (KIND == KIND_SS ? 1 : 2) * B_PLANE);
        if (p.mode == 0) {
          if (k0 < p.C1) tma_load_2d(st, &mapA, k0, tc_.m0, bar_full(s));
          else tma_load_2d(st, &mapA2, k0 - p.C1, tc_.m0, bar_full(s));
        } else {
          const int tap = kb / cblocks, cb = kb - tap * cblocks;
          const int dy = tap / 3, dx = tap - dy * 3;
          tma_load_4d(st, &mapA, cb * TBK, tc_.x0 * p.cstride + dx - p.cpad, tc_.y0 * p.cstride + dy - p.cpad, tc_.b0,
                      bar_full(s));                                                   // OOB -> zeros = padding
        }
        tma_load_2d(sb, &mapB, k0, tc_.n0, bar_full(s));
        if (KIND != KIND_SS) tma_load_2d(sb + B_PLANE, &mapBlo, k0, tc_.n0, bar_full(s));
      }
      if (staged) {
        // the epilogue's slots, as ring stages nst, nst + 1, ...: each frees as the consumers retire the stage it held, and the
        // residual boxes land there while the last stages' wgmmas run
        if (p.residual) mbar_expect_tx(bar_res, BN * TBM * 4);
        for (int k = 0; k < EPI_SLOTS; ++k, ++it) {
          const int s = it % STAGES;
          mbar_wait(bar_empty(s), ((it / STAGES) & 1) ^ 1);
          if (!p.residual) continue;
          for (int b = k * EPI_PER_SLOT; b < min(BN / TBK, (k + 1) * EPI_PER_SLOT); ++b) {
            const uint32_t dst = epi_box(b);
            if (p.mode == 0) tma_load_2d(dst, &mapR, tc_.n0 + b * TBK, tc_.m0, bar_res);
            else tma_load_4d(dst, &mapR, tc_.n0 + b * TBK, tc_.x0, tc_.y0, tc_.b0, bar_res);
          }
        }
        if (!p.residual) mbar_arrive(bar_res);
      }
    }
    return;
  }

  // ============================================================================= consumer warpgroups
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wg = (warp >> 2) - 1;                  // 0, 1: rows [64 wg, 64 wg + 64) of the tile
  const int wi = warp & 3, g = lane >> 2, qd = lane & 3;
  const int r0 = wg * 64 + wi * 16 + g;            // tile rows r0 and r0 + 8 of this thread
  const int ea = H16 ? h16_a_exp(p) : 0;
  const float asc = exp2i(ea);
  float omax_cta = 0.f;                            // PERSIST: range of C over the CTA's work items
  int g0 = 0;                                      // PERSIST: ring stage of the work item's first stage
#pragma unroll 1
  for (int t = blockIdx.x, item = 0;;) {           // PERSIST: work items t = blockIdx.x, + gridDim.x, ... (item counts them); else one
    const int kchunk = (tc_.kb1 - tc_.kb0) <= 2 * CF::KCHUNK ? 2 * CF::KCHUNK : CF::KCHUNK;
    // conv: pixel of each of this thread's two rows (the epilogue masks rows outside the map)
    int px[2] = {0, 0}, py[2] = {0, 0}, pb[2] = {0, 0};
    if (p.mode == 1) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int r = r0 + 8 * i;
        px[i] = tc_.x0 + r % p.bw; py[i] = tc_.y0 + (r / p.bw) % p.bh; pb[i] = tc_.b0 + r / (p.bw * p.bh);
      }
    }

    float acc[NACC], tot[NACC];
#pragma unroll
    for (int j = 0; j < NACC; ++j) { acc[j] = 0.f; tot[j] = 0.f; }

    // Software pipeline over the stages of the work item: while the wgmmas of stage it run, stage it + 1's A is split into the
    // other fragment set; wgmma.wait_group 1 then retires stage it - 1, whose smem slot goes back to the producer.
    struct Frag { uint32_t h[KSTEPS][4], l[KSTEPS][4]; };     // A fragments of one stage's K steps (rows r0 / r0 + 8), hi / lo

    // wait for stage it to land, then split its A into f
    auto load_split = [&](int it, Frag& f) {
      const int s = (g0 + it) % STAGES;
      mbar_wait(bar_full(s), ((g0 + it) / STAGES) & 1);
      const uint32_t st = base + s * STAGE_BYTES;
      if (KIND == KIND_SS) {
        // raw fp32 B tile -> TF32 hi in place, lo into the second plane (both consumer warpgroups, then a named barrier)
        const uint32_t sb = st + A_BYTES;
        const int ct = threadIdx.x - 128;
#pragma unroll 4
        for (int i = ct; i < B_PLANE / 16; i += 256) {
          const uint32_t a = sb + (uint32_t)i * 16u;
          uint32_t v[4], h[4], l[4];
          asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v[0]), "=r"(v[1]), "=r"(v[2]), "=r"(v[3]) : "r"(a));
#pragma unroll
          for (int c = 0; c < 4; ++c) { h[c] = rn_tf32(v[c]); l[c] = tf32_lo(__uint_as_float(v[c]), h[c]); }
          asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(h[0]), "r"(h[1]), "r"(h[2]), "r"(h[3]) : "memory");
          asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a + B_PLANE), "r"(l[0]), "r"(l[1]), "r"(l[2]), "r"(l[3]) : "memory");
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the tensor core
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
#pragma unroll
      for (int kk = 0; kk < KSTEPS; ++kk) {
        if (H16) {
#pragma unroll
          for (int i = 0; i < 2; ++i) {                 // i: row r0 + 8 i
            const int r = r0 + 8 * i;
#pragma unroll
            for (int hk = 0; hk < 2; ++hk) {            // hk: k 2qd (+1) or 2qd + 8 (+1)
              const int k = kk * 16 + hk * 8 + 2 * qd;
              float2 x;
              asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(x.x), "=f"(x.y)
                           : "r"(st + (uint32_t)r * 128u + ((((uint32_t)k >> 2) ^ (uint32_t)(r & 7)) << 4) + (uint32_t)(k & 3) * 4u));
              if (ea != 0) { x.x *= asc; x.y *= asc; }
              const __half2 h = __floats2half2_rn(x.x, x.y);       // .x (low half) = even k
              f.h[kk][hk * 2 + i] = *reinterpret_cast<const uint32_t*>(&h);
              if (!FAST) {
                const float2 hf = __half22float2(h);
                const __half2 l = __floats2half2_rn(x.x - hf.x, x.y - hf.y);
                f.l[kk][hk * 2 + i] = *reinterpret_cast<const uint32_t*>(&l);
              }
            }
          }
        } else {
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int r = r0 + 8 * i;
#pragma unroll
            for (int hk = 0; hk < 2; ++hk) {            // k = 8 kk + qd (+4)
              const int k = kk * 8 + hk * 4 + qd;
              float x;
              asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x)
                           : "r"(st + (uint32_t)r * 128u + ((((uint32_t)k >> 2) ^ (uint32_t)(r & 7)) << 4) + (uint32_t)(k & 3) * 4u));
              const uint32_t h = rn_tf32(__float_as_uint(x));
              f.h[kk][hk * 2 + i] = h;
              f.l[kk][hk * 2 + i] = tf32_lo(x, h);
            }
          }
        }
      }
    };

    // the wgmmas of stage it from f: one straight-line batch, small terms first
    auto mma = [&](int it, const Frag& f) {
      const uint32_t sb = base + ((g0 + it) % STAGES) * STAGE_BYTES + A_BYTES;
      const uint64_t bhi = H16 ? make_desc_sw64(sb) : make_desc(sb), blo = H16 ? make_desc_sw64(sb + B_PLANE) : make_desc(sb + B_PLANE);
      wgmma_pin(acc);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KSTEPS; ++kk) {
        const uint64_t adv = (uint64_t)kk * 2u;       // 32 bytes per K step along the B row (64 B fp16 / 128 B fp32)
        if (H16) {
          if (!FAST) {
            Wgmma<BN>::f16_rs(acc, f.l[kk], bhi + adv);
            Wgmma<BN>::f16_rs(acc, f.h[kk], blo + adv);
          }
          Wgmma<BN>::f16_rs(acc, f.h[kk], bhi + adv);
        } else {
          Wgmma<BN>::tf32_rs(acc, f.l[kk], bhi + adv);
          Wgmma<BN>::tf32_rs(acc, f.h[kk], blo + adv);
          Wgmma<BN>::tf32_rs(acc, f.h[kk], bhi + adv);
        }
      }
      wgmma_commit();
    };

    // stage it: its fragments are in cur; nxt held stage it - 1's
    int kin = 0;
    auto step = [&](int it, const Frag& cur, Frag& nxt) {
      mma(it, cur);
      wgmma_wait1();                                  // stage it - 1 has retired: its slot and its fragment set are free
      if (it > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty((g0 + it - 1) % STAGES));
      }
      if (it + 1 < nst) load_split(it + 1, nxt);
      if (++kin == kchunk || it == nst - 1) {        // chunk complete: retire it, round-to-nearest fp32 add into the total
        wgmma_wait0();
        wgmma_pin(acc);
#pragma unroll
        for (int j = 0; j < NACC; ++j) { tot[j] += acc[j]; acc[j] = 0.f; }
        kin = 0;
      }
    };

    Frag fa, fb;
    load_split(0, fa);
    if (threadIdx.x == 128 && item == 0) TL_STAMP(2);
#pragma unroll 1
    for (int it = 0; it < nst; it += 2) {
      step(it, fa, fb);
      if (it + 1 < nst) step(it + 1, fb, fa);
    }
    if (PERSIST) {
      // the last stage has retired (chunk end): its slot goes back to the producer, which fills the next work item's stages
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty((g0 + nst - 1) % STAGES));
    }
    // (otherwise the last stage's slot is not handed back: the producer has loaded everything)
    if (threadIdx.x == 128) TL_STAMP(3);

    // ============================================================================= epilogue (straight from registers)
    // accumulator element j*4 + i*2 + c: tile row r0 + 8 i, column n0 + 8 j + 2 qd + c
    const bool fin = PERSIST || p.splits == 1;       // otherwise: raw partial sums to ws[split][M][N]
    const float alpha = H16 ? p.alpha * exp2i(-ea) * exp2i(-p.b_exp) : p.alpha;
    long long mrow[2];
    bool rok[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = r0 + 8 * i;
      if (p.mode != 1) {
        mrow[i] = (long long)tc_.m0 + r;
        rok[i] = mrow[i] < p.M;
      } else {
        // rows of a tile that overhangs the map's right / bottom edge (or the batch) are not pixels: nothing is stored for them
        rok[i] = pb[i] < p.B && px[i] < p.W && py[i] < p.H;
        mrow[i] = ((long long)pb[i] * p.H + py[i]) * p.W + px[i];
      }
    }
    float omax = 0.f;
    const int n0 = tc_.n0, nend = tc_.nend;
    if (!fin) {
      float* const dst = p.ws + (long long)tc_.split * p.M * p.N;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int n = n0 + 8 * j + 2 * qd + c;
            if (rok[i] && n < nend) dst[mrow[i] * p.N + n] = tot[j * 4 + i * 2 + c];
          }
      return;
    }
    // pass 1: alpha, bias, per-image row vector
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int n = n0 + 8 * j + 2 * qd + c;
        const float bv = (p.bias && n < nend) ? p.bias[n] : 0.f;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float v = alpha * tot[j * 4 + i * 2 + c] + bv;
          if (p.rowvec && rok[i] && n < nend) v += p.rowvec[(mrow[i] / p.rows_per_batch) * p.ld_rowvec + n];
          tot[j * 4 + i * 2 + c] = v;
        }
      }
    if (!PERSIST && p.out_nchw) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (!rok[i]) continue;
        const long long bimg = mrow[i] / p.rows_per_img, rimg = mrow[i] - bimg * p.rows_per_img;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int n = n0 + 8 * j + 2 * qd + c;
            if (n < nend) p.C[(bimg * p.N + n) * p.rows_per_img + rimg] = tot[j * 4 + i * 2 + c];
          }
      }
      return;
    }
    if (!PERSIST && p.Ct_hi && n0 >= p.t_col0) {
      // transposed TF32-plane output (V^T)
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int n = n0 + 8 * j + 2 * qd + c;
            if (rok[i] && n < nend) {
              const float o = tot[j * 4 + i * 2 + c];
              const uint32_t hi = rn_tf32(__float_as_uint(o));
              const long long at = (long long)(n - p.t_col0) * p.ldt + mrow[i];
              p.Ct_hi[at] = __uint_as_float(hi);
              p.Ct_lo[at] = __uint_as_float(tf32_lo(o, hi));
              omax = fmaxf(omax, fabsf(o));
            }
          }
    } else {
      float* const dst = p.C + tc_.zb * p.sC_b + tc_.zh * p.sC_h;
      float* const dst_lo = p.C_lo ? p.C_lo + tc_.zb * p.sC_b + tc_.zh * p.sC_h : nullptr;
      // one loop body, compiled for each store path: STAGED writes every row and column of the tile into the epilogue's boxes (rows
      // and columns outside C are clipped by the TMA store), the other path stores the valid elements to global memory
      auto store_tile = [&](auto staged_c) {
        constexpr bool STAGED = decltype(staged_c)::value;
        // GEGLU tiles are [32 value | 32 gate] blocks: accumulator group j (value) pairs with j + 4 (gate)
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          if (p.geglu && (j & 4)) continue;
          const int n = n0 + 8 * j + 2 * qd;             // even; N % 4 == 0 (eligibility), so n + 1 < nend whenever n < nend
          const int nout = p.geglu ? (n >> 6) * 32 + (n & 63) : n;
          // STAGED: the column pair's box and its column in the box (GEGLU: boxes of the BN / 2 output columns)
          const int box = p.geglu ? j >> 3 : j >> 2, cc = 8 * (j & 3) + 2 * qd;
          float cs[2] = {0.f, 0.f}, cq[2] = {0.f, 0.f};
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            float2 o = make_float2(tot[j * 4 + i * 2], tot[j * 4 + i * 2 + 1]);
            if (p.geglu) {
              const float g0 = tot[(j + 4) * 4 + i * 2], g1 = tot[(j + 4) * 4 + i * 2 + 1];
              o.x *= 0.5f * g0 * (1.f + erff(g0 * 0.70710678118654752440f));     // exact-erf GELU as F.gelu
              o.y *= 0.5f * g1 * (1.f + erff(g1 * 0.70710678118654752440f));
            }
            if (STAGED) {
              // the 128B-swizzled box layout; the residual box holds its value at the same address
              const int r = r0 + 8 * i;
              const uint32_t a = epi_box(box) + (uint32_t)r * 128u + ((((uint32_t)cc >> 2) ^ (uint32_t)(r & 7)) << 4) + (uint32_t)(cc & 3) * 4u;
              if (p.residual) {
                float2 rv;
                asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(rv.x), "=f"(rv.y) : "r"(a));
                o.x += rv.x;
                o.y += rv.y;
              }
              asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(o.x), "f"(o.y) : "memory");
            }
            if (!rok[i] || n >= nend) continue;
            if (!STAGED && p.residual) {
              o.x += p.residual[mrow[i] * p.ldr + n];
              o.y += p.residual[mrow[i] * p.ldr + n + 1];
            }
            if (p.c_stats) { cs[0] += o.x; cq[0] += o.x * o.x; cs[1] += o.y; cq[1] += o.y * o.y; }
            if (!STAGED) {
              float* const d = dst + mrow[i] * p.ldc + nout;
              if (dst_lo) {                          // operand planes for a following tensor-core consumer
                const uint32_t hx = rn_tf32(__float_as_uint(o.x)), hy = rn_tf32(__float_as_uint(o.y));
                *reinterpret_cast<float2*>(dst_lo + mrow[i] * p.ldc + nout) = make_float2(__uint_as_float(tf32_lo(o.x, hx)), __uint_as_float(tf32_lo(o.y, hy)));
                o = make_float2(__uint_as_float(hx), __uint_as_float(hy));
              }
              *reinterpret_cast<float2*>(d) = o;
            }
            omax = fmaxf(omax, fmaxf(fabsf(o.x), fabsf(o.y)));
          }
          if (p.c_stats) {
            // GroupNorm statistics: fold the warp's 16 rows (one image: host-checked), one fp64 atomic per (column, statistic)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
#pragma unroll
              for (int o2 = 4; o2 < 32; o2 <<= 1) {
                cs[c] += __shfl_xor_sync(0xffffffffu, cs[c], o2);
                cq[c] += __shfl_xor_sync(0xffffffffu, cq[c], o2);
              }
            }
            const long long mq = __shfl_sync(0xffffffffu, rok[0] ? mrow[0] : -1LL, 0);     // first row of the warp
            if (g == 0 && mq >= 0 && n < nend) {
              double* sp = p.c_stats + ((mq / p.rows_per_batch) * p.N + n) * 2;
              atomicAdd(sp, (double)cs[0]); atomicAdd(sp + 1, (double)cq[0]);
              atomicAdd(sp + 2, (double)cs[1]); atomicAdd(sp + 3, (double)cq[1]);
            }
          }
        }
      };
      if (!staged) {
        store_tile(std::false_type());
      } else {
        mbar_wait(bar_res, PERSIST ? item & 1 : 0);  // the boxes' slots are free and the residual boxes have landed
        if (threadIdx.x == 128) TL_STAMP(4);
        store_tile(std::true_type());
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the TMA store
        asm volatile("bar.sync 2, 256;" ::: "memory");                 // the consumer warpgroups' rows are all written
        if (PERSIST) {
          if (threadIdx.x == 128) mbar_arrive(bar_out);                // thread 32 stores them
        } else if (threadIdx.x == 128) {
          const int c0 = p.geglu ? n0 / 2 : n0, ncols = p.geglu ? p.N / 2 : p.N;
          for (int b = 0; b < (p.geglu ? BN / 64 : BN / TBK) && c0 + b * TBK < ncols; ++b) {
            if (p.mode == 0) tma_store_2d(epi_box(b), &mapC, c0 + b * TBK, tc_.m0);
            else tma_store_4d(epi_box(b), &mapC, c0 + b * TBK, tc_.x0, tc_.y0, tc_.b0);
          }
          bulk_commit();
          TL_STAMP(5);
          bulk_wait0();                              // written, not only read: a dependent launch reads C after its griddepcontrol.wait
          TL_STAMP(6);
        }
      }
    }
    omax_cta = PERSIST ? fmaxf(omax_cta, omax) : omax;
    if (!PERSIST) break;
    t += gridDim.x;
    if (t >= p.total_tiles) break;
    ++item;
    g0 += nst;
    tc_ = tile_coord(p, t, num_kb);
    nst = tc_.kb1 - tc_.kb0;
  }
  if (p.c_amax) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) omax_cta = fmaxf(omax_cta, __shfl_xor_sync(0xffffffffu, omax_cta, o));
    if (lane == 0) atomicMax(reinterpret_cast<unsigned int*>(p.c_amax), __float_as_uint(omax_cta));     // non-negative floats order like their bit patterns
  }
}

// C = alpha * sum_s ws[s] (+bias) (+row vector) (+residual): fixed summation order, so split-K stays deterministic
__global__ void splitk_reduce_kernel(const float* ws, int splits, TcParams p, int h16) {
  pdl_trigger();
  pdl_wait();
  const long long total4 = (long long)p.M * p.N / 4;
  const float alpha = h16 ? p.alpha * exp2i(-h16_a_exp(p)) * exp2i(-p.b_exp) : p.alpha;
  float omax = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
    const long long e = i * 4;
    const long long m = e / p.N;
    const int n = (int)(e - m * p.N);
    float4 a = *reinterpret_cast<const float4*>(ws + e);
    for (int s = 1; s < splits; ++s) {
      const float4 b = *reinterpret_cast<const float4*>(ws + (long long)s * p.M * p.N + e);
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    a.x *= alpha; a.y *= alpha; a.z *= alpha; a.w *= alpha;
    if (p.bias) { a.x += p.bias[n]; a.y += p.bias[n + 1]; a.z += p.bias[n + 2]; a.w += p.bias[n + 3]; }    // any alignment: gemm_tc does not check the bias
    if (p.rowvec) { const float4 t = *reinterpret_cast<const float4*>(p.rowvec + (m / p.rows_per_batch) * p.ld_rowvec + n); a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w; }
    if (p.residual) { const float4 t = *reinterpret_cast<const float4*>(p.residual + m * p.ldr + n); a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w; }
    if (p.C_lo) {
      float4 hi, lo;
      hi.x = __uint_as_float(rn_tf32(__float_as_uint(a.x))); lo.x = __uint_as_float(rn_tf32(__float_as_uint(a.x - hi.x)));
      hi.y = __uint_as_float(rn_tf32(__float_as_uint(a.y))); lo.y = __uint_as_float(rn_tf32(__float_as_uint(a.y - hi.y)));
      hi.z = __uint_as_float(rn_tf32(__float_as_uint(a.z))); lo.z = __uint_as_float(rn_tf32(__float_as_uint(a.z - hi.z)));
      hi.w = __uint_as_float(rn_tf32(__float_as_uint(a.w))); lo.w = __uint_as_float(rn_tf32(__float_as_uint(a.w - hi.w)));
      *reinterpret_cast<float4*>(p.C_lo + m * p.ldc + n) = lo;
      a = hi;
    }
    *reinterpret_cast<float4*>(p.C + m * p.ldc + n) = a;
    omax = fmaxf(omax, fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w))));
  }
  if (p.c_amax) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) omax = fmaxf(omax, __shfl_xor_sync(0xffffffffu, omax, o));
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned int*>(p.c_amax), __float_as_uint(omax));
  }
}

// x -> (rn_tf32(x), rn_tf32(x - rn_tf32(x)))  : one-time preparation of the weight planes for the TS variant
__global__ void split_planes_kernel(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t b = __float_as_uint(w[i]);
    const uint32_t h = rn_tf32(b);
    hi[i] = __uint_as_float(h);
    lo[i] = __uint_as_float(rn_tf32(__float_as_uint(w[i] - __uint_as_float(h))));
  }
}

// w' = w * 2^exp ; hi = fp16(w'), lo = fp16(w' - hi): one-time preparation of the weight planes for KIND_H16
__global__ void split_planes_h16_kernel(const float* __restrict__ w, __half* __restrict__ hi, __half* __restrict__ lo, size_t n, float scale) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float x = w[i] * scale;
    const __half h = __float2half_rn(x);
    hi[i] = h;
    lo[i] = __float2half_rn(x - __half2float(h));
  }
}

__global__ void amax_rows_kernel(const float* __restrict__ x, long long rows, int C, long long ld, float* __restrict__ slot) {
  float m = 0.f;
  const long long total = rows * (long long)(C >> 2);
  const int c4n = C >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / c4n;
    const int c4 = (int)(i - r * c4n);
    const float4 v = *reinterpret_cast<const float4*>(x + r * ld + 4 * c4);
    m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned int*>(slot), __float_as_uint(m));
}

// any C / stride (few-channel tensors: a 3-channel VQ latent)
__global__ void amax_rows_scalar_kernel(const float* __restrict__ x, long long rows, int C, long long ld, float* __restrict__ slot) {
  float m = 0.f;
  const long long total = rows * (long long)C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C;
    m = fmaxf(m, fabsf(x[r * ld + (i - r * C)]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned int*>(slot), __float_as_uint(m));
}

template <int KIND, int BN, bool PERSIST = false>
void set_smem_attr() {
  CDX_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<KIND, BN, PERSIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<KIND, BN, PERSIST>::SMEM_BYTES));
}

// cudaFuncSetAttribute is per DEVICE: remember which devices of this process have it (engines on several devices share the library)
void ensure_attr(int device) {
  static bool attr_set[64] = {};
  static std::mutex mtx;
  std::lock_guard<std::mutex> lock(mtx);
  const int d = device & 63;
  if (!attr_set[d]) {
    set_smem_attr<KIND_SS, 128>();
    set_smem_attr<KIND_TS, 128>();
    set_smem_attr<KIND_TS, 64>();
    set_smem_attr<KIND_H16, 128>();
    set_smem_attr<KIND_H16, 64>();
    set_smem_attr<KIND_H16_FAST, 128>();
    set_smem_attr<KIND_H16_FAST, 64>();
    set_smem_attr<KIND_H16, 128, true>();
    set_smem_attr<KIND_H16, 64, true>();
    set_smem_attr<KIND_H16_FAST, 128, true>();
    set_smem_attr<KIND_H16_FAST, 64, true>();
    attr_set[d] = true;
  }
}

template <int KIND, int BN>
void launch_gemm(const TcParams& p, const CUtensorMap& mA, const CUtensorMap& mA2, const CUtensorMap& mB, const CUtensorMap& mBlo,
                 const CUtensorMap& mR, const CUtensorMap& mC, cudaStream_t s) {
  launch_ex(tc_gemm_kernel<KIND, BN>, dim3((unsigned)p.total_tiles), dim3(TC_THREADS), Cfg<KIND, BN>::SMEM_BYTES, s, 1, mA, mA2, mB, mBlo, mR, mC, p);
}

// persistent grid: `ctas` CTAs walk the p.total_tiles work items
template <int KIND, int BN>
void launch_gemm_persist(const TcParams& p, int ctas, const CUtensorMap& mA, const CUtensorMap& mA2, const CUtensorMap& mB,
                         const CUtensorMap& mBlo, const CUtensorMap& mR, const CUtensorMap& mC, cudaStream_t s) {
  launch_ex(tc_gemm_kernel<KIND, BN, true>, dim3((unsigned)ctas), dim3(TC_THREADS), Cfg<KIND, BN, true>::SMEM_BYTES, s, 1, mA, mA2, mB, mBlo, mR, mC, p);
}

}  // namespace

void split_planes(Engine& e, const float* w, float* hi, float* lo, size_t n, cudaStream_t s) {
  if (e.dry()) return;
  size_t blocks = (n + 255) / 256;
  if (blocks > (size_t)e.num_sms * 16) blocks = (size_t)e.num_sms * 16;
  split_planes_kernel<<<(unsigned)(blocks ? blocks : 1), 256, 0, s>>>(w, hi, lo, n);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}

void split_planes_h16(Engine& e, const float* w, void* hi, void* lo, size_t n, int exp, cudaStream_t s) {
  if (e.dry()) return;
  size_t blocks = (n + 255) / 256;
  if (blocks > (size_t)e.num_sms * 16) blocks = (size_t)e.num_sms * 16;
  split_planes_h16_kernel<<<(unsigned)(blocks ? blocks : 1), 256, 0, s>>>(w, (__half*)hi, (__half*)lo, n, ldexpf(1.f, exp));
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}

void amax_rows(Engine& e, const float* x, long long rows, int C, long long ld, float* slot, cudaStream_t s) {
  if (e.dry()) return;
  if ((C & 3) || (ld & 3) || !a16(x)) {
    const long long total = rows * (long long)C;
    const int blocks = (int)std::min<long long>((total + 255) / 256, (long long)e.num_sms * 8);
    amax_rows_scalar_kernel<<<blocks > 0 ? blocks : 1, 256, 0, s>>>(x, rows, C, ld, slot);
    CDX_CUDA(cudaGetLastError());
    e.launches++;
    return;
  }
  const long long total = rows * (long long)(C >> 2);
  const int blocks = (int)std::min<long long>((total + 255) / 256, (long long)e.num_sms * 8);
  amax_rows_kernel<<<blocks > 0 ? blocks : 1, 256, 0, s>>>(x, rows, C, ld, slot);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}

int h16_exp_host(float amax) {
  if (!(amax > 0.f) || !std::isfinite(amax)) return 0;
  int ex;
  frexpf(amax, &ex);                    // amax = f * 2^ex, f in [0.5, 1)  ->  floor(log2 amax) = ex - 1
  return std::min(std::max(14 - (ex - 1), -100), 100);
}

// softmax(q k^T * scale) v on the tensor cores: two batched 3xTF32 contractions (KIND_SS) around the row-softmax kernel.
//   q, k : [B, N*, ...] token matrices (row strides ldq / ldk, head h at column h*head_stride)
//   vt   : V transposed, [heads*d, B*Nk] (row c = channel, column b*Nk + j), produced by a swapped-role GEMM
//   out  : [B, Nq, ldo], head h at column h*d
// Requires Nk % 32 == 0 (a K block must not run into the next sample's columns of vt), d % 4 == 0.
bool attention_tc(Engine& e, const float* q, int ldq, const float* k, int ldk, int head_stride, const float* vt, float* out, int ldo, int B,
                  int Nq, int Nk, int heads, int d, float scale, cudaStream_t s) {
  if ((Nk % TBK) || (d & 3) || (ldq & 3) || (ldk & 3) || (head_stride & 3) || (ldo & 3) || Nq < 64) return false;
  if (!a16(q) || !a16(k) || !a16(vt) || !a16(out)) return false;
  Scope sc(e.arena);
  const int ldS = Nk;
  float* S = (float*)e.arena.alloc((size_t)B * heads * Nq * ldS * sizeof(float));
  if (e.dry()) return true;
  ensure_attr(e.device);
  TcParams p;
  // ---- S = scale * Q K^T
  {
    memset(&p, 0, sizeof(p));
    p.mode = 2; p.M = Nq; p.N = Nk; p.K = d; p.heads = heads; p.alpha = scale;
    p.C = S; p.ldc = ldS; p.sC_b = (long long)heads * Nq * ldS; p.sC_h = (long long)Nq * ldS;
    p.rows_per_batch = 1;
    const int code[4] = {0, 2, 1, 3};      // dims {d, heads, rows, B}
    for (int i = 0; i < 4; ++i) { p.a_code[i] = code[i]; p.b_code[i] = code[i]; }
    uint64_t da[4] = {(uint64_t)d, (uint64_t)heads, (uint64_t)Nq, (uint64_t)B};
    uint64_t sa[3] = {(uint64_t)head_stride * 4, (uint64_t)ldq * 4, (uint64_t)Nq * ldq * 4};
    uint64_t db[4] = {(uint64_t)d, (uint64_t)heads, (uint64_t)Nk, (uint64_t)B};
    uint64_t sb[3] = {(uint64_t)head_stride * 4, (uint64_t)ldk * 4, (uint64_t)Nk * ldk * 4};
    uint32_t bx[4] = {TBK, 1, TBM, 1};
    const CUtensorMap& mA = get_map(q, 4, da, sa, bx);
    const CUtensorMap& mB = get_map(k, 4, db, sb, bx);
    ProfScope ps(e, s, PROF_BATCHED_TC, 2.0 * Nq * Nk * d * B * heads, 4.0 * B * heads * ((double)Nq * d + (double)Nk * d + (double)Nq * Nk), 1);
    p.splits = 1; p.kb_per_split = cdiv(d, TBK);
    p.tn_w = TBN;
    p.tiles_m = cdiv(Nq, TBM); p.tiles_n = cdiv(Nk, TBN); p.total_tiles = p.tiles_m * p.tiles_n * B * heads;
    launch_gemm<KIND_SS, 128>(p, mA, mA, mB, mB, mA, mA, s);
    CDX_CUDA(cudaGetLastError());
    e.launches++;
  }
  softmax_rows(e, S, (long long)B * heads * Nq, Nk, ldS, s);
  // ---- O = P V   (B operand = V^T rows h*d .. h*d+d-1, K along the sample's Nk columns)
  {
    memset(&p, 0, sizeof(p));
    p.mode = 2; p.M = Nq; p.N = d; p.K = Nk; p.heads = heads; p.alpha = 1.f;
    p.C = out; p.ldc = ldo; p.sC_b = (long long)Nq * ldo; p.sC_h = d;
    p.rows_per_batch = 1;
    const int ac[4] = {0, 1, 2, 3};        // P dims {Nk, Nq, heads, B}
    const int bc[4] = {0, 3, 1, 4};        // V^T dims {Nk, B, heads*d, 1}
    for (int i = 0; i < 4; ++i) { p.a_code[i] = ac[i]; p.b_code[i] = bc[i]; }
    p.b_rowoff_h = d;
    uint64_t da[4] = {(uint64_t)Nk, (uint64_t)Nq, (uint64_t)heads, (uint64_t)B};
    uint64_t sa[3] = {(uint64_t)ldS * 4, (uint64_t)Nq * ldS * 4, (uint64_t)heads * Nq * ldS * 4};
    uint32_t bxa[4] = {TBK, TBM, 1, 1};
    uint64_t db[4] = {(uint64_t)Nk, (uint64_t)B, (uint64_t)heads * d, 1};
    uint64_t sb[3] = {(uint64_t)Nk * 4, (uint64_t)B * Nk * 4, (uint64_t)B * Nk * 4 * heads * d};
    uint32_t bxb[4] = {TBK, 1, TBN, 1};
    const CUtensorMap& mA = get_map(S, 4, da, sa, bxa);
    const CUtensorMap& mB = get_map(vt, 4, db, sb, bxb);
    ProfScope ps(e, s, PROF_BATCHED_TC, 2.0 * Nq * Nk * d * B * heads, 4.0 * B * heads * ((double)Nq * Nk + (double)Nk * d + (double)Nq * d), 1);
    p.splits = 1; p.kb_per_split = cdiv(Nk, TBK);
    p.tn_w = TBN;
    p.tiles_m = cdiv(Nq, TBM); p.tiles_n = cdiv(d, TBN); p.total_tiles = p.tiles_m * p.tiles_n * B * heads;
    launch_gemm<KIND_SS, 128>(p, mA, mA, mB, mB, mA, mA, s);
    CDX_CUDA(cudaGetLastError());
    e.launches++;
  }
  return true;
}

// Pixel box of a conv3x3 M tile for an output map whose sides are not both powers of two: bw x bh pixels of bn images, bw*bh*bn == 128,
// so every factor is a power of two and the box generally overhangs the map.  The box that covers [B, H, W] with the fewest tiles
// wins (fewest masked rows); ties go to the smallest halo per tile, bn * (bw + 2) * (bh + 2) pixels fetched (then the wider box: longer
// contiguous TMA rows).  Tiles past the map's edge read TMA's zero fill and their rows are masked in the epilogue.
static void conv_ragged_tile(int W, int H, int B, int stride, int* bw_out, int* bh_out, int* bn_out) {
  long long best_tiles = -1, best_halo = 0;
  for (int bw = TBM; bw >= 1; bw >>= 1) {
    for (int bh = TBM / bw; bh >= 1; bh >>= 1) {
      const int bn = TBM / (bw * bh);
      if (bw * stride > 256 || bh * stride > 256) continue;
      const long long tiles = (long long)cdiv(W, bw) * cdiv(H, bh) * cdiv(B, bn);
      const long long halo = (long long)bn * (bw + 2) * (bh + 2);
      if (best_tiles < 0 || tiles < best_tiles || (tiles == best_tiles && halo < best_halo)) {
        best_tiles = tiles; best_halo = halo;
        *bw_out = bw; *bh_out = bh; *bn_out = bn;
      }
    }
  }
}

bool gemm_tc(Engine& e, const GemmArgs& a, cudaStream_t s, int* side_done) {
  // ---- eligibility (everything else takes the FFMA tiles)
  if (a.batch * a.heads != 1 || a.b_kn) return false;
  if (a.geglu && ((a.N % TBN) || a.out_nchw || a.Cout_lo || a.residual || a.rowvec || a.mode != 0)) return false;
  if (a.Cout_lo && a.out_nchw) return false;
  if (a.Ct_hi && (a.mode != 0 || !a.Ct_lo || a.out_nchw || a.geglu || a.residual || a.rowvec || (a.t_col0 % TBN) || a.t_col0 >= a.N)) return false;
  if (a.out_nchw && (a.rowvec || a.residual)) return false;
  if (!a.out_nchw && ((a.N & 3) || (a.ldc & 3) || !a16(a.Cout))) return false;   // (the NCHW epilogue stores scalars: any N)
  if (!a16(a.Bw) || (a.ldb & 3)) return false;
  if (a.rowvec && (!a16(a.rowvec) || (a.ld_rowvec & 3))) return false;
  if (a.residual && (!a16(a.residual) || (a.ldr & 3))) return false;
  if (!a16(a.A) || (a.lda & 3)) return false;
  if (a.M < 64) return false;
  if (a.N < 32 && a.M < 2048) return false;         // tiny problems: tile quantisation loses to the FFMA 64x64 tiles; thin-N with a
                                                    // large M (e.g. the 320 -> 4 output conv) still wins by a wide margin

  TcParams p;
  memset(&p, 0, sizeof(p));
  p.M = a.M; p.N = a.N; p.K = a.K;
  p.C = a.Cout; p.ldc = a.ldc;
  p.C_lo = a.out_nchw ? nullptr : a.Cout_lo;
  p.Ct_hi = a.Ct_hi; p.Ct_lo = a.Ct_lo; p.t_col0 = a.t_col0; p.ldt = a.ldt;
  p.bias = a.bias;
  p.rowvec = a.rowvec; p.ld_rowvec = a.ld_rowvec; p.rows_per_batch = a.rows_per_batch > 0 ? a.rows_per_batch : 1;
  p.residual = a.residual; p.ldr = a.ldr;
  p.alpha = a.alpha;
  p.geglu = a.geglu;
  p.out_nchw = a.out_nchw; p.rows_per_img = a.rows_per_img > 0 ? a.rows_per_img : 1;
  p.heads = 1;
  const CUtensorMap *mA, *mA2, *mB, *mBlo;
  if (a.mode == 0) {
    if (a.K & 3) return false;
    if (a.A2) {
      if ((a.C1 % TBK) || !a16(a.A2) || (a.lda2 & 3) || (a.C2 & 3)) return false;
    }
    p.mode = 0; p.C1 = a.C1; p.C2 = a.C2;
    {
      uint64_t d[2] = {(uint64_t)a.C1, (uint64_t)a.M}, st[1] = {(uint64_t)a.lda * 4};
      uint32_t bx[2] = {TBK, TBM};
      mA = &get_map(a.A, 2, d, st, bx);
    }
    if (a.A2) {
      uint64_t d[2] = {(uint64_t)a.C2, (uint64_t)a.M}, st[1] = {(uint64_t)a.lda2 * 4};
      uint32_t bx[2] = {TBK, TBM};
      mA2 = &get_map(a.A2, 2, d, st, bx);
    } else {
      mA2 = mA;
    }
    p.tiles_m = cdiv(a.M, TBM);
  } else {
    if ((a.stride != 1 && a.stride != 2) || a.up != 1) return false;
    if (a.C1 % TBK) return false;
    if (a.Hin != a.Hout * a.stride || a.Win != a.Wout * a.stride) return false;
    const int B = a.M / (a.Hout * a.Wout);
    int bw, bh, bn;
    if (pow2(a.Hout) && pow2(a.Wout)) {
      bw = a.Wout < 16 ? a.Wout : 16;
      bh = a.Hout < TBM / bw ? a.Hout : TBM / bw;
      bn = TBM / (bw * bh);
    } else {
      conv_ragged_tile(a.Wout, a.Hout, B, a.stride, &bw, &bh, &bn);
    }
    if (bn > 256 || bw * a.stride > 256 || bh * a.stride > 256) return false;
    p.mode = 1; p.C1 = a.C1; p.H = a.Hout; p.W = a.Wout; p.B = B;      // H, W: OUTPUT grid (tile -> row mapping)
    p.bw = bw; p.bh = bh; p.bn = bn;
    p.cstride = a.stride; p.cpad = a.pad;
    p.tiles_x = cdiv(a.Wout, bw); p.tiles_y = cdiv(a.Hout, bh);
    uint64_t d[4] = {(uint64_t)a.C1, (uint64_t)a.Win, (uint64_t)a.Hin, (uint64_t)B};
    uint64_t st[3] = {(uint64_t)a.lda * 4, (uint64_t)a.lda * 4 * a.Win, (uint64_t)a.lda * 4 * a.Win * a.Hin};
    // stride 2 (Downsample convs): TMA traverses every 2nd pixel; box = 2x the number of pixels wanted
    uint32_t bx[4] = {TBK, (uint32_t)(bw * a.stride), (uint32_t)(bh * a.stride), (uint32_t)bn};
    uint32_t es[4] = {1, (uint32_t)a.stride, (uint32_t)a.stride, 1};
    mA = &get_map(a.A, 4, d, st, bx, es);
    mA2 = mA;
    p.tiles_m = p.tiles_x * p.tiles_y * cdiv(B, bn);
  }
  // ---- operand path: fp16-split (KIND_H16) when the engine selects it, the weights have fp16 planes and the geometry allows it
  // (K a multiple of 32: whole 32-K ring stages; fp16 B rows 16-byte aligned); else TF32 planes (KIND_TS); else SS
  const bool ts = a.Bw_hi != nullptr && a.Bw_lo != nullptr && a16(a.Bw_hi) && a16(a.Bw_lo);
  const bool h16 = e.tc_kind >= 1 && a.Bw_h_hi && a.Bw_h_lo && a16(a.Bw_h_hi) && a16(a.Bw_h_lo) && (a.K % TBK) == 0 && (a.ldb % 8) == 0 &&
                   (!a.A2 || (a.C2 % TBK) == 0);
  // The planner counts fp16-split work in 64-K blocks (its cost constants are per 64 K), so its choice of (w, S) -- and with it the
  // split-K boundaries -- does not depend on the ring's stage size; kb_per_split is converted to 32-K stages below.
  const int bk = h16 ? 64 : TBK;
  const int num_kb = cdiv(a.K, bk);
  // Work partition: tile width w (128 or 64 columns: the two wgmma widths compiled in) and split-K factor S, chosen together against
  // wave quantisation of one-CTA-per-work-item launches on num_sms SMs with a cost model in cycles: one k-block of a w-wide tile
  // ~ kc0 + kc1 w, ~3000 per work item for the epilogue, plus the split-K partial-sum traffic (S writes + S reads + 1 write of M*N
  // floats at ~3 TB/s); a split must buy >= 10 %.  (A model of the kernel's structure, not a fit to measurements.)  Unsplit work
  // that runs persistent (fp16 split, dense, staged store) overlaps each item's epilogue with the next item's main loop: its ~3000
  // is charged once per CTA.
  const bool persist_ok = e.persist && h16 && a.mode == 0 && !a.out_nchw && !a.Cout_lo && !a.Ct_hi;
  int best_w = TBN, best_s = 1;
  {
    // exact key (no hashing of packed fields: nothing can collide) of everything the cost model reads -- M too, through the split-K
    // traffic term: two shapes of one 128-row band may plan differently, and each must run its own plan whichever was planned first
    static std::map<std::array<int64_t, 6>, int> plan_cache;
    static std::mutex plan_mutex;                                          // engines on different devices may plan concurrently
    std::lock_guard<std::mutex> plan_lock(plan_mutex);
    const std::array<int64_t, 6> key = {a.M, p.tiles_m, a.N, num_kb, ((a.geglu || a.Ct_hi) ? 1 : 0) | (a.out_nchw ? 2 : 0) | (h16 ? 4 : 0) | (ts ? 8 : 0) |
                                        (persist_ok ? 16 : 0), e.num_sms};
    const double kc0 = h16 ? 700.0 : 400.0, kc1 = h16 ? 6.0 : 3.0;
    const int min_kbs = h16 ? 4 : 8;
    auto it = plan_cache.find(key);
    if (it != plan_cache.end()) {
      best_w = it->second >> 8;
      best_s = it->second & 255;
    } else {
      const bool only128 = a.geglu || a.Ct_hi || (!h16 && !ts);
      double best = 1e30;
      for (int w = TBN; w >= 64; w -= 64) {
        if (w == 64 && only128) break;
        const int tn = cdiv(a.N, w);
        double base = 0.0;
        for (int S = 1; S <= 8; ++S) {
          const int kbs = cdiv(num_kb, S);
          const int Sx = cdiv(num_kb, kbs);                                  // no empty splits
          if (S > 1 && (Sx != S || kbs < min_kbs || a.out_nchw || a.geglu || a.Ct_hi || (long long)p.tiles_m * tn >= 4LL * e.num_sms)) continue;
          const long long items = (long long)p.tiles_m * tn * S;
          const double waves = (double)cdiv(items, (long long)e.num_sms);
          double cost = S == 1 && persist_ok ? waves * kbs * (kc0 + kc1 * w) + 3000.0 : waves * (kbs * (kc0 + kc1 * w) + 3000.0);
          if (S == 1) base = cost;
          else cost += 4000.0 + (2.0 * S + 1.0) * (double)a.M * a.N * 4.0 / 3e12 * 1.8e9;
          if (cost < best - 1e-9 && (S == 1 || cost < 0.9 * base)) { best = cost; best_w = w; best_s = S; }
        }
      }
      plan_cache[key] = (best_w << 8) | best_s;
    }
  }
  p.tn_w = best_w;
  p.tiles_n = cdiv(a.N, best_w);
  const int tiles = p.tiles_m * p.tiles_n;
  p.kb_per_split = cdiv(num_kb, best_s);
  p.splits = cdiv(num_kb, p.kb_per_split);            // no empty splits
  p.kb_per_split *= bk / TBK;                         // in the kernel's 32-K stages
  p.total_tiles = tiles * p.splits;
  Scope ws_scope(e.arena);
  if (p.splits > 1) p.ws = (float*)e.arena.alloc((size_t)p.splits * a.M * a.N * sizeof(float));
  // fp16-split path: the A operand's range.  Tracked by its producer (a.a_amax), else measured here (one small extra launch).
  if (h16) {
    p.a_amax = a.a_amax;
    p.a2_amax = a.A2 ? a.a2_amax : nullptr;
    if (!p.a_amax) {
      float* slot = e.amax_slot();
      if (a.mode == 1) amax_rows(e, a.A, (long long)(a.M / (a.Hout * a.Wout)) * a.Hin * a.Win, a.C1, a.lda, slot, s);
      else amax_rows(e, a.A, a.M, a.C1, a.lda, slot, s);
      p.a_amax = slot;
    }
    if (a.A2 && !p.a2_amax) {
      float* slot = e.amax_slot();
      amax_rows(e, a.A2, a.M, a.C2, a.lda2, slot, s);
      p.a2_amax = slot;
    }
    p.b_exp = a.b_exp;
  }
  const bool fast = h16 && e.tc_kind == 2;
  // side outputs fused into the epilogue: range of C always (the split-K reduce kernel covers the split case); GroupNorm
  // statistics when every 32-row quadrant of a tile lies inside one image and the epilogue is the final one
  p.c_amax = a.out_nchw ? nullptr : a.c_amax;
  // (a tile that overhangs its map may start a warp on a masked row: its statistics are left to the standalone pass)
  const bool quad_ok = a.mode == 1 ? ((p.bw * p.bh) % 32 == 0 && p.tiles_x * p.bw == p.W && p.tiles_y * p.bh == p.H) : (a.rows_per_batch % 32 == 0);
  p.c_stats = (a.c_stats && quad_ok && p.splits == 1 && !a.out_nchw && !a.geglu && !a.Ct_hi && !a.Cout_lo && a.ldc == a.N) ? a.c_stats : nullptr;
  if (side_done)
    *side_done = (p.c_amax ? 1 : 0) | (p.c_stats ? 2 : 0) | (p.splits > 1 ? 4 : 0) |
                 route_plan(fast ? ROUTE_KIND_H16_FAST : h16 ? ROUTE_KIND_H16 : ts ? ROUTE_KIND_TS : ROUTE_KIND_SS, p.tn_w, p.splits);
  if (e.dry()) return true;
  if (h16) {
    uint64_t d[2] = {(uint64_t)a.K, (uint64_t)a.N}, st[1] = {(uint64_t)a.ldb * 2};
    uint32_t bx[2] = {(uint32_t)TBK, (uint32_t)p.tn_w};          // 32 fp16 = 64-byte rows, 64B swizzle
    mB = &get_map(a.Bw_h_hi, 2, d, st, bx, nullptr, 2, 64);
    mBlo = &get_map(a.Bw_h_lo, 2, d, st, bx, nullptr, 2, 64);
  } else {
    uint64_t d[2] = {(uint64_t)a.K, (uint64_t)a.N}, st[1] = {(uint64_t)a.ldb * 4};
    uint32_t bx[2] = {TBK, (uint32_t)p.tn_w};
    mB = &get_map(ts ? a.Bw_hi : a.Bw, 2, d, st, bx);
    mBlo = ts ? &get_map(a.Bw_lo, 2, d, st, bx) : mB;
  }
  // staged epilogue: C (GEGLU: its N / 2 output columns) and the residual as 32-column boxes of the tile's 128 rows -- [M] rows, or
  // for a conv the NHWC output grid in the A box's pixel order {bw, bh, bn}
  const CUtensorMap *mR = mA, *mC = mA;
  if (staged_store(p)) {
    auto out_map = [&](const float* ptr, int cols, int ld) -> const CUtensorMap& {
      if (a.mode == 0) {
        uint64_t d[2] = {(uint64_t)cols, (uint64_t)a.M}, st[1] = {(uint64_t)ld * 4};
        uint32_t bx[2] = {TBK, TBM};
        return get_map(ptr, 2, d, st, bx);
      }
      uint64_t d[4] = {(uint64_t)cols, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.B};
      uint64_t st[3] = {(uint64_t)ld * 4, (uint64_t)ld * 4 * p.W, (uint64_t)ld * 4 * p.W * p.H};
      uint32_t bx[4] = {TBK, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
      return get_map(ptr, 4, d, st, bx);
    };
    mC = &out_map(a.Cout, a.geglu ? a.N / 2 : a.N, a.ldc);
    if (a.residual) mR = &out_map(a.residual, a.N, a.ldr);
  }
  ensure_attr(e.device);
  ProfScope ps(e, s, a.mode == 1 ? PROF_CONV_TC : PROF_DENSE_TC, 2.0 * a.M * a.N * a.K,
               4.0 * ((double)a.M * a.K / (a.mode == 1 ? 9 : 1) + (double)a.N * a.K + (double)a.M * a.N), 1);
  ps.note("M%d N%d K%d w%d tiles%d S%d %s%s%s%s%s box%dx%dx%d", a.M, a.N, a.K, p.tn_w, tiles, p.splits, h16 ? (fast ? "H16x1" : "H16") : ts ? "TS" : "SS",
          a.Cout_lo ? " planes" : "", a.geglu ? " geglu" : "", a.residual ? " res" : "", persist_ok && staged_store(p) ? " persist" : "", p.bw, p.bh, p.bn);
  const bool persist = persist_ok && staged_store(p);
  const int ctas = (int)std::min<long long>(p.total_tiles, e.persist_grid > 0 ? std::min(e.persist_grid, e.num_sms) : e.num_sms);
  if (persist && fast && p.tn_w == 128) launch_gemm_persist<KIND_H16_FAST, 128>(p, ctas, *mA, *mA2, *mB, *mBlo, *mR, *mC, s);
  else if (persist && fast) launch_gemm_persist<KIND_H16_FAST, 64>(p, ctas, *mA, *mA2, *mB, *mBlo, *mR, *mC, s);
  else if (persist && p.tn_w == 128) launch_gemm_persist<KIND_H16, 128>(p, ctas, *mA, *mA2, *mB, *mBlo, *mR, *mC, s);
  else if (persist) launch_gemm_persist<KIND_H16, 64>(p, ctas, *mA, *mA2, *mB, *mBlo, *mR, *mC, s);
  else if (fast && p.tn_w == 128) launch_gemm<KIND_H16_FAST, 128>(p, *mA, *mA2, *mB, *mBlo, *mR, *mC, s);
  else if (fast) launch_gemm<KIND_H16_FAST, 64>(p, *mA, *mA2, *mB, *mBlo, *mR, *mC, s);
  else if (h16 && p.tn_w == 128) launch_gemm<KIND_H16, 128>(p, *mA, *mA2, *mB, *mBlo, *mR, *mC, s);
  else if (h16) launch_gemm<KIND_H16, 64>(p, *mA, *mA2, *mB, *mBlo, *mR, *mC, s);
  else if (ts && p.tn_w == 128) launch_gemm<KIND_TS, 128>(p, *mA, *mA2, *mB, *mBlo, *mR, *mC, s);
  else if (ts) launch_gemm<KIND_TS, 64>(p, *mA, *mA2, *mB, *mBlo, *mR, *mC, s);
  else launch_gemm<KIND_SS, 128>(p, *mA, *mA2, *mB, *mBlo, *mR, *mC, s);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
  if (p.splits > 1) {
    const long long total4 = (long long)a.M * a.N / 4;
    const int blocks = (int)std::min<long long>((total4 + 255) / 256, (long long)e.num_sms * 8);
    launch_ex(splitk_reduce_kernel, dim3((unsigned)blocks), dim3(256), 0, s, 1, p.ws, p.splits, p, h16 ? 1 : 0);
    CDX_CUDA(cudaGetLastError());
    e.launches++;
  }
  return true;
}

}  // namespace cdx

#ifdef CDX_GEMM_TIMELINE
// Timeline probe variant only: point the GEMM's stamps at `buf` (TL_SLOTS uint64 per CTA of the largest grid the caller runs; null:
// no stamps).  Returns 0 on success.
extern "C" int cdx_gemm_timeline_buffer(void* buf) {
  return cudaMemcpyToSymbol(cdx::g_gemm_timeline, &buf, sizeof(buf)) == cudaSuccess ? 0 : 1;
}
#endif
