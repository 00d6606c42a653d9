// kernels_norm.cu -- HBM-bound normalisation kernels: GroupNorm(32)(+scale-shift)(+SiLU), LayerNorm, row softmax.
//
// GroupNorm follows GroupNorm32 / Normalize (util.py:215-217 eps 1e-5; attention.py:76-77 and model.py:38-39 eps 1e-6)
// on NHWC activations, optionally over the channel concatenation of two tensors (the U-Net skip `th.cat`, OAI:736)
// so that the concat is never materialised before the norm.
//
// Statistics are per-(image, channel) fp64 sums  stats[(b*C + c)*2 + {sum, sum of squares}]  attached to the TENSOR, not to the
// norm: the tensor-core GEMM that produces an activation adds them from its epilogue registers (kernels_tc.cu), so a GroupNorm
// over it -- or over the concat of two such tensors, channel sums being additive -- costs no statistics pass at all; tensors
// from other producers get them from gn_stats_kernel (one read).  The apply kernel then is the algorithmic one read + one write:
// every block folds the channel sums of its image into the 32 group means / rstds (fp64), y = x * sc + sh per channel (the form
// ATen's CPU kernel uses), optional (1 + scale) / shift of the improved-DDPM scale-shift norm, optional SiLU, and it tracks
// max |y| for the fp16-split GEMM that consumes y.
// Row-mapped apply (src_img): the block writing image b reads image src_img[b]'s input, statistics and scale / shift, so image b
// receives exactly image src_img[b]'s normalised activation (Plug-and-Play feature injection: the conv after the norm sees the
// source row's operand and adds the target's own residual).  The bytes moved and the launch are the plain apply's.
#include <algorithm>

#include "tc_common.cuh"      // pdl_trigger / pdl_wait / launch_ex

namespace cdx {
namespace {

constexpr int GN_GROUPS = 32;

// slot <- max(slot, block-wide max of v): one atomic per block at most, and none once the slot already holds a larger value
// (same-address atomics serialise in L2: one per warp costs more than the kernel itself on the big activations)
__device__ __forceinline__ void block_amax(float v, float* slot) {
  __shared__ float s_wmax[32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = (blockDim.x + 31) >> 5;
  if (lane == 0) s_wmax[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < nwarps ? s_wmax[lane] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (lane == 0 && v > *reinterpret_cast<volatile float*>(slot)) atomicMax(reinterpret_cast<unsigned int*>(slot), __float_as_uint(v));
  }
}

// per-(image, channel) sums of one source: grid (row chunks, B); thread (tr, tc) owns float4 channel slots tc, tc+ncol, ...
__global__ void __launch_bounds__(256) gn_stats_kernel(const float* __restrict__ x, int C, int HW, int rows_per_chunk, double* __restrict__ stats) {
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int r0 = chunk * rows_per_chunk;
  const int r1 = min(HW, r0 + rows_per_chunk);
  const int C4 = C >> 2;
  const int ncol = min(C4, (int)blockDim.x);
  const int nrow_par = blockDim.x / ncol;
  const int tr = threadIdx.x / ncol, tc = threadIdx.x - tr * ncol;
  if (tr >= nrow_par) return;
  for (int c4 = tc; c4 < C4; c4 += ncol) {
    const int c = c4 * 4;
    double s[4] = {0.0, 0.0, 0.0, 0.0}, q[4] = {0.0, 0.0, 0.0, 0.0};
    const float* base = x + (long long)b * HW * C + c;
    int r = r0 + tr;
    for (; r + 3 * nrow_par < r1; r += 4 * nrow_par) {      // 4 independent 128-bit loads in flight per thread
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = *reinterpret_cast<const float4*>(base + (long long)(r + u * nrow_par) * C);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const double d0 = v[u].x, d1 = v[u].y, d2 = v[u].z, d3 = v[u].w;
        s[0] += d0; q[0] += d0 * d0;
        s[1] += d1; q[1] += d1 * d1;
        s[2] += d2; q[2] += d2 * d2;
        s[3] += d3; q[3] += d3 * d3;
      }
    }
    for (; r < r1; r += nrow_par) {
      const float4 v = *reinterpret_cast<const float4*>(base + (long long)r * C);
      const double d0 = v.x, d1 = v.y, d2 = v.z, d3 = v.w;
      s[0] += d0; q[0] += d0 * d0;
      s[1] += d1; q[1] += d1 * d1;
      s[2] += d2; q[2] += d2 * d2;
      s[3] += d3; q[3] += d3 * d3;
    }
    double* o = stats + ((long long)b * C + c) * 2;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      atomicAdd(o + 2 * j, s[j]);
      atomicAdd(o + 2 * j + 1, q[j]);
    }
  }
}

// grid (row chunks, B); thread (tr, tc) owns channel vectors tc, tc+ncol, ... (so group / affine coefficients are hoisted out
// of the row loop) and walks the chunk's rows 4 at a time.  Dynamic smem: float2 (sc, sh) per channel.  ab_out (optional): the
// first row chunk of each image stores that table, ab_out[b*C + c] = (a, o) with y = silu?(x * a + o).  src_img (optional,
// device [B]): image b is written from image src_img[b]'s input, statistics and scale / shift (the file header's row-mapped apply).
__global__ void __launch_bounds__(256) gn_apply_kernel(const float* x1, int C1, const float* x2, int C2,
                                                       const float* gamma, const float* beta,
                                                       const double* st1, const double* st2, double inv_count,
                                                       float eps, int silu,
                                                       const float* scale, const float* shift,
                                                       int ld_ss, float* y, int HW, int rows_per_chunk, float* amax,
                                                       float2* ab_out, const int* src_img) {
  tc::pdl_trigger();
  tc::pdl_wait();
  const int C = C1 + C2;
  const int cpg = C / GN_GROUPS;
  const int C4 = C >> 2;
  const int bo = blockIdx.y;                                            // the image written
  const int b = src_img ? __ldcg(src_img + bo) : bo;                    // the image read (coherent: after the dependent-launch wait)
  const int r0 = blockIdx.x * rows_per_chunk;
  const int r1 = min(HW, r0 + rows_per_chunk);
  const int ncol = min(C4, (int)blockDim.x);
  const int nrow_par = blockDim.x / ncol;
  const int tr = threadIdx.x / ncol, tc = threadIdx.x - tr * ncol;
  // every block folds the channel sums of its image into the group statistics itself (fixed order, fp64)
  __shared__ float mean_rstd[GN_GROUPS * 2];
  extern __shared__ float2 s_aff[];     // [C]: y = x * .x + .y
  {
    const int g = threadIdx.x >> 3, l8 = threadIdx.x & 7;     // 8 threads per group
    double s = 0.0, q = 0.0;
    for (int j = l8; j < cpg; j += 8) {
      const int c = g * cpg + j;
      const double* o = (c < C1) ? st1 + ((long long)b * C1 + c) * 2 : st2 + ((long long)b * C2 + (c - C1)) * 2;
      s += o[0];
      q += o[1];
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
    if (l8 == 0) {
      const double mean = s * inv_count;
      double var = q * inv_count - mean * mean;
      if (var < 0.0) var = 0.0;
      mean_rstd[g * 2 + 0] = (float)mean;
      mean_rstd[g * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int g = c / cpg;
    const float mean = mean_rstd[g * 2 + 0], rstd = mean_rstd[g * 2 + 1];
    float a = rstd * gamma[c];
    float o = beta[c] - mean * a;
    if (scale) {      // gn(x) * (1 + scale) + shift   (improved-DDPM scale-shift norm)
      const float s1 = 1.f + scale[(long long)b * ld_ss + c];
      a *= s1;
      o = o * s1 + shift[(long long)b * ld_ss + c];
    }
    s_aff[c] = make_float2(a, o);
  }
  __syncthreads();
  if (ab_out && blockIdx.x == 0)
    for (int c = threadIdx.x; c < C; c += blockDim.x) ab_out[(long long)bo * C + c] = s_aff[c];
  float vmax = 0.f;
  if (tr < nrow_par) {
    for (int c4 = tc; c4 < C4; c4 += ncol) {
      const int c = c4 * 4;
      const float2 a0 = s_aff[c], a1 = s_aff[c + 1], a2 = s_aff[c + 2], a3 = s_aff[c + 3];
      const float* src = (c < C1) ? (x1 + (long long)b * HW * C1 + c) : (x2 + (long long)b * HW * C2 + (c - C1));
      const int ldx = (c < C1) ? C1 : C2;
      float* dst = y + (long long)bo * HW * C + c;
      auto act = [&](float4 v) {
        float t[4] = {fmaf(v.x, a0.x, a0.y), fmaf(v.y, a1.x, a1.y), fmaf(v.z, a2.x, a2.y), fmaf(v.w, a3.x, a3.y)};
        if (silu) {
#pragma unroll
          for (int j = 0; j < 4; ++j) t[j] = __fdividef(t[j], 1.f + __expf(-t[j]));
        }
        vmax = fmaxf(vmax, fmaxf(fmaxf(fabsf(t[0]), fabsf(t[1])), fmaxf(fabsf(t[2]), fabsf(t[3]))));
        return make_float4(t[0], t[1], t[2], t[3]);
      };
      int r = r0 + tr;
      for (; r + 3 * nrow_par < r1; r += 4 * nrow_par) {
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = *reinterpret_cast<const float4*>(src + (long long)(r + u * nrow_par) * ldx);
#pragma unroll
        for (int u = 0; u < 4; ++u) *reinterpret_cast<float4*>(dst + (long long)(r + u * nrow_par) * C) = act(v[u]);
      }
      for (; r < r1; r += nrow_par)
        *reinterpret_cast<float4*>(dst + (long long)r * C) = act(*reinterpret_cast<const float4*>(src + (long long)r * ldx));
    }
  }
  if (amax) block_amax(vmax, amax);
}

// one warp per row, the row held in registers (NV float4 per lane: C <= 128 NV): one read, one write.  Persistent warps walk the
// rows two at a time (both rows' loads in flight before either reduction).
template <int NV>
__global__ void __launch_bounds__(256) layernorm_kernel(const float* x, const float* gamma,
                                                        const float* beta, float* y, int M, int C,
                                                        float eps, float* amax) {
  tc::pdl_trigger();
  tc::pdl_wait();
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int C4 = C >> 2;
  float vmax = 0.f;
  float4 g[NV], bt[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c4 = lane + 32 * i;
    g[i] = c4 < C4 ? *reinterpret_cast<const float4*>(gamma + c4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    bt[i] = c4 < C4 ? *reinterpret_cast<const float4*>(beta + c4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int row0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 2; row0 < M; row0 += nwarps * 2) {
    float4 v[2][NV];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const bool ok = row0 + r < M;
      const float* xr = x + (long long)(row0 + r) * C;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c4 = lane + 32 * i;
        v[r][i] = (ok && c4 < C4) ? *reinterpret_cast<const float4*>(xr + c4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      if (row0 + r >= M) break;
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) s += (v[r][i].x + v[r][i].y) + (v[r][i].z + v[r][i].w);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const float mean = s / (float)C;
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        if (lane + 32 * i < C4) {
          const float a = v[r][i].x - mean, b = v[r][i].y - mean, c = v[r][i].z - mean, d = v[r][i].w - mean;
          q += (a * a + b * b) + (c * c + d * d);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      const float rstd = 1.f / sqrtf(q / (float)C + eps);
      float* yr = y + (long long)(row0 + r) * C;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c4 = lane + 32 * i;
        if (c4 < C4) {
          float4 o;
          o.x = (v[r][i].x - mean) * rstd * g[i].x + bt[i].x;
          o.y = (v[r][i].y - mean) * rstd * g[i].y + bt[i].y;
          o.z = (v[r][i].z - mean) * rstd * g[i].z + bt[i].z;
          o.w = (v[r][i].w - mean) * rstd * g[i].w + bt[i].w;
          vmax = fmaxf(vmax, fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w))));
          *reinterpret_cast<float4*>(yr + c4 * 4) = o;
        }
      }
    }
  }
  if (amax) block_amax(vmax, amax);
}

// in-place softmax over rows of length L (row stride ld); one warp per row, three passes (row stays in L1/L2)
__global__ void __launch_bounds__(256) softmax_kernel(float* __restrict__ x, long long rows, int L0, int ld, int causal_nq) {
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= rows) return;
  float* r = x + warp * ld;
  int L = L0;
  if (causal_nq > 0) {                       // causal mask (CLIP text tower): query i attends to keys 0..i, masked probabilities are 0
    L = min(L0, (int)(warp % causal_nq) + 1);
    for (int i = L + lane; i < L0; i += 32) r[i] = 0.f;
  }
  float mx = -INFINITY;
  for (int i = lane; i < L; i += 32) mx = fmaxf(mx, r[i]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float s = 0.f;
  for (int i = lane; i < L; i += 32) {
    const float ev = expf(r[i] - mx);
    r[i] = ev;
    s += ev;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float inv = 1.f / s;
  for (int i = lane; i < L; i += 32) r[i] = r[i] * inv;
}

}  // namespace

double* gn_channel_stats(Engine& e, const float* x, int C, int B, int HW, cudaStream_t s) {
  double* st = e.stat_alloc((size_t)B * C * 2);
  gn_channel_stats_into(e, x, C, B, HW, st, s);
  return st;
}

void gn_channel_stats_into(Engine& e, const float* x, int C, int B, int HW, double* st, cudaStream_t s) {
  CDX_CHECK(C % 4 == 0, "groupnorm stats: C=%d must be a multiple of 4", C);
  if (e.dry()) return;
  int nchunk = cdiv(4LL * e.num_sms, B);
  if (nchunk > HW) nchunk = HW;
  if (nchunk < 1) nchunk = 1;
  const int rows_per_chunk = cdiv(HW, nchunk);
  nchunk = cdiv(HW, rows_per_chunk);
  ProfScope ps(e, s, PROF_GROUPNORM, 0.0, 0.0, 1);      // (the algorithmic bytes are booked by the apply pass)
  gn_stats_kernel<<<dim3(nchunk, B), 256, 0, s>>>(x, C, HW, rows_per_chunk, st);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}

void groupnorm(Engine& e, const float* x1, int C1, const float* x2, int C2, const float* gamma, const float* beta, float eps,
               bool silu, const float* scale, const float* shift, int ld_ss, float* y, int B, int HW, cudaStream_t s,
               const double* st1, const double* st2, float* amax, float2* ab_out, const int* src_img) {
  const int C = C1 + C2;
  CDX_CHECK(C % GN_GROUPS == 0, "groupnorm: C=%d not divisible by 32", C);
  CDX_CHECK(C1 % 4 == 0 && C2 % 4 == 0, "groupnorm: channel counts must be multiples of 4 (C1=%d C2=%d)", C1, C2);
  if (!st1) st1 = gn_channel_stats(e, x1, C1, B, HW, s);
  if (x2 && !st2) st2 = gn_channel_stats(e, x2, C2, B, HW, s);
  if (e.dry()) return;
  ProfScope ps(e, s, PROF_GROUPNORM, 0.0, 2.0 * 4.0 * B * (double)HW * C, 1);   // algorithmic: one read + one write
  int achunk = cdiv(4LL * e.num_sms, B);      // ~4 blocks per SM in total: the per-block prologue (group statistics, affine table) is amortised
  if (achunk > HW / 8) achunk = std::max(1, HW / 8);
  const int arows = cdiv(HW, achunk);
  achunk = cdiv(HW, arows);
  tc::launch_ex(gn_apply_kernel, dim3((unsigned)achunk, (unsigned)B), dim3(256), (size_t)C * sizeof(float2), s, 1, x1, C1, x2, C2, gamma, beta, st1, st2,
                1.0 / ((double)HW * (C / GN_GROUPS)), eps, silu ? 1 : 0, scale, shift, ld_ss, y, HW, arows, amax, ab_out, src_img);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}

void layernorm(Engine& e, const float* x, const float* gamma, const float* beta, float* y, int M, int C, cudaStream_t s, float* amax) {
  CDX_CHECK(C % 4 == 0 && C <= 128 * 16, "layernorm: C=%d must be a multiple of 4 and <= 2048", C);
  if (e.dry()) return;
  ProfScope ps(e, s, PROF_LAYERNORM, 0.0, 2.0 * 4.0 * (double)M * C, 1);
  const int nv = cdiv(C, 128);
  const int blocks = (int)std::min<long long>(cdiv((long long)cdiv(M, 2) * 32, 256), (long long)e.num_sms * 8);
  if (nv <= 3) tc::launch_ex(layernorm_kernel<3>, dim3((unsigned)blocks), dim3(256), 0, s, 1, x, gamma, beta, y, M, C, 1e-5f, amax);
  else if (nv <= 6) tc::launch_ex(layernorm_kernel<6>, dim3((unsigned)blocks), dim3(256), 0, s, 1, x, gamma, beta, y, M, C, 1e-5f, amax);
  else if (nv <= 10) tc::launch_ex(layernorm_kernel<10>, dim3((unsigned)blocks), dim3(256), 0, s, 1, x, gamma, beta, y, M, C, 1e-5f, amax);
  else tc::launch_ex(layernorm_kernel<16>, dim3((unsigned)blocks), dim3(256), 0, s, 1, x, gamma, beta, y, M, C, 1e-5f, amax);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}

void softmax_rows(Engine& e, float* x, long long rows, int L, int ld, cudaStream_t s, int causal_nq) {
  if (e.dry()) return;
  ProfScope ps(e, s, PROF_SOFTMAX, 0.0, 2.0 * 4.0 * (double)rows * L, 1);
  softmax_kernel<<<cdiv(rows * 32, 256), 256, 0, s>>>(x, rows, L, ld, causal_nq);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}

}  // namespace cdx
