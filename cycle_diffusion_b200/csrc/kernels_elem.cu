// kernels_elem.cu -- elementwise / layout kernels and the fused per-step scheduler kernels.
//
// Scheduler kernels restate, op for op and with round-to-nearest intrinsics (no FMA contraction), the reference's
// per-step tensor arithmetic so that they are bit-exact against the reference CPU path:
//   ddim_posterior_sample   DDIMSampler.sample_xt_next          ddim.py:582-601
//   ddim_compute_eps        CFG combine + compute_eps tail      ddim.py:555-559, 575-579
//   ddim_step_with_eps      CFG combine + p_sample_ddim_with_eps tail   ddim.py:613-617, 634-645
//   pixel_*                 sample_xt_next / compute_eps / denoising_step_with_eps   ddpm_ddim_wrapper.py:114-307
//   vae_posterior           DiagonalGaussianDistribution.sample * scale_factor      distributions.py:24-37, ddpm.py:536-543
// Each is one launch instead of the reference's ~8-10 elementwise launches per step (SURVEY.md 2.2).
#include "common.cuh"

namespace cdx {
namespace {

#define MUL(a, b) __fmul_rn((a), (b))
#define ADD(a, b) __fadd_rn((a), (b))
#define SUB(a, b) __fsub_rn((a), (b))
#define DIV(a, b) __fdiv_rn((a), (b))

inline int grid_for(size_t n, int num_sms) {
  size_t b = (n + 255) / 256;
  size_t cap = (size_t)num_sms * 16;
  return (int)(b < cap ? (b ? b : 1) : cap);
}
#define GRID_STRIDE(i, n) for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += (size_t)gridDim.x * blockDim.x)

__global__ void affine_kernel(const float* __restrict__ x, float a, float b, float* __restrict__ y, size_t n) {
  GRID_STRIDE(i, n) y[i] = ADD(MUL(a, x[i]), b);
}
__global__ void shift_scale_kernel(const float* __restrict__ x, float b, float a, float* __restrict__ y, size_t n) {
  GRID_STRIDE(i, n) y[i] = MUL(ADD(x[i], b), a);
}
__global__ void q_sample_kernel(const float* __restrict__ x0, const float* __restrict__ nz, float sa, float s1, float* __restrict__ y, size_t n) {
  GRID_STRIDE(i, n) y[i] = ADD(MUL(sa, x0[i]), MUL(s1, nz[i]));
}
__global__ void silu_kernel(const float* __restrict__ x, float* __restrict__ y, size_t n) {
  GRID_STRIDE(i, n) { const float v = x[i]; y[i] = v / (1.f + expf(-v)); }
}
__global__ void add_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ y, size_t n) {
  GRID_STRIDE(i, n) y[i] = a[i] + b[i];
}
__global__ void copy_kernel(const float* __restrict__ a, float* __restrict__ y, size_t n) {
  GRID_STRIDE(i, n) y[i] = a[i];
}
// x [M,2C] -> y [M,C] = x[:, :C] * gelu_erf(x[:, C:])   (attention.py:42-44)
__global__ void geglu_kernel(const float* __restrict__ x, float* __restrict__ y, size_t M, int C, int interleaved) {
  const size_t n = M * (size_t)C;
  GRID_STRIDE(i, n) {
    const size_t m = i / C;
    const int c = (int)(i - m * C);
    const int cv = interleaved ? ((c >> 5) << 6) + (c & 31) : c;      // [32 value | 32 gate] blocks (see Param::geglu)
    const int cg = interleaved ? cv + 32 : C + c;
    const float v = x[m * 2 * C + cv];
    const float g = x[m * 2 * C + cg];
    y[i] = v * (0.5f * g * (1.f + erff(g * 0.70710678118654752440f)));
  }
}
// rows [0, rows/2) are value rows, [rows/2, rows) gate rows -> blocks of 32 value rows followed by their 32 gate rows
__global__ void interleave_geglu_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, int rows, int rowlen) {
  const size_t n = (size_t)rows * rowlen;
  const int half = rows / 2;
  GRID_STRIDE(i, n) {
    const int r = (int)(i / rowlen);
    const int c = (int)(i - (size_t)r * rowlen);
    const int j = r < half ? r : r - half;
    const int dr = ((j >> 5) << 6) + (j & 31) + (r < half ? 0 : 32);
    dst[(size_t)dr * rowlen + c] = src[i];
  }
}
__global__ void avgpool2_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int C) {
  const int Ho = H / 2, Wo = W / 2;
  const size_t n = (size_t)B * Ho * Wo * C;
  GRID_STRIDE(i, n) {
    const int c = (int)(i % C);
    size_t r = i / C;
    const int ox = (int)(r % Wo); r /= Wo;
    const int oy = (int)(r % Ho);
    const int b = (int)(r / Ho);
    const float* p = x + (((size_t)b * H + 2 * oy) * W + 2 * ox) * C + c;
    // ATen avg_pool2d sums the window then divides
    y[i] = (p[0] + p[C] + p[(size_t)W * C] + p[(size_t)W * C + C]) * 0.25f;
  }
}
__global__ void upsample2_kernel(const float* __restrict__ x, float* __restrict__ y, int B, int H, int W, int C) {
  const int Ho = H * 2, Wo = W * 2;
  const size_t n = (size_t)B * Ho * Wo * C;
  GRID_STRIDE(i, n) {
    const int c = (int)(i % C);
    size_t r = i / C;
    const int ox = (int)(r % Wo); r /= Wo;
    const int oy = (int)(r % Ho);
    const int b = (int)(r / Ho);
    y[i] = x[(((size_t)b * H + (oy >> 1)) * W + (ox >> 1)) * C + c];
  }
}
// tiled transposes between [B,C,HW] and [B,HW,C]
__global__ void transpose_kernel(const float* __restrict__ x, float* __restrict__ y, int R, int Cc) {
  // x: [b][R][Cc] -> y: [b][Cc][R]
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const float* xb = x + (size_t)b * R * Cc;
  float* yb = y + (size_t)b * R * Cc;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int r = r0 + j, c = c0 + threadIdx.x;
    if (r < R && c < Cc) tile[j][threadIdx.x] = xb[(size_t)r * Cc + c];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (r < R && c < Cc) yb[(size_t)c * R + r] = tile[threadIdx.x][j];
  }
}
// [cos | sin] (util.py:152-172, nn.py:103-122) or, sin_first, [sin | cos] (ddpm/diffusion.py:6-25)
__global__ void temb_kernel(const float* __restrict__ t, const float* __restrict__ freqs, float* __restrict__ emb, int B, int half, int sin_first) {
  const int n = B * half;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int b = i / half, j = i - b * half;
    const float a = MUL(t[b], freqs[j]);
    emb[(size_t)b * 2 * half + (sin_first ? half : 0) + j] = cosf(a);
    emb[(size_t)b * 2 * half + (sin_first ? 0 : half) + j] = sinf(a);
  }
}
// OIHW (3x3) -> O,kh,kw,I
// OIHW -> O,kh,kw,Ip with the input channels zero-padded from I to Ip (Ip == I: plain repack)
__global__ void repack_conv_kernel(const float* __restrict__ w, float* __restrict__ o, int O, int I, int Ip) {
  const size_t n = (size_t)O * Ip * 9;
  GRID_STRIDE(idx, n) {
    const int i = (int)(idx % Ip);
    size_t r = idx / Ip;
    const int tap = (int)(r % 9);
    const int oc = (int)(r / 9);
    o[idx] = i < I ? w[((size_t)oc * I + i) * 9 + tap] : 0.f;
  }
}
// CLIPTextEmbeddings: out[b, l, :] = token_embedding[ids[b, l]] + position_embedding[l]
__global__ void embed_tokens_kernel(const int* __restrict__ ids, const float* __restrict__ tok, const float* __restrict__ pos,
                                    float* __restrict__ out, int B, int L, int W, int vocab) {
  const size_t n = (size_t)B * L * W;
  GRID_STRIDE(idx, n) {
    const int c = (int)(idx % W);
    const size_t bl = idx / W;
    const int l = (int)(bl % L);
    int id = ids[bl];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    out[idx] = tok[(size_t)id * W + c] + pos[(size_t)l * W + c];
  }
}
// quick-GELU (HF activations.QuickGELUActivation): x * sigmoid(1.702 x)
__global__ void quick_gelu_kernel(const float* __restrict__ x, float* __restrict__ y, size_t n) {
  GRID_STRIDE(i, n) {
    const float v = x[i];
    y[i] = v * (1.f / (1.f + expf(-1.702f * v)));
  }
}
// exact (erf) GELU, nn.GELU() default
__global__ void gelu_kernel(const float* __restrict__ x, float* __restrict__ y, size_t n) {
  GRID_STRIDE(i, n) {
    const float v = x[i];
    y[i] = 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
  }
}
// x [rows][C] -> y [rows][Cp], zero fill
__global__ void pad_channels_kernel(const float* __restrict__ x, float* __restrict__ y, size_t rows, int C, int Cp) {
  const size_t n = rows * (size_t)Cp;
  GRID_STRIDE(idx, n) {
    const int c = (int)(idx % Cp);
    const size_t r = idx / Cp;
    y[idx] = c < C ? x[r * C + c] : 0.f;
  }
}

__global__ void vae_posterior_kernel(const float* __restrict__ mom, const float* __restrict__ nz, float sf, float* __restrict__ out,
                                     int B, int C, int hw) {
  const size_t n = (size_t)B * C * hw;
  GRID_STRIDE(i, n) {
    const size_t b = i / ((size_t)C * hw);
    const size_t r = i - b * (size_t)C * hw;
    const float mean = mom[b * 2 * C * hw + r];
    float z = mean;
    if (nz) {
      float lv = mom[b * 2 * C * hw + (size_t)C * hw + r];
      lv = fminf(fmaxf(lv, -30.0f), 20.0f);
      const float sd = expf(MUL(0.5f, lv));
      z = ADD(mean, MUL(sd, nz[i]));
    }
    out[i] = MUL(sf, z);
  }
}

__device__ __forceinline__ float cfg_combine(const float* e_c, const float* e_uc, float scale, size_t i) {
  const float ec = e_c[i];
  if (e_uc == nullptr) return ec;
  const float eu = e_uc[i];
  return ADD(eu, MUL(scale, SUB(ec, eu)));      // e_t_uncond + s * (e_t - e_t_uncond), ddim.py:559
}

__global__ void ddim_posterior_kernel(const float* __restrict__ x0, const float* __restrict__ xt, const float* __restrict__ nz,
                                      cdx_ddim_coef c, float* __restrict__ out, size_t n) {
  GRID_STRIDE(i, n) {
    const float e_t = DIV(SUB(xt[i], MUL(c.sqrt_at, x0[i])), c.sqrt_1m_at);       // ddim.py:597
    const float dir = MUL(c.dir_coef, e_t);                                       // :598
    const float noise = MUL(c.sigma, nz[i]);                                      // :599
    out[i] = ADD(ADD(MUL(c.sqrt_aprev, x0[i]), dir), noise);                      // :600
  }
}
__global__ void ddim_compute_eps_kernel(const float* __restrict__ xt, const float* __restrict__ xn, const float* __restrict__ e_c,
                                        const float* __restrict__ e_uc, float scale, cdx_ddim_coef c, float* __restrict__ out, size_t n) {
  GRID_STRIDE(i, n) {
    const float e_t = cfg_combine(e_c, e_uc, scale, i);
    const float pred_x0 = DIV(SUB(xt[i], MUL(c.sqrt_1m_at_tab, e_t)), c.sqrt_at);          // ddim.py:576
    const float dir = MUL(c.dir_coef, e_t);                                                // :578
    out[i] = DIV(DIV(SUB(SUB(xn[i], MUL(c.sqrt_aprev, pred_x0)), dir), c.sigma), 1.0f);    // :579 (temperature 1)
  }
}
__global__ void ddim_step_kernel(const float* __restrict__ x, const float* __restrict__ e_c, const float* __restrict__ e_uc, float scale,
                                 const float* __restrict__ eps, cdx_ddim_coef c, float* __restrict__ out, size_t n) {
  GRID_STRIDE(i, n) {
    const float e_t = cfg_combine(e_c, e_uc, scale, i);
    const float pred_x0 = DIV(SUB(x[i], MUL(c.sqrt_1m_at_tab, e_t)), c.sqrt_at);           // ddim.py:634
    const float dir = MUL(c.dir_coef, e_t);                                                // :638
    const float noise = MUL(MUL(c.sigma, eps[i]), 1.0f);                                   // :642
    out[i] = ADD(ADD(MUL(c.sqrt_aprev, pred_x0), dir), noise);                             // :645
  }
}

__device__ __forceinline__ float ddim_posterior_f(float x0, float xt, float nz, const cdx_ddim_coef& c) {
  const float e_t = DIV(SUB(xt, MUL(c.sqrt_at, x0)), c.sqrt_1m_at);       // ddim.py:597
  const float dir = MUL(c.dir_coef, e_t);                                 // :598
  const float noise = MUL(c.sigma, nz);                                   // :599
  return ADD(ADD(MUL(c.sqrt_aprev, x0), dir), noise);                     // :600
}

// e_t and pred_x0 of one chain from the guidance-combined U-Net output `o` at x_t = `x`: eps-prediction as ddim.py:576 / :634;
// v-prediction (SD 2 LatentDiffusion.predict_eps_from_z_and_v / predict_start_from_z_and_v), each product rounded before the add
template <int PRED>
__device__ __forceinline__ void eps_x0(float o, float x, const cdx_ddim_coef& c, float vsa, float vs1, float& e_t, float& pred_x0) {
  if constexpr (PRED == 0) {
    e_t = o;
    pred_x0 = DIV(SUB(x, MUL(c.sqrt_1m_at_tab, e_t)), c.sqrt_at);
  } else {
    e_t = ADD(MUL(vsa, o), MUL(vs1, x));
    pred_x0 = SUB(MUL(vsa, x), MUL(vs1, o));
  }
}

// eps-hat of one chain from its own U-Net rows.  A chain on one row takes that row's output unchanged; a chain on two rows at scale
// 1 or 0 takes its cond or uncond row unchanged (the reference's single-forward value bit for bit), else ddim.py:559.
__device__ __forceinline__ float chain_eps_hat(const float* eout, const Chain& ch, size_t r, int chw) {
  const float ec = __ldcg(eout + (size_t)ch.row * chw + r);
  if (ch.row2 < 0 || ch.scale == 1.0f) return ec;
  const float eu = __ldcg(eout + (size_t)ch.row2 * chw + r);
  if (ch.scale == 0.0f) return eu;
  return ADD(eu, MUL(ch.scale, SUB(ec, eu)));                  // ddim.py:559
}
__device__ __forceinline__ void chain_put(float* xin, const Chain& ch, size_t r, int chw, float v) {
  xin[(size_t)ch.row * chw + r] = v;
  if (ch.row2 >= 0) xin[(size_t)ch.row2 * chw + r] = v;
}
// x_T of every element group, shared by its source chain and its K target chains, and the first U-Net input: drawn from x0
// (ddim.py:477-479) when the loop has a source chain, else slot 0 of the recovered noises (SDW:153).  Every input was written by the
// copies and launches just before, so all loads take the coherent path.  DRAWS (solver 1 and 2): the first next x is next == 3's
// independent draw instead of next == 1's posterior sample.
template <int DRAWS = 0>
__global__ void latent_chains_init_kernel(const LatentChains a) {
  GRID_STRIDE(i, a.n) {
    const size_t j = i / a.chw, r = i - j * a.chw;
    float xT;
    if (a.src) {
      const float x0 = __ldcg(a.x0 + i);
      xT = ADD(MUL(a.sa, x0), MUL(a.s1, __ldcg(a.noise0 + i)));                                // ddim.py:477-479
      if (a.z_out) a.z_out[j * a.z_stride + r] = xT;
      a.xt[i] = xT;
      if constexpr (DRAWS) {
        if (a.next == 3) a.xn[i] = ADD(MUL(a.qa, x0), MUL(a.q1, __ldcg(a.noise_next + i)));
        else if (a.next == 2) a.xn[i] = x0;
      } else {
        if (a.next == 1) a.xn[i] = ddim_posterior_f(x0, xT, __ldcg(a.noise_next + i), a.cnext);
        else if (a.next == 2) a.xn[i] = x0;
      }
      chain_put(a.xin, a.chains[j], r, a.chw, xT);
    } else {
      xT = __ldcg(a.eps_in + j * a.eps_stride + r);
    }
    for (int k = 0; k < a.K; ++k) {
      const size_t t = j * a.K + k;
      a.yt[t * a.chw + r] = xT;
      chain_put(a.xin, a.chains[a.n_src + t], r, a.chw, xT);
      for (int q = 0; q < a.sg_m; ++q) a.xin[(size_t)a.sg_rows[t * a.sg_m + q] * a.chw + r] = xT;      // SEGA concept rows
    }
  }
}
// LEDITS++'s implicit masks.  The 3x3 smoothing of a raw attention map m (gh x gw, gh, gw >= 2) with reflect padding of 1 (index -1
// -> 1, n -> n - 2), as diffusers' GaussianSmoothing(kernel_size=3, sigma=0.5): weights w_ab = fp32(g_a g_b / (sum g)^2), g = (e^-1,
// 1, e^-1) formed in double (corner, edge, centre below); the nine products in row-major order, each rounded, added left to right.
// The threshold stage and the step kernel both call it, so the mask the step applies is the one the stage thresholded.
constexpr float LEDITS_W_CORNER = 0x1.6ffa7p-5f, LEDITS_W_EDGE = 0x1.f42264p-4f, LEDITS_W_CENTRE = 0x1.53e064p-2f;
__device__ __forceinline__ int ledits_reflect(int i, int n) { return i < 0 ? 1 : i >= n ? n - 2 : i; }
__device__ __forceinline__ float ledits_smooth(const float* m, int gh, int gw, int y, int x) {
  float s = 0.f;
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int b = 0; b < 3; ++b) {
      const float w = (a == 1 && b == 1) ? LEDITS_W_CENTRE : (a == 1 || b == 1) ? LEDITS_W_EDGE : LEDITS_W_CORNER;
      const float pr = MUL(w, __ldcg(m + (size_t)ledits_reflect(y + a - 1, gh) * gw + ledits_reflect(x + b - 1, gw)));
      s = (a || b) ? ADD(s, pr) : pr;
    }
  return s;
}
// sum over channels c = 0, 1, ... of |sc * (o_k - o_uc)| at latent pixel p (ok, ou: the rows' [C, hw] planes), one rounded op each
__device__ __forceinline__ float ledits_chansum(const float* ok, const float* ou, int C, int hw, int p, float sc) {
  float s = 0.f;
  for (int c = 0; c < C; ++c) {
    const float v = fabsf(MUL(sc, SUB(__ldcg(ok + (size_t)c * hw + p), __ldcg(ou + (size_t)c * hw + p))));
    s = c ? ADD(s, v) : v;
  }
  return s;
}

// One step of the loop: the source half once per source chain, the target half once per target chain with the recovered noise held
// in a register.  Under v-prediction each target chain forms e_t and pred_x0 from its own x_t and v.  MASK (the driver guarantees a
// source chain at every step): each target x_{t-1} is blended with the source's x_{t-1}, a posterior sample of q(x_{t-1} | x_t, x0)
// of the real image at the same noise level (x0 itself on the last step), so the unmasked region stays on the image's trajectory.
// SEGA (a.sg_m > 0): each target chain's guidance-combined output takes its semantic guidance term G (LatentChains), formed from its
// concept rows, its uncond row, the step's thresholds and its momentum before the e_t / pred_x0 conversion; its concept rows are
// written with its next x_t.  SEGA = 1 + a.sg_mask: 1 SEGA's per-channel thresholds, 2 LEDITS++'s
// attention mask, 3 the attention mask and the channel-summed one.
// SOLVER (LatentChains::solver): 0 the DDIM step on the posterior chain, 1 the DDIM step on independent draws (next == 3 in place of
// next == 1), 2 the SDE-DPM-Solver++ step on independent draws.
// the SDE-DPM-Solver++ mean of one chain at x with x0-prediction D; hist holds the chain's previous D and takes this one
__device__ __forceinline__ float dpm_mean(const LatentChains& a, float x, float D, float* hist) {
  float mu = ADD(MUL(a.dc.a, x), MUL(a.dc.b, D));
  if (a.dc.order == 2) mu = ADD(mu, MUL(a.dc.c, SUB(D, __ldcg(hist))));
  *hist = D;                                                     // each element's history has one owner thread
  return mu;
}
template <int PRED, int MASK, int SEGA = 0, int SOLVER = 0>
__global__ void latent_chains_step_kernel(const LatentChains a) {
  GRID_STRIDE(i, a.n) {
    const size_t j = i / a.chw, r = i - j * a.chw;
    float eps, xn = 0.f;
    if (a.src) {
      const Chain src = a.chains[j];
      const float o = chain_eps_hat(a.eout, src, r, a.chw);
      const float xt = __ldcg(a.xt + i);
      xn = __ldcg(a.xn + i);
      float e_t, pred_x0;
      eps_x0<PRED>(o, xt, a.c, a.vsa, a.vs1, e_t, pred_x0);                                     // ddim.py:576
      if constexpr (SOLVER == 2) {
        eps = DIV(SUB(xn, dpm_mean(a, xt, pred_x0, a.d_src + i)), a.dc.n);
      } else {
        const float dir = MUL(a.c.dir_coef, e_t);                                                // :578
        eps = DIV(DIV(SUB(SUB(xn, MUL(a.c.sqrt_aprev, pred_x0)), dir), a.c.sigma), 1.0f);       // :579 (temperature 1)
      }
      if (a.z_out) a.z_out[j * a.z_stride + r] = eps;
      if constexpr (SOLVER) {
        if (a.next == 3) a.xn2[i] = ADD(MUL(a.qa, __ldcg(a.x0 + i)), MUL(a.q1, __ldcg(a.noise_next + i)));
        else if (a.next == 2) a.xn2[i] = __ldcg(a.x0 + i);
      } else {
        if (a.next == 1) a.xn2[i] = ddim_posterior_f(__ldcg(a.x0 + i), xn, __ldcg(a.noise_next + i), a.cnext);
        else if (a.next == 2) a.xn2[i] = __ldcg(a.x0 + i);                                      // ddim.py:583-584
      }
      chain_put(a.xin, src, r, a.chw, xn);
    } else {
      eps = __ldcg(a.eps_in + j * a.eps_stride + r);
    }
    float m = 1.f;
    if constexpr (MASK) m = __ldcg(a.mask + j * a.hw + (int)r % a.hw);
    for (int k = 0; k < a.K; ++k) {
      const size_t t = j * a.K + k, ti = t * a.chw + r;
      const Chain tc = a.chains[a.n_src + t];
      float ot = chain_eps_hat(a.eout, tc, r, a.chw);
      if constexpr (SEGA) {
        const float ou = __ldcg(a.eout + (size_t)(tc.row2 >= 0 ? tc.row2 : tc.row) * a.chw + r);
        const int C = a.chw / a.hw, ch = (int)r / a.hw;
        float S = 0.f;
        for (int q = 0; q < a.sg_m; ++q) {
          const int tq = (int)t * a.sg_m + q;
          const float psi = MUL(a.sg_scale[q], SUB(__ldcg(a.eout + (size_t)a.sg_rows[tq] * a.chw + r), ou));
          float g;
          if constexpr (SEGA == 1) {
            g = ((a.sg_active >> q) & 1u) && fabsf(psi) >= __ldcg(a.sg_thr + (size_t)tq * C + ch) ? psi : 0.f;
          } else {               // LEDITS++: the concept's attention mask, and with SEGA == 3 its channel-summed mask
            bool keep = (a.sg_active >> q) & 1u;
            if (keep) {
              const int px = (int)r % a.hw, y = px / a.w, x = px - y * a.w;
              keep = ledits_smooth(a.sg_map + (size_t)tq * a.sg_gh * a.sg_gw, a.sg_gh, a.sg_gw, y / 4, x / 4) >= __ldcg(a.sg_thr + (size_t)tq * 2);
              if constexpr (SEGA == 3)
                keep = keep && ledits_chansum(a.eout + (size_t)a.sg_rows[tq] * a.chw, a.eout + (size_t)(tc.row2 >= 0 ? tc.row2 : tc.row) * a.chw, C,
                                              a.hw, px, a.sg_scale[q]) >= __ldcg(a.sg_thr + (size_t)tq * 2 + 1);
            }
            g = keep ? psi : 0.f;
          }
          S = q ? ADD(S, g) : g;
        }
        const float nu = __ldcg(a.sg_nu + ti);
        const float G = ADD(S, MUL(a.sg_mu, nu));
        a.sg_nu[ti] = ADD(MUL(a.sg_beta, nu), MUL(a.sg_beta1, G));
        if (a.sg_apply) ot = ADD(ot, G);
      }
      const float y = __ldcg(a.yt + ti);
      float et, px0;
      eps_x0<PRED>(ot, y, a.c, a.vsa, a.vs1, et, px0);                                          // ddim.py:634
      float yn;
      if constexpr (SOLVER == 2) {
        yn = ADD(dpm_mean(a, y, px0, a.d_tgt + ti), MUL(a.dc.n, eps));
      } else {
        const float tdir = MUL(a.c.dir_coef, et);                                               // :638
        const float noise = MUL(MUL(a.c.sigma, eps), 1.0f);                                     // :642
        yn = ADD(ADD(MUL(a.c.sqrt_aprev, px0), tdir), noise);                                   // :645
      }
      if constexpr (MASK) {
        if (m == 0.0f) yn = xn;
        else if (m != 1.0f) yn = ADD(xn, MUL(m, SUB(yn, xn)));
      }
      a.y_out[ti] = yn;
      chain_put(a.xin, tc, r, a.chw, yn);
      if constexpr (SEGA)
        for (int q = 0; q < a.sg_m; ++q) a.xin[(size_t)a.sg_rows[t * a.sg_m + q] * a.chw + r] = yn;
    }
  }
}

// SEGA's threshold stage (semantic_thresholds): block b owns plane b = (t*sg_m + k)*C + c, the hw values a = |psi_k| of target chain
// t, concept k, channel c.  Non-negative floats order as their bit patterns, so the rank-th smallest value is found by a radix select
// of 8 bits per pass: each pass histograms the values that match the digits found so far and keeps the digit whose bin holds the
// rank.  The values are recomputed from eout on every pass, so any plane size runs with a 1 KB histogram.  After the last pass the
// bin is one value, v_lo, and the rank's place among its copies says whether v_hi (rank + 1) is v_lo too; else one more pass takes
// the smallest value above v_lo.
constexpr int SEMANTIC_THREADS = 512;
__device__ __forceinline__ unsigned semantic_abs_bits(const float* ok, const float* ou, int p, float sc) {
  return __float_as_uint(fabsf(MUL(sc, SUB(__ldcg(ok + p), __ldcg(ou + p)))));
}
// *out <- Q(lambda, the n values val(p)) by the radix select and the lerp above (thread 0 writes).  val returns the bit pattern of a
// non-negative float
template <class Val>
__device__ __forceinline__ void semantic_select(const Val& val, int n, float lambda, float* out, unsigned* hist, unsigned& s_digit,
                                                unsigned& s_below, unsigned& s_count, unsigned& s_min) {
  const float rk = MUL(lambda, (float)(n - 1));
  const float fl = floorf(rk);
  const unsigned lo = (unsigned)fl, hi = (unsigned)ceilf(rk);
  const float w = SUB(rk, fl);
  unsigned prefix = 0, known = 0, want = lo, count = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += SEMANTIC_THREADS) hist[i] = 0;
    __syncthreads();
    for (int p = threadIdx.x; p < n; p += SEMANTIC_THREADS) {
      const unsigned u = val(p);
      if ((u & known) == prefix) atomicAdd(&hist[(u >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 32) {          // warp 0: lane l sums bins [8l, 8l + 8), an exclusive scan finds the lane holding `want`
      const int lane = threadIdx.x;
      unsigned cnt[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) { cnt[j] = hist[lane * 8 + j]; sum += cnt[j]; }
      unsigned incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      unsigned run = incl - sum;
      if (want >= run && want < incl) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (want < run + cnt[j]) { s_digit = lane * 8 + j; s_below = run; s_count = cnt[j]; break; }
          run += cnt[j];
        }
      }
    }
    __syncthreads();
    prefix |= s_digit << shift;
    known |= 255u << shift;
    want -= s_below;
    count = s_count;
  }
  // prefix = v_lo; `want` is the rank among its `count` copies
  const bool above = hi != lo && want + 1 >= count;
  if (above) {
    if (threadIdx.x == 0) s_min = 0xffffffffu;
    __syncthreads();
    unsigned m = 0xffffffffu;
    for (int p = threadIdx.x; p < n; p += SEMANTIC_THREADS) {
      const unsigned u = val(p);
      if (u > prefix) m = min(m, u);
    }
    atomicMin(&s_min, m);
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float vlo = __uint_as_float(prefix), vhi = above ? __uint_as_float(s_min) : vlo;
    *out = w < 0.5f ? ADD(vlo, MUL(w, SUB(vhi, vlo))) : SUB(vhi, MUL(SUB(vhi, vlo), SUB(1.0f, w)));   // ATen lerp
  }
}
// MASKM (LatentChains::sg_mask) 0: SEGA's planes.  1, 2: block b owns concept row tq = b / P (P = MASKM planes per row), plane kind
// b % P: 0 the smoothed attention map (threshold at sg_thr[tq*2]), 1 the channel sum of |psi_k| (at sg_thr[tq*2 + 1])
template <int MASKM>
__global__ void __launch_bounds__(SEMANTIC_THREADS) semantic_threshold_kernel(const LatentChains a) {
  __shared__ unsigned hist[256];
  __shared__ unsigned s_digit, s_below, s_count, s_min;
  const int C = a.chw / a.hw;
  if constexpr (MASKM == 0) {
    const int n = a.hw, plane = blockIdx.x;
    const int c = plane % C, tq = plane / C, q = tq % a.sg_m, t = tq / a.sg_m;
    const Chain tc = a.chains[a.n_src + t];
    const float* ou = a.eout + (size_t)(tc.row2 >= 0 ? tc.row2 : tc.row) * a.chw + (size_t)c * n;
    const float* ok = a.eout + (size_t)a.sg_rows[tq] * a.chw + (size_t)c * n;
    const float sc = a.sg_scale[q];
    semantic_select([&](int p) { return semantic_abs_bits(ok, ou, p, sc); }, n, a.sg_lambda[q], a.sg_thr + plane, hist, s_digit, s_below,
                    s_count, s_min);
  } else {
    const int tq = blockIdx.x / MASKM, kind = blockIdx.x % MASKM, q = tq % a.sg_m, t = tq / a.sg_m;
    float* out = a.sg_thr + (size_t)tq * 2 + kind;
    if (kind == 0) {
      const int gh = a.sg_gh, gw = a.sg_gw;
      const float* mp = a.sg_map + (size_t)tq * gh * gw;
      semantic_select([&](int p) { return __float_as_uint(ledits_smooth(mp, gh, gw, p / gw, p % gw)); }, gh * gw, a.sg_lambda[q], out, hist,
                      s_digit, s_below, s_count, s_min);
    } else {
      const Chain tc = a.chains[a.n_src + t];
      const float* ou = a.eout + (size_t)(tc.row2 >= 0 ? tc.row2 : tc.row) * a.chw;
      const float* ok = a.eout + (size_t)a.sg_rows[tq] * a.chw;
      const float sc = a.sg_scale[q];
      semantic_select([&](int p) { return __float_as_uint(ledits_chansum(ok, ou, C, a.hw, p, sc)); }, a.hw, a.sg_lambda[q], out, hist, s_digit,
                      s_below, s_count, s_min);
    }
  }
}

// [B,1,H,W] -> [B,1,H/f,W/f]: the f x f block summed row by row, left to right, then divided by f*f (ATen's avg_pool2d order)
__global__ void mask_pool_kernel(const float* __restrict__ m, float* __restrict__ out, int B, int H, int W, int f) {
  const int Ho = H / f, Wo = W / f;
  const size_t n = (size_t)B * Ho * Wo;
  GRID_STRIDE(i, n) {
    const int ox = (int)(i % Wo);
    const size_t r = i / Wo;
    const int oy = (int)(r % Ho);
    const size_t b = r / Ho;
    const float* p = m + (b * H + (size_t)oy * f) * W + (size_t)ox * f;
    float sum = 0.f;
    for (int dy = 0; dy < f; ++dy)
      for (int dx = 0; dx < f; ++dx) sum = ADD(sum, p[(size_t)dy * W + dx]);
    out[i] = DIV(sum, (float)(f * f));
  }
}
// paste-back: out = m*clamp((dec + 1)*0.5, 0, 1) + (1 - m)*image over [B,C,H,W], m = mask[b, 0, y, x]; the decode is post-processed
// as shift_scale + clamp do it, so m == 1 gives exactly the unmasked output and m == 0 exactly the input image
__global__ void mask_composite_kernel(const float* __restrict__ dec, const float* __restrict__ img, const float* __restrict__ mask,
                                      float* __restrict__ out, int C, size_t hw, size_t n) {
  GRID_STRIDE(i, n) {
    const size_t p = i % hw, b = i / hw / C;
    const float m = mask[b * hw + p], x = img[i];
    const float d = fminf(fmaxf(MUL(ADD(dec[i], 1.0f), 0.5f), 0.f), 1.f);
    out[i] = m == 0.0f ? x : (m == 1.0f ? d : ADD(MUL(m, d), MUL(SUB(1.0f, m), x)));
  }
}

// DiffEdit mask.  Pair q = k*B + b (map k of image b) of pairs [p0, p1): both of its U-Net rows get q_sample(x0[b], noise[b, k]) in
// q_sample_kernel's op order; a pair's rows are 2*(q - p0) (source condition) and 2*(q - p0) + 1 (target condition).
__global__ void edit_rows_kernel(const float* __restrict__ x0, const float* __restrict__ noise, float sa, float s1, float* __restrict__ xin,
                                 int B, int n_maps, int chw, int p0, size_t n) {
  GRID_STRIDE(i, n) {
    const int r = (int)(i / chw), q = p0 + r, b = q % B, k = q / B;
    const size_t c = i - (size_t)r * chw;
    const float v = ADD(MUL(sa, x0[(size_t)b * chw + c]), MUL(s1, noise[((size_t)b * n_maps + k) * chw + c]));
    xin[(size_t)2 * r * chw + c] = v;
    xin[(size_t)(2 * r + 1) * chw + c] = v;
  }
}
// acc[b, p] += sum_c |vscale * (tgt - src)| (c ascending, fp32) for every pair q = k*B + b of [p0, p1), k ascending: one thread per
// (image, latent pixel), so the adds into acc happen in map order however the maps are split over launches.  Pair q's predictions
// sit at src + off(q), tgt + off(q), off(q) = b*sb + k*sk - off0.  vscale = 1 (eps) leaves the difference unchanged exactly.
// Coherent loads: the predictions come from the U-Net launches just before, acc from the previous accumulate launch.
__global__ void edit_map_accum_kernel(const float* src, const float* tgt, long long sb, long long sk, long long off0, float vscale,
                                      float* acc, int B, int C, int hw, int p0, int p1) {
  const size_t n = (size_t)B * hw;
  GRID_STRIDE(i, n) {
    const int b = (int)(i / hw), p = (int)(i - (size_t)b * hw);
    int k = p0 > b ? (p0 - b + B - 1) / B : 0;
    if (k * B + b >= p1) continue;
    float a = __ldcg(acc + i);
    for (; k * B + b < p1; ++k) {
      const long long off = (long long)b * sb + (long long)k * sk - off0 + p;
      float s = 0.f;
      for (int c = 0; c < C; ++c) {
        const long long o = off + (long long)c * hw;
        s = ADD(s, fabsf(MUL(vscale, SUB(__ldcg(tgt + o), __ldcg(src + o)))));
      }
      a = ADD(a, s);
    }
    acc[i] = a;
  }
}
// One block of EDIT_MASK_THREADS per image: map = acc / (n*C); mean = fp32(sum_p map in fp64 / hw), summed in a fixed order (each
// thread strides the pixels, then a fixed tree over the block); M = ratio * mean; mask = min(map, M) / M > 0.5 when M > 0, else 0.
// Writes the map, the latent mask and, optionally, the mask nearest-upsampled by f.
constexpr int EDIT_MASK_THREADS = 256;
__global__ void __launch_bounds__(EDIT_MASK_THREADS) edit_mask_kernel(const float* acc, float div, float ratio, float* __restrict__ map_out,
                                                                      float* __restrict__ mask_out, float* __restrict__ img_out, int f, int h,
                                                                      int w) {
  __shared__ double part[EDIT_MASK_THREADS];
  __shared__ float thr;
  const int b = blockIdx.x, hw = h * w;
  const float* a = acc + (size_t)b * hw;
  double sum = 0.0;
  for (int p = threadIdx.x; p < hw; p += EDIT_MASK_THREADS) sum += (double)DIV(__ldcg(a + p), div);
  part[threadIdx.x] = sum;
  __syncthreads();
  for (int o = EDIT_MASK_THREADS / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) part[threadIdx.x] += part[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) thr = MUL(ratio, (float)(part[0] / (double)hw));
  __syncthreads();
  const float M = thr;
  for (int p = threadIdx.x; p < hw; p += EDIT_MASK_THREADS) {
    const float m = DIV(__ldcg(a + p), div);
    map_out[(size_t)b * hw + p] = m;
    mask_out[(size_t)b * hw + p] = (M > 0.f && DIV(fminf(m, M), M) > 0.5f) ? 1.f : 0.f;
  }
  if (!img_out) return;
  const int W = w * f;
  const size_t HW = (size_t)hw * f * f;
  for (size_t i = threadIdx.x; i < HW; i += EDIT_MASK_THREADS) {
    const int y = (int)(i / W), x = (int)(i - (size_t)y * W);
    const float m = DIV(__ldcg(a + (y / f) * w + x / f), div);
    img_out[(size_t)b * HW + i] = (M > 0.f && DIV(fminf(m, M), M) > 0.5f) ? 1.f : 0.f;
  }
}

// does candidate (sa, ia) beat (sb, ib) under torch.argmax?  larger wins, NaN beats any number, ties and NaN pairs go to the lower
// index; an index < 0 is an empty slot
__device__ __forceinline__ bool select_better(float sa, long long ia, float sb, long long ib) {
  if (ia < 0) return false;
  if (ib < 0) return true;
  const bool na = sa != sa, nb = sb != sb;
  if (na || nb) return na && (!nb || ia < ib);
  return sa > sb || (sa == sb && ia < ib);
}
// one block per sample: the chunk's best candidate of sample b (a block reduction under select_better, so the result does not depend
// on the order candidates arrive in), then the running best; the winner's image is copied only when it replaces the best
__global__ void ensemble_select_kernel(int n, const float* scores, const long long* cand, const int* sample, const float* images,
                                       float* best_score, long long* best_idx, float* best_img, float* score_mat, int n_total, size_t img_n) {
  __shared__ float ss[256];
  __shared__ long long si[256];
  __shared__ int sr[256];
  __shared__ int win;
  const int b = blockIdx.x, tid = threadIdx.x;
  float bs = 0.f;
  long long bi = -1;
  int br = -1;
  for (int c = tid; c < n; c += blockDim.x) {
    const long long ci = __ldcg(cand + c);
    if (__ldcg(sample + c) != b || ci < 0 || ci >= n_total) continue;
    const float v = __ldcg(scores + c);
    score_mat[(size_t)b * n_total + ci] = v;
    if (select_better(v, ci, bs, bi)) { bs = v; bi = ci; br = c; }
  }
  ss[tid] = bs; si[tid] = bi; sr[tid] = br;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if (tid < o && select_better(ss[tid + o], si[tid + o], ss[tid], si[tid])) { ss[tid] = ss[tid + o]; si[tid] = si[tid + o]; sr[tid] = sr[tid + o]; }
    __syncthreads();
  }
  if (tid == 0) {
    win = -1;
    if (select_better(ss[0], si[0], __ldcg(best_score + b), __ldcg(best_idx + b))) {
      best_score[b] = ss[0]; best_idx[b] = si[0]; win = sr[0];
    }
  }
  __syncthreads();
  if (win < 0) return;
  const float* src = images + (size_t)win * img_n;
  float* dst = best_img + (size_t)b * img_n;
  for (size_t p = tid; p < img_n; p += blockDim.x) dst[p] = __ldcg(src + p);
}

__global__ void pixel_posterior_kernel(const float* __restrict__ x0, const float* __restrict__ xt, const float* __restrict__ nz,
                                       cdx_pixel_coef c, float* __restrict__ out, size_t n) {
  GRID_STRIDE(i, n) {
    if (c.ddpm) {
      const float mean = ADD(MUL(c.w0, x0[i]), MUL(c.wt, xt[i]));                           // DW:293
      out[i] = ADD(mean, MUL(c.post_std, nz[i]));                                           // DW:297
    } else {
      const float et = DIV(SUB(xt[i], MUL(c.sqrt_at, x0[i])), c.sqrt_1m_at);                // DW:299
      out[i] = ADD(ADD(MUL(c.sqrt_at_next, x0[i]), MUL(c.c2, et)), MUL(c.c1, nz[i]));       // DW:302
    }
  }
}
__global__ void pixel_compute_eps_kernel(const float* __restrict__ xt, const float* __restrict__ xn, const float* __restrict__ et_,
                                         cdx_pixel_coef c, float* __restrict__ out, int B, int chw, int net_chw) {
  const size_t n = (size_t)B * chw;
  GRID_STRIDE(i, n) {
    const size_t b = i / chw;
    const float et = et_[b * net_chw + (i - b * chw)];
    if (c.ddpm) {
      const float mean = MUL(c.inv_sqrt_1m_bt, SUB(xt[i], MUL(c.weight, et)));             // DW:266
      out[i] = DIV(SUB(xn[i], mean), c.std_model);                                          // DW:268
    } else {
      const float x0_t = DIV(SUB(xt[i], MUL(et, c.sqrt_1m_at)), c.sqrt_at);                 // DW:271
      out[i] = DIV(SUB(SUB(xn[i], MUL(c.sqrt_at_next, x0_t)), MUL(c.c2, et)), c.c1);        // DW:275
    }
  }
}
__global__ void pixel_step_kernel(const float* __restrict__ xt, const float* __restrict__ et_, const float* __restrict__ eps,
                                  cdx_pixel_coef c, float* __restrict__ out, int B, int chw, int net_chw) {
  const size_t n = (size_t)B * chw;
  GRID_STRIDE(i, n) {
    const size_t b = i / chw;
    const float et = et_[b * net_chw + (i - b * chw)];
    const float nz = eps ? eps[i] : 0.f;
    if (c.ddpm) {
      const float mean = MUL(c.inv_sqrt_1m_bt, SUB(xt[i], MUL(c.weight, et)));             // DW:204
      out[i] = ADD(mean, MUL(MUL(c.mask, c.std_model), nz));                                // DW:208
    } else {
      const float x0_t = DIV(SUB(xt[i], MUL(et, c.sqrt_1m_at)), c.sqrt_at);                 // DW:213
      out[i] = ADD(ADD(MUL(c.sqrt_at_next, x0_t), MUL(c.c2, et)), MUL(c.c1, nz));           // DW:222
    }
  }
}
// One step of the two-model pixel loop: the three kernels above in one launch, same op order, x_{t-1} of the source chain and the
// recovered noise held in registers.  xs / ys (source x_t, target x_t) are advanced in place.  Every input but x0 and the noise
// slice was written by the launches just before this one, so all loads take the coherent path.
__global__ void pixel_lockstep_kernel(const float* x0, float* xs, float* ys, const float* es_, const float* et_, const float* nz,
                                      cdx_pixel_coef c, int B, int chw, int net_chw_s, int net_chw_t) {
  const size_t n = (size_t)B * chw;
  GRID_STRIDE(i, n) {
    const size_t b = i / chw, r = i - b * chw;
    const float x0v = __ldcg(x0 + i), xt = __ldcg(xs + i), yt = __ldcg(ys + i), z = __ldcg(nz + i);
    const float es = __ldcg(es_ + b * net_chw_s + r), et = __ldcg(et_ + b * net_chw_t + r);
    float yn, xn;
    if (c.ddpm) {
      xn = ADD(ADD(MUL(c.w0, x0v), MUL(c.wt, xt)), MUL(c.post_std, z));                     // DW:293, 297
      const float mean_s = MUL(c.inv_sqrt_1m_bt, SUB(xt, MUL(c.weight, es)));               // DW:266
      const float eps = DIV(SUB(xn, mean_s), c.std_model);                                  // DW:268
      const float mean_t = MUL(c.inv_sqrt_1m_bt, SUB(yt, MUL(c.weight, et)));               // DW:204
      yn = ADD(mean_t, MUL(MUL(c.mask, c.std_model), eps));                                 // DW:208
    } else {
      const float e_post = DIV(SUB(xt, MUL(c.sqrt_at, x0v)), c.sqrt_1m_at);                 // DW:299
      xn = ADD(ADD(MUL(c.sqrt_at_next, x0v), MUL(c.c2, e_post)), MUL(c.c1, z));            // DW:302
      const float x0_s = DIV(SUB(xt, MUL(es, c.sqrt_1m_at)), c.sqrt_at);                    // DW:271
      const float eps = DIV(SUB(SUB(xn, MUL(c.sqrt_at_next, x0_s)), MUL(c.c2, es)), c.c1);  // DW:275
      const float x0_t = DIV(SUB(yt, MUL(et, c.sqrt_1m_at)), c.sqrt_at);                    // DW:213
      yn = ADD(ADD(MUL(c.sqrt_at_next, x0_t), MUL(c.c2, et)), MUL(c.c1, eps));              // DW:222
    }
    xs[i] = xn;
    ys[i] = yn;
  }
}

}  // namespace

#define LAUNCH1(kernel, n, ...)                                   \
  do {                                                            \
    if (e.dry()) break;                                           \
    kernel<<<grid_for((n), e.num_sms), 256, 0, s>>>(__VA_ARGS__); \
    CDX_CUDA(cudaGetLastError());                                 \
    e.launches++;                                                 \
  } while (0)


// ------------------------------------------------------------------------------------------------ Directional-CLIP / metrics (8f-3)
// torch upsample_bicubic2d (aten/src/ATen/native/UpSample.h): A = -0.75, align_corners = False: src = (dst + 0.5) * scale - 0.5,
// 4 taps at floor(src) - 1 .. + 2 with clamped indices; weights from the cubic convolution polynomials.  Then (x - mean) / std.
__device__ __forceinline__ float cubic1(float x, float A) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; }
__device__ __forceinline__ float cubic2(float x, float A) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; }
__device__ __forceinline__ void cubic_coeffs(float t, float w[4]) {
  const float A = -0.75f;
  w[0] = cubic2(t + 1.f, A); w[1] = cubic1(t, A); w[2] = cubic1(1.f - t, A); w[3] = cubic2(2.f - t, A);
}
__global__ void clip_preprocess_kernel(const float* __restrict__ img, int B, int R, int size, float* __restrict__ out) {
  const float mean[3] = {0.48145466f, 0.4578275f, 0.40821073f}, sd[3] = {0.26862954f, 0.26130258f, 0.27577711f};   // clip.py _transform
  const float scale = (float)R / (float)size;
  const size_t n = (size_t)B * 3 * size * size;
  GRID_STRIDE(i, n) {
    const int x = (int)(i % size), y = (int)((i / size) % size), c = (int)((i / ((size_t)size * size)) % 3), b = (int)(i / ((size_t)3 * size * size));
    const float sy = ((float)y + 0.5f) * scale - 0.5f, sx = ((float)x + 0.5f) * scale - 0.5f;
    const float fy = floorf(sy), fx = floorf(sx);
    float wy[4], wx[4];
    cubic_coeffs(sy - fy, wy);
    cubic_coeffs(sx - fx, wx);
    const float* src = img + ((size_t)b * 3 + c) * R * R;
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int yy = min(max((int)fy - 1 + j, 0), R - 1);
      float row = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int xx = min(max((int)fx - 1 + k, 0), R - 1);
        row += src[(size_t)yy * R + xx] * wx[k];
      }
      acc += row * wy[j];
    }
    out[i] = (acc - mean[c]) / sd[c];
  }
}
// patch matrix for the stride-P patch embedding (conv P x P, stride P, no bias == GEMM): row = (b, py, px), col = (c, dy, dx)
__global__ void patchify_kernel(const float* __restrict__ img, float* __restrict__ out, int B, int S, int P) {
  const int np = S / P, K = 3 * P * P;
  const size_t n = (size_t)B * np * np * K;
  GRID_STRIDE(i, n) {
    const int col = (int)(i % K);
    const size_t row = i / K;
    const int px = (int)(row % np), py = (int)((row / np) % np), b = (int)(row / ((size_t)np * np));
    const int dx = col % P, dy = (col / P) % P, c = col / (P * P);
    out[i] = img[(((size_t)b * 3 + c) * S + (py * P + dy)) * S + px * P + dx];
  }
}
// x[b, 0] = class_embedding + pos[0]; x[b, 1 + i] = patch_i + pos[1 + i]      (CLIPVisionEmbeddings.forward)
__global__ void vit_tokens_kernel(const float* __restrict__ patches, const float* __restrict__ cls, const float* __restrict__ pos,
                                  float* __restrict__ out, int B, int N, int W) {
  const size_t n = (size_t)B * (N + 1) * W;
  GRID_STRIDE(i, n) {
    const int c = (int)(i % W);
    const int t = (int)((i / W) % (N + 1));
    const size_t b = i / ((size_t)(N + 1) * W);
    const float v = t == 0 ? cls[c] : patches[(b * N + (t - 1)) * W + c];
    out[i] = v + pos[(size_t)t * W + c];
  }
}
__global__ void gather_rows_kernel(const float* __restrict__ x, const int* __restrict__ rows, float* __restrict__ out, int B, int L, int W) {
  const size_t n = (size_t)B * W;
  GRID_STRIDE(i, n) {
    const size_t b = i / W;
    const int c = (int)(i - b * W);
    const int r = rows ? rows[b] : 0;
    out[i] = x[(b * L + r) * W + c];
  }
}
__global__ void eot_rows_kernel(const int* __restrict__ ids, int* __restrict__ rows, int B, int L) {      // text.argmax(dim=-1): first maximum
  GRID_STRIDE(b, (size_t)B) {
    int best = 0, bv = ids[b * L];
    for (int l = 1; l < L; ++l) {
      const int v = ids[b * L + l];
      if (v > bv) { bv = v; best = l; }
    }
    rows[b] = best;
  }
}
// one warp per sample
__global__ void dclip_scores_kernel(const float* __restrict__ img_f, const float* __restrict__ orig_f, const float* __restrict__ enc_f,
                                    const float* __restrict__ dec_f, int B, int D, float* __restrict__ clip_out, float* __restrict__ dclip_out) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  auto wsum = [&](float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
  };
  const float *pi = img_f + (size_t)b * D, *po = orig_f + (size_t)b * D, *pe = enc_f + (size_t)b * D, *pd = dec_f + (size_t)b * D;
  float si = 0.f, so = 0.f, se = 0.f, sd = 0.f;
  for (int c = lane; c < D; c += 32) { si += pi[c] * pi[c]; so += po[c] * po[c]; se += pe[c] * pe[c]; sd += pd[c] * pd[c]; }
  const float ni = sqrtf(wsum(si)), no = sqrtf(wsum(so)), ne = sqrtf(wsum(se)), nd = sqrtf(wsum(sd));
  float clip = 0.f, di2 = 0.f, dt2 = 0.f, dd = 0.f;
  for (int c = lane; c < D; c += 32) {
    const float a = pi[c] / ni, o = po[c] / no, e_ = pe[c] / ne, d = pd[c] / nd;
    clip += a * d;
    const float di = a - o, dt = d - e_;
    di2 += di * di; dt2 += dt * dt; dd += di * dt;
  }
  clip = wsum(clip); di2 = wsum(di2); dt2 = wsum(dt2); dd = wsum(dd);
  if (lane == 0) {
    clip_out[b] = clip;
    dclip_out[b] = dd / (sqrtf(di2) * sqrtf(dt2));         // <di / |di|, dt / |dt|>
  }
}
// PSNR / L2 partial sums (fp64) and SSIM over the valid region; grid = (tiles, B); out[b] = {sum sq diff, ssim sum over 3 channels}
__global__ void image_metrics_kernel(const float* __restrict__ a, const float* __restrict__ b_, int H, int W, double* __restrict__ acc) {
  const int img = blockIdx.y;
  const float* A = a + (size_t)img * 3 * H * W;
  const float* Bp = b_ + (size_t)img * 3 * H * W;
  __shared__ double gw[11];
  if (threadIdx.x == 0) {                 // cv2.getGaussianKernel(11, 1.5): exp(-(i-5)^2 / (2 sigma^2)), normalised
    double s = 0.0;
    for (int i = 0; i < 11; ++i) { gw[i] = exp(-((double)(i - 5) * (i - 5)) / (2.0 * 1.5 * 1.5)); s += gw[i]; }
    for (int i = 0; i < 11; ++i) gw[i] /= s;
  }
  __syncthreads();
  const int vh = H - 10, vw = W - 10;
  const size_t nvalid = (size_t)3 * vh * vw, npix = (size_t)3 * H * W;
  double sq = 0.0, ss = 0.0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < npix; i += (size_t)gridDim.x * blockDim.x) {
    const float x = fminf(fmaxf(A[i], 0.f), 1.f), y = fminf(fmaxf(Bp[i], 0.f), 1.f);
    const float d = x - y;
    sq += (double)(d * d);                 // fp32 subtract / square as torch does, fp64 accumulation
  }
  const double C1 = (0.01 * 255) * (0.01 * 255), C2 = (0.03 * 255) * (0.03 * 255);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvalid; i += (size_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % vw), y = (int)((i / vw) % vh), c = (int)(i / ((size_t)vw * vh));
    const float* pa = A + (size_t)c * H * W;
    const float* pb = Bp + (size_t)c * H * W;
    double m1 = 0, m2 = 0, s11 = 0, s22 = 0, s12 = 0;
    for (int dy = 0; dy < 11; ++dy) {
      for (int dx = 0; dx < 11; ++dx) {
        const double w = gw[dy] * gw[dx];
        // (img.numpy() * 255): fp32 product, then astype(float64)
        const double u = (double)(fminf(fmaxf(pa[(size_t)(y + dy) * W + x + dx], 0.f), 1.f) * 255.f);
        const double v = (double)(fminf(fmaxf(pb[(size_t)(y + dy) * W + x + dx], 0.f), 1.f) * 255.f);
        m1 += w * u; m2 += w * v; s11 += w * u * u; s22 += w * v * v; s12 += w * u * v;
      }
    }
    const double v1 = s11 - m1 * m1, v2 = s22 - m2 * m2, cv = s12 - m1 * m2;
    ss += ((2 * m1 * m2 + C1) * (2 * cv + C2)) / ((m1 * m1 + m2 * m2 + C1) * (v1 + v2 + C2));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { sq += __shfl_xor_sync(0xffffffffu, sq, o); ss += __shfl_xor_sync(0xffffffffu, ss, o); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(acc + 2 * img, sq); atomicAdd(acc + 2 * img + 1, ss); }
}
__global__ void image_metrics_final_kernel(const double* __restrict__ acc, int B, int H, int W, float* __restrict__ out) {
  GRID_STRIDE(b, (size_t)B) {
    const double sq = acc[2 * b], ss = acc[2 * b + 1];
    const float mse = (float)(sq / ((double)3 * H * W));
    out[3 * b + 0] = mse == 0.f ? 100.f : 10.f * log10f(1.f / mse);
    out[3 * b + 1] = (float)(ss / ((double)3 * (H - 10) * (W - 10)));
    out[3 * b + 2] = sqrtf((float)sq);
  }
}

void latent_chains_init(Engine& e, const LatentChains& a, cudaStream_t s) {
  if (a.solver) LAUNCH1(latent_chains_init_kernel<1>, a.n, a);
  else LAUNCH1(latent_chains_init_kernel<0>, a.n, a);
}
template <int SOLVER>
void launch_step(Engine& e, const LatentChains& a, cudaStream_t s) {
  if (a.sg_m && a.sg_mask) {
    CDX_CHECK(a.sg_mask <= 2 && a.sg_map && a.sg_gh >= 2 && a.sg_gw >= 2 && a.w > 0 && a.hw == (4 * a.sg_gh) * (4 * a.sg_gw) && a.w == 4 * a.sg_gw,
              "latent_chains_step: mask mode %d over a %dx%d map, hw=%d w=%d", a.sg_mask, a.sg_gh, a.sg_gw, a.hw, a.w);
    if (a.sg_mask == 1) {
      if (a.mask) {
        if (a.pred) LAUNCH1((latent_chains_step_kernel<1, 1, 2, SOLVER>), a.n, a);
        else LAUNCH1((latent_chains_step_kernel<0, 1, 2, SOLVER>), a.n, a);
      } else {
        if (a.pred) LAUNCH1((latent_chains_step_kernel<1, 0, 2, SOLVER>), a.n, a);
        else LAUNCH1((latent_chains_step_kernel<0, 0, 2, SOLVER>), a.n, a);
      }
    } else {
      if (a.mask) {
        if (a.pred) LAUNCH1((latent_chains_step_kernel<1, 1, 3, SOLVER>), a.n, a);
        else LAUNCH1((latent_chains_step_kernel<0, 1, 3, SOLVER>), a.n, a);
      } else {
        if (a.pred) LAUNCH1((latent_chains_step_kernel<1, 0, 3, SOLVER>), a.n, a);
        else LAUNCH1((latent_chains_step_kernel<0, 0, 3, SOLVER>), a.n, a);
      }
    }
    return;
  }
  if (a.sg_m) {
    if (a.mask) {
      if (a.pred) LAUNCH1((latent_chains_step_kernel<1, 1, 1, SOLVER>), a.n, a);
      else LAUNCH1((latent_chains_step_kernel<0, 1, 1, SOLVER>), a.n, a);
    } else {
      if (a.pred) LAUNCH1((latent_chains_step_kernel<1, 0, 1, SOLVER>), a.n, a);
      else LAUNCH1((latent_chains_step_kernel<0, 0, 1, SOLVER>), a.n, a);
    }
    return;
  }
  if (a.mask) {
    if (a.pred) LAUNCH1((latent_chains_step_kernel<1, 1, 0, SOLVER>), a.n, a);
    else LAUNCH1((latent_chains_step_kernel<0, 1, 0, SOLVER>), a.n, a);
  } else {
    if (a.pred) LAUNCH1((latent_chains_step_kernel<1, 0, 0, SOLVER>), a.n, a);
    else LAUNCH1((latent_chains_step_kernel<0, 0, 0, SOLVER>), a.n, a);
  }
}
void latent_chains_step(Engine& e, const LatentChains& a, cudaStream_t s) {
  CDX_CHECK(a.solver >= 0 && a.solver <= 2, "latent_chains_step: solver %d", a.solver);
  if (a.solver == 2) launch_step<2>(e, a, s);
  else if (a.solver == 1) launch_step<1>(e, a, s);
  else launch_step<0>(e, a, s);
}
void semantic_thresholds(Engine& e, const LatentChains& a, cudaStream_t s) {
  CDX_CHECK(a.sg_m >= 1 && a.sg_m <= SEMANTIC_MAX_CONCEPTS && a.hw > 0 && a.chw % a.hw == 0, "semantic_thresholds: m=%d chw=%d hw=%d", a.sg_m,
            a.chw, a.hw);
  if (e.dry()) return;
  const long long rows = (long long)a.n_src * a.K * a.sg_m;
  if (a.sg_mask) {
    CDX_CHECK(a.sg_mask <= 2 && a.sg_map && a.sg_gh >= 2 && a.sg_gw >= 2 && a.hw == (4 * a.sg_gh) * (4 * a.sg_gw),
              "semantic_thresholds: mask mode %d over a %dx%d map, hw=%d", a.sg_mask, a.sg_gh, a.sg_gw, a.hw);
    if (rows == 0) return;
    const long long blocks = rows * a.sg_mask;
    ProfScope ps(e, s, PROF_ELEMENTWISE, 0.0, 4.0 * rows * ((double)a.sg_gh * a.sg_gw + (a.sg_mask == 2 ? 2.0 * a.chw : 0.0)), 1);
    ps.note("semantic attention-mask thresholds %lld rows, %dx%d maps%s", rows, a.sg_gh, a.sg_gw, a.sg_mask == 2 ? " + channel sums" : "");
    if (a.sg_mask == 1) semantic_threshold_kernel<1><<<(unsigned)blocks, SEMANTIC_THREADS, 0, s>>>(a);
    else semantic_threshold_kernel<2><<<(unsigned)blocks, SEMANTIC_THREADS, 0, s>>>(a);
    CDX_CUDA(cudaGetLastError());
    e.launches++;
    return;
  }
  const long long planes = rows * (a.chw / a.hw);
  if (planes == 0) return;
  ProfScope ps(e, s, PROF_ELEMENTWISE, 0.0, 2.0 * 4.0 * planes * a.hw, 1);     // algorithmic: o_k and o_uc read once
  ps.note("semantic thresholds %lld planes x %d", planes, a.hw);
  semantic_threshold_kernel<0><<<(unsigned)planes, SEMANTIC_THREADS, 0, s>>>(a);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}
void mask_pool(Engine& e, const float* mask, float* out, int B, int H, int W, int f, cudaStream_t s) {
  CDX_CHECK(B >= 1 && f >= 1 && H >= f && W >= f && H % f == 0 && W % f == 0, "mask_pool: %dx%d mask, factor %d", H, W, f);
  LAUNCH1(mask_pool_kernel, (size_t)B * (H / f) * (W / f), mask, out, B, H, W, f);
}
void mask_composite(Engine& e, const float* dec, const float* image, const float* mask, float* out, int B, int C, int H, int W,
                    cudaStream_t s) {
  CDX_CHECK(B >= 1 && C >= 1 && H >= 1 && W >= 1, "mask_composite: B=%d C=%d %dx%d", B, C, H, W);
  const size_t n = (size_t)B * C * H * W;
  LAUNCH1(mask_composite_kernel, n, dec, image, mask, out, C, (size_t)H * W, n);
}
void edit_rows(Engine& e, const float* x0, const float* noise, float sa, float s1, float* xin, int B, int n_maps, int chw, int p0, int p1,
               cudaStream_t s) {
  const size_t n = (size_t)(p1 - p0) * chw;
  LAUNCH1(edit_rows_kernel, n, x0, noise, sa, s1, xin, B, n_maps, chw, p0, n);
}
void edit_map_accum(Engine& e, const float* src, const float* tgt, long long sb, long long sk, long long off0, float vscale, float* acc, int B,
                    int C, int hw, int p0, int p1, cudaStream_t s) {
  LAUNCH1(edit_map_accum_kernel, (size_t)B * hw, src, tgt, sb, sk, off0, vscale, acc, B, C, hw, p0, p1);
}
void edit_mask(Engine& e, const float* acc, int n_maps, float ratio, float* map_out, float* mask_out, float* img_out, int f, int B, int C, int h,
               int w, cudaStream_t s) {
  CDX_CHECK(B >= 1 && C >= 1 && h >= 1 && w >= 1 && n_maps >= 1 && f >= 1, "edit_mask: B=%d C=%d %dx%d n_maps=%d f=%d", B, C, h, w, n_maps, f);
  if (e.dry()) return;
  edit_mask_kernel<<<B, EDIT_MASK_THREADS, 0, s>>>(acc, (float)(n_maps * C), ratio, map_out, mask_out, img_out, f, h, w);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}
void ensemble_select(Engine& e, int n, const float* scores, const long long* cand, const int* sample, const float* images, float* best_score,
                     long long* best_idx, float* best_img, float* score_mat, int B, int n_total, size_t img_n, cudaStream_t s) {
  if (e.dry() || n <= 0 || B <= 0) return;
  ensemble_select_kernel<<<B, 256, 0, s>>>(n, scores, cand, sample, images, best_score, best_idx, best_img, score_mat, n_total, img_n);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}
void affine(Engine& e, const float* x, float a, float b, float* out, size_t n, cudaStream_t s) { LAUNCH1(affine_kernel, n, x, a, b, out, n); }
void shift_scale(Engine& e, const float* x, float b, float a, float* out, size_t n, cudaStream_t s) { LAUNCH1(shift_scale_kernel, n, x, b, a, out, n); }
void q_sample(Engine& e, const float* x0, const float* nz, float sa, float s1, float* out, size_t n, cudaStream_t s) { LAUNCH1(q_sample_kernel, n, x0, nz, sa, s1, out, n); }
void silu(Engine& e, const float* x, float* y, size_t n, cudaStream_t s) { LAUNCH1(silu_kernel, n, x, y, n); }
void add(Engine& e, const float* a, const float* b, float* y, size_t n, cudaStream_t s) { LAUNCH1(add_kernel, n, a, b, y, n); }
void copy_rows(Engine& e, const float* a, float* y, size_t n, cudaStream_t s) { LAUNCH1(copy_kernel, n, a, y, n); }
void geglu(Engine& e, const float* x, float* y, int M, int C, cudaStream_t s, bool interleaved) {
  LAUNCH1(geglu_kernel, (size_t)M * C, x, y, (size_t)M, C, interleaved ? 1 : 0);
}
void interleave_geglu_rows(Engine& e, const float* src, float* dst, int rows, int rowlen, cudaStream_t s) {
  CDX_CHECK(rows % 128 == 0, "interleave_geglu_rows: %d rows", rows);
  LAUNCH1(interleave_geglu_rows_kernel, (size_t)rows * rowlen, src, dst, rows, rowlen);
}
void avgpool2(Engine& e, const float* x, float* y, int B, int H, int W, int C, cudaStream_t s) {
  CDX_CHECK(H % 2 == 0 && W % 2 == 0, "avgpool2: odd size %dx%d", H, W);
  LAUNCH1(avgpool2_kernel, (size_t)B * (H / 2) * (W / 2) * C, x, y, B, H, W, C);
}
void upsample2(Engine& e, const float* x, float* y, int B, int H, int W, int C, cudaStream_t s) {
  LAUNCH1(upsample2_kernel, (size_t)B * H * W * 4 * C, x, y, B, H, W, C);
}
void nchw_to_nhwc(Engine& e, const float* x, float* y, int B, int C, int HW, cudaStream_t s) {
  if (e.dry()) return;
  // x [b][C][HW] -> y [b][HW][C]
  transpose_kernel<<<dim3(cdiv(HW, 32), cdiv(C, 32), B), dim3(32, 8), 0, s>>>(x, y, C, HW);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}
void nhwc_to_nchw(Engine& e, const float* x, float* y, int B, int C, int HW, cudaStream_t s) {
  if (e.dry()) return;
  transpose_kernel<<<dim3(cdiv(C, 32), cdiv(HW, 32), B), dim3(32, 8), 0, s>>>(x, y, HW, C);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}
void timestep_embedding(Engine& e, const float* t, const float* freqs, float* emb, int B, int half, cudaStream_t s, bool sin_first) {
  if (e.dry()) return;
  temb_kernel<<<cdiv(B * half, 256), 256, 0, s>>>(t, freqs, emb, B, half, sin_first ? 1 : 0);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}
void repack_conv3x3(Engine& e, const float* w, float* o, int O, int I, cudaStream_t s, int Ipad) {
  const int Ip = Ipad > 0 ? Ipad : I;
  LAUNCH1(repack_conv_kernel, (size_t)O * Ip * 9, w, o, O, I, Ip);
}
void embed_tokens(Engine& e, const int* ids, const float* tok, const float* pos, float* out, int B, int L, int W, int vocab, cudaStream_t s) {
  LAUNCH1(embed_tokens_kernel, (size_t)B * L * W, ids, tok, pos, out, B, L, W, vocab);
}
void quick_gelu(Engine& e, const float* x, float* y, size_t n, cudaStream_t s) { LAUNCH1(quick_gelu_kernel, n, x, y, n); }
void gelu(Engine& e, const float* x, float* y, size_t n, cudaStream_t s) { LAUNCH1(gelu_kernel, n, x, y, n); }
void pad_channels(Engine& e, const float* x, float* y, size_t rows, int C, int Cp, cudaStream_t s) {
  LAUNCH1(pad_channels_kernel, rows * (size_t)Cp, x, y, rows, C, Cp);
}
void vae_posterior(Engine& e, const float* mom, const float* nz, float sf, float* out, int B, int C, int hw, cudaStream_t s) {
  LAUNCH1(vae_posterior_kernel, (size_t)B * C * hw, mom, nz, sf, out, B, C, hw);
}
void ddim_posterior_sample(Engine& e, const float* x0, const float* xt, const float* nz, const cdx_ddim_coef& c, float* out, size_t n, cudaStream_t s) {
  LAUNCH1(ddim_posterior_kernel, n, x0, xt, nz, c, out, n);
}
void ddim_compute_eps(Engine& e, const float* xt, const float* xn, const float* e_c, const float* e_uc, float scale, const cdx_ddim_coef& c,
                      float* out, size_t n, cudaStream_t s) {
  LAUNCH1(ddim_compute_eps_kernel, n, xt, xn, e_c, e_uc, scale, c, out, n);
}
void ddim_step_with_eps(Engine& e, const float* x, const float* e_c, const float* e_uc, float scale, const float* eps, const cdx_ddim_coef& c,
                        float* out, size_t n, cudaStream_t s) {
  LAUNCH1(ddim_step_kernel, n, x, e_c, e_uc, scale, eps, c, out, n);
}
void pixel_posterior_sample(Engine& e, const float* x0, const float* xt, const float* nz, const cdx_pixel_coef& c, float* out, size_t n, cudaStream_t s) {
  LAUNCH1(pixel_posterior_kernel, n, x0, xt, nz, c, out, n);
}
void pixel_compute_eps(Engine& e, const float* xt, const float* xn, const float* et, const cdx_pixel_coef& c, float* out, int B, int chw,
                       int net_chw, cudaStream_t s) {
  LAUNCH1(pixel_compute_eps_kernel, (size_t)B * chw, xt, xn, et, c, out, B, chw, net_chw);
}
void pixel_step_with_eps(Engine& e, const float* xt, const float* et, const float* eps, const cdx_pixel_coef& c, float* out, int B, int chw,
                         int net_chw, cudaStream_t s) {
  LAUNCH1(pixel_step_kernel, (size_t)B * chw, xt, et, eps, c, out, B, chw, net_chw);
}
void pixel_lockstep_step(Engine& e, const float* x0, float* xs, float* ys, const float* et_src, const float* et_tgt, const float* noise,
                         const cdx_pixel_coef& c, int B, int chw, int net_chw_src, int net_chw_tgt, cudaStream_t s) {
  LAUNCH1(pixel_lockstep_kernel, (size_t)B * chw, x0, xs, ys, et_src, et_tgt, noise, c, B, chw, net_chw_src, net_chw_tgt);
}

// softmax(q k^T * scale) v through two batched contractions and a row softmax.  Scores live in the arena
// ([B*heads, Nq, ldS]); the fused wgmma flash kernel supersedes this when eligible.
void attention(Engine& e, const float* q, int ldq, const float* k, int ldk, const float* v, int ldv, float* out, int ldo, int B, int Nq,
               int Nk, int heads, int d, int head_stride, float scale, cudaStream_t s, bool causal) {
  Scope sc(e.arena);
  const int ldS = (Nk + 3) & ~3;
  float* S = (float*)e.arena.alloc((size_t)B * heads * Nq * ldS * sizeof(float));
  GemmArgs g;
  g.M = Nq; g.N = Nk; g.K = d; g.mode = 0;
  g.A = q; g.lda = ldq; g.C1 = d;
  g.Bw = k; g.ldb = ldk; g.b_kn = 0;
  g.Cout = S; g.ldc = ldS; g.alpha = scale;
  g.batch = B; g.heads = heads;
  g.sA_b = (long long)Nq * ldq; g.sA_h = head_stride;
  g.sB_b = (long long)Nk * ldk; g.sB_h = head_stride;
  g.sC_b = (long long)heads * Nq * ldS; g.sC_h = (long long)Nq * ldS;
  gemm(e, g, s);
  softmax_rows(e, S, (long long)B * heads * Nq, Nk, ldS, s, causal ? Nq : 0);
  GemmArgs h;
  h.M = Nq; h.N = d; h.K = Nk; h.mode = 0;
  h.A = S; h.lda = ldS; h.C1 = Nk;
  h.Bw = v; h.ldb = ldv; h.b_kn = 1;
  h.Cout = out; h.ldc = ldo;
  h.batch = B; h.heads = heads;
  h.sA_b = (long long)heads * Nq * ldS; h.sA_h = (long long)Nq * ldS;
  h.sB_b = (long long)Nk * ldv; h.sB_h = head_stride;
  h.sC_b = (long long)Nq * ldo; h.sC_h = d;
  gemm(e, h, s);
}

}  // namespace cdx

namespace cdx {
namespace {
// one warp per latent pixel; lanes stride over the codebook, (distance, index) min-reduced with ties to the LOWER index (torch.argmin)
__global__ void vq_quantize_kernel(const float* __restrict__ z, const float* __restrict__ cb, float* __restrict__ out, size_t npix, int dim, int n_embed) {
  const size_t pix = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (pix >= npix) return;
  const float* zp = z + pix * dim;
  float zz = 0.f;
  for (int c = 0; c < dim; ++c) zz += zp[c] * zp[c];
  float best = 3.4e38f;
  int bi = 0x7fffffff;
  for (int k = lane; k < n_embed; k += 32) {
    const float* e = cb + (size_t)k * dim;
    float ee = 0.f, dot = 0.f;
    for (int c = 0; c < dim; ++c) { ee += e[c] * e[c]; dot += zp[c] * e[c]; }
    const float d = (zz + ee) - 2.f * dot;
    if (d < best) { best = d; bi = k; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob < best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  for (int c = lane; c < dim; c += 32) out[pix * dim + c] = zp[c] + (cb[(size_t)bi * dim + c] - zp[c]);      // z + (z_q - z).detach()
}
}  // namespace
void vq_quantize(Engine& e, const float* z, const float* codebook, float* out, size_t npix, int dim, int n_embed, cudaStream_t s) {
  if (e.dry()) return;
  vq_quantize_kernel<<<(unsigned)((npix + 7) / 8), 256, 0, s>>>(z, codebook, out, npix, dim, n_embed);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}
void clip_preprocess(Engine& e, const float* img, int B, int R, int size, float* out, cudaStream_t s) {
  LAUNCH1(clip_preprocess_kernel, (size_t)B * 3 * size * size, img, B, R, size, out);
}
void patchify(Engine& e, const float* img, float* out, int B, int S, int P, cudaStream_t s) {
  LAUNCH1(patchify_kernel, (size_t)B * 3 * S * S, img, out, B, S, P);
}
void vit_tokens(Engine& e, const float* patches, const float* cls, const float* pos, float* out, int B, int N, int W, cudaStream_t s) {
  LAUNCH1(vit_tokens_kernel, (size_t)B * (N + 1) * W, patches, cls, pos, out, B, N, W);
}
void gather_rows(Engine& e, const float* x, const int* rows, float* out, int B, int L, int W, cudaStream_t s) {
  LAUNCH1(gather_rows_kernel, (size_t)B * W, x, rows, out, B, L, W);
}
void eot_rows(Engine& e, const int* ids, int* rows, int B, int L, cudaStream_t s) { LAUNCH1(eot_rows_kernel, (size_t)B, ids, rows, B, L); }
void dclip_scores(Engine& e, const float* img_f, const float* orig_f, const float* enc_f, const float* dec_f, int B, int D, float* clip_out,
                  float* dclip_out, cudaStream_t s) {
  if (e.dry()) return;
  dclip_scores_kernel<<<cdiv(B, 4), 128, 0, s>>>(img_f, orig_f, enc_f, dec_f, B, D, clip_out, dclip_out);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}
void image_metrics(Engine& e, const float* a, const float* b, int B, int H, int W, float* out, cudaStream_t s) {
  CDX_CHECK(H > 10 && W > 10, "image_metrics: %dx%d is smaller than the 11x11 SSIM window", H, W);
  Scope sc(e.arena);
  double* acc = (double*)e.arena.alloc((size_t)B * 2 * sizeof(double));
  if (e.dry()) return;
  CDX_CUDA(cudaMemsetAsync(acc, 0, (size_t)B * 2 * sizeof(double), s));
  const int tiles = std::min(e.num_sms * 4, cdiv((long long)3 * H * W, 256));
  image_metrics_kernel<<<dim3(tiles, B), 256, 0, s>>>(a, b, H, W, acc);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
  LAUNCH1(image_metrics_final_kernel, (size_t)B, acc, B, H, W, out);
}
}  // namespace cdx

// ------------------------------------------------------------------------------------------------ Prompt-to-Prompt's LocalBlend
namespace cdx {
namespace {
constexpr int BLEND_THREADS = 256;
__global__ void blend_weights_kernel(const float* v, const float* A, const float* d, float* out, int L) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= L) return;
  float r = 0.f;
  if (A) {
    for (int n = 0; n < L; ++n) r = fmaf(A[(size_t)q * L + n], v[n], r);
  } else {
    r = d ? __fmul_rn(d[q], v[q]) : v[q];
  }
  out[q] = r;
}
// one CTA per image: the running sums, their maxima, the grid mask in shared memory, then the latent mask
__global__ void __launch_bounds__(BLEND_THREADS) local_blend_mask_kernel(const float* maps, int n_terms, int n_vec, float* run,
                                                                         const float* umask, float th_blend, float th_sub, float* mask,
                                                                         int gh, int gw) {
  extern __shared__ unsigned char cell[];          // [gh*gw]: the grid mask
  __shared__ float red[BLEND_THREADS];
  __shared__ float mx[4];
  const int b = blockIdx.x, G = gh * gw;
  float* R = run + (size_t)b * n_vec * G;
  for (int p = threadIdx.x; p < G; p += BLEND_THREADS)
    for (int v = 0; v < n_vec; ++v) {
      const float* m = maps + (size_t)(b * n_vec + v) * n_terms * G + p;
      float wsum = m[0];
      for (int t = 1; t < n_terms; ++t) wsum = __fadd_rn(wsum, m[(size_t)t * G]);
      R[(size_t)v * G + p] = __fadd_rn(R[(size_t)v * G + p], wsum);
    }
  __syncthreads();
  // the maximum of each running map (the 3x3 max-pool keeps it); the maps are >= 0
  for (int v = 0; v < n_vec; ++v) {
    float m = 0.f;
    for (int p = threadIdx.x; p < G; p += BLEND_THREADS) m = fmaxf(m, R[(size_t)v * G + p]);
    red[threadIdx.x] = m;
    __syncthreads();
    for (int o = BLEND_THREADS / 2; o > 0; o >>= 1) {
      if (threadIdx.x < o) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + o]);
      __syncthreads();
    }
    if (threadIdx.x == 0) mx[v] = red[0];
    __syncthreads();
  }
  for (int p = threadIdx.x; p < G; p += BLEND_THREADS) {
    const int y = p / gw, x = p - y * gw;
    bool keep = false;
    for (int v = 0; v < 2; ++v) {                  // blend words: pooled map / max > th_blend, source OR target
      const float* r = R + (size_t)v * G;
      float pm = r[p];
      for (int yy = max(y - 1, 0); yy <= min(y + 1, gh - 1); ++yy)
        for (int xx = max(x - 1, 0); xx <= min(x + 1, gw - 1); ++xx) pm = fmaxf(pm, r[yy * gw + xx]);
      keep |= mx[v] > 0.f && __fdiv_rn(pm, mx[v]) > th_blend;
    }
    for (int v = 2; v < n_vec; ++v)                // subtract words: map / max > th_sub removes the cell
      keep &= !(mx[v] > 0.f && __fdiv_rn(R[(size_t)v * G + p], mx[v]) > th_sub);
    cell[p] = keep;
  }
  __syncthreads();
  const int w = 4 * gw, hw = 16 * G;
  for (int i = threadIdx.x; i < hw; i += BLEND_THREADS) {
    const int y = i / w, x = i - y * w;
    mask[(size_t)b * hw + i] = cell[(y >> 2) * gw + (x >> 2)] ? (umask ? umask[(size_t)b * hw + i] : 1.f) : 0.f;
  }
}
}  // namespace

void blend_weights(Engine& e, const float* v, const float* A, const float* d, float* out, int L, cudaStream_t s) {
  CDX_CHECK(v && out && L >= 1 && !(A && d), "blend_weights: L=%d", L);
  if (e.dry()) return;
  blend_weights_kernel<<<cdiv(L, 128), 128, 0, s>>>(v, A, d, out, L);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}

void local_blend_mask(Engine& e, const float* maps, int n_terms, int n_vec, float* run, const float* umask, float th_blend, float th_sub,
                      float* mask, int B, int h, int w, cudaStream_t s) {
  CDX_CHECK(maps && run && mask && B >= 1 && h >= 4 && w >= 4 && h % 4 == 0 && w % 4 == 0 && n_terms >= 1 && (n_vec == 2 || n_vec == 4),
            "local_blend_mask: B=%d %dx%d (multiples of 4) n_terms=%d n_vec=%d", B, h, w, n_terms, n_vec);
  CDX_CHECK(th_blend >= 0.f && th_blend < 1.f && th_sub >= 0.f && th_sub < 1.f, "local_blend_mask: thresholds %g, %g outside [0, 1)", th_blend,
            th_sub);
  const int gh = h / 4, gw = w / 4;
  CDX_CHECK((size_t)gh * gw <= 48 * 1024, "local_blend_mask: a %dx%d grid", gh, gw);
  if (e.dry()) return;
  ProfScope ps(e, s, PROF_ELEMENTWISE, 0.0, 4.0 * B * ((double)n_vec * gh * gw * (n_terms + 2) + (umask ? 2.0 : 1.0) * h * w), 1);
  local_blend_mask_kernel<<<B, BLEND_THREADS, (size_t)gh * gw, s>>>(maps, n_terms, n_vec, run, umask, th_blend, th_sub, mask, gh, gw);
  CDX_CUDA(cudaGetLastError());
  e.launches++;
}
}  // namespace cdx
