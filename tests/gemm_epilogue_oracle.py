"""References for the GEMM epilogue tests (tests/test_gemm_epilogue_gpu.py), pinned on the CPU by tests/test_gemm_epilogue_cpu.py.

rn_tf32 is the kernels' rounding of an fp32 value to a TF32 plane, (bits + 0x1000) & 0xFFFFE000: round half away from zero on the
magnitude (not round-to-even), emulated here in integer arithmetic on the bit patterns.

GEGLU bound.  With u = 2^-24 the kernels compute o = v * (0.5f * g * (1 + erff(g * 0.70710678f))) in fp32 from the fp32 value
v and gate g.  t = g * c carries two roundings (c and the product): |t - g/sqrt2| <= 2u |t|, which moves erf by at most
(2/sqrt(pi)) exp(-t^2) * 2u |t|; erff is within 2 ulp (CUDA programming guide, <= 4u relative); 1 + erf adds u |1 + erf| and
leaves the absolute error of erf as it is (it cancels towards g -> -inf, so that error is not relative to 1 + erf); 0.5 * g is
exact and the two remaining products add u each:
    |o - o64| <= 0.5 |v| |g| (d_erf + u |1 + erf|) + 2u |o64|,   d_erf = 4u |erf(t)| + (2/sqrt(pi)) exp(-t^2) 2u |t|.

fp16-split floor.  The fp16-split GEMM stores x * 2^e (e from the operand's range slot, x * 2^e < 2^15) as hi = fp16(x'),
lo = fp16(x' - hi).  x' - hi is exact in fp32; rounding it to fp16 costs 2^-11 of |lo| <= 2^-22 |x'| while lo is normal, and half the
subnormal spacing, 2^-25, once it is not.  So each element of A carries an absolute error of up to 2^-25 2^-e_a on top of the
relative one, and each weight 2^-25 2^-b_exp.  Over a dot product that is
    floor[m, n] = 2^-25 (2^-e_a sum_k |W[n, k]| + 2^-b_exp sum_k |A[m, k]|),
which is added to the per-op relative budget.  It matters when a tracked slot or the net's weight range is far above the values
that take part: a conservative slot 2^8 above the true range costs 8 bits of every A element.
"""
import math

import torch

U = 2.0 ** -24


def rn_tf32(x):
    """the kernels' TF32 rounding of a float32 tensor (bit pattern (b + 0x1000) & 0xFFFFE000), as float32"""
    b = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = ((b + 0x1000) & 0xFFFFE000) & 0xFFFFFFFF
    r = torch.where(r >= 2 ** 31, r - 2 ** 32, r)
    return r.to(torch.int32).view(torch.float32)


def tf32_planes(y):
    """(hi, lo) planes of a float32 tensor as the epilogue stores them: hi = rn_tf32(y), lo = rn_tf32(y - hi) (fp32 difference)"""
    hi = rn_tf32(y)
    return hi, rn_tf32(y - hi)


def h16_exp(amax):
    """exponent e with amax * 2^e in [2^14, 2^15), clamped to [-100, 100]; 0 for a zero or non-finite range (h16_exp_host)"""
    amax = float(amax)
    if not (amax > 0.0) or not math.isfinite(amax):
        return 0
    _, ex = math.frexp(amax)
    return min(max(14 - (ex - 1), -100), 100)


def split_floor(a_abs_sum, w_abs_sum, e_a, b_exp):
    """the fp16-split floor of the module docstring: a_abs_sum [M] = sum_k |A[m, k]|, w_abs_sum [N] = sum_k |W[n, k]| (float64)"""
    return 2.0 ** -25 * (2.0 ** -e_a * w_abs_sum[None, :] + 2.0 ** -b_exp * a_abs_sum[:, None])


def split_h16(x, e):
    """float64 value of the two fp16 planes of float32 x at exponent e, (hi + lo) * 2^-e"""
    xs = x.float() * 2.0 ** e
    hi = xs.half().float()
    lo = (xs - hi).half().float()
    return (hi.double() + lo.double()) * 2.0 ** -e


def deinterleave_geglu(w):
    """[N, K] weights in [32 value | 32 gate] row blocks -> (value rows [N/2, K], gate rows [N/2, K])"""
    N = w.shape[0]
    blk = w.reshape(N // 64, 2, 32, *w.shape[1:])
    return blk[:, 0].reshape(N // 2, *w.shape[1:]), blk[:, 1].reshape(N // 2, *w.shape[1:])


def geglu_ref(y):
    """value * gelu(gate) of an [M, N] product over [32 value | 32 gate] column blocks -> (o [M, N/2], v, g), float64"""
    v, g = (t.t() for t in deinterleave_geglu(y.double().t()))
    return v * 0.5 * g * (1.0 + torch.erf(g / math.sqrt(2.0))), v, g


def geglu_bound(v, g):
    """the GEGLU bound of the module docstring, elementwise (float64 v, g)"""
    t = g / math.sqrt(2.0)
    erf = torch.erf(t)
    d_erf = 4 * U * erf.abs() + 2.0 / math.sqrt(math.pi) * torch.exp(-t * t) * 2 * U * t.abs()
    o = v * 0.5 * g * (1.0 + erf)
    return 0.5 * v.abs() * g.abs() * (d_erf + U * (1.0 + erf).abs()) + 2 * U * o.abs()


def nchw_index(b, n, r, N, rows_per_img):
    """element offset of row m = b * rows_per_img + r, column n in the epilogue's NCHW store"""
    return (b * N + n) * rows_per_img + r


def ct_index(m, n, t_col0, ldt):
    """element offset of row m, column n >= t_col0 in a transposed plane"""
    return (n - t_col0) * ldt + m
