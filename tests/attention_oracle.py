"""float64 reference and derived error bound for attention as the kernels compute it (tests/test_attention_bound_gpu.py), pinned on the
CPU by tests/test_attention_bound_cpu.py.

out[b, i, h*d + c] = sum_j w_ij v[b, j, h*d + c],  w_ij = softmax_j(scale <q_i, k_j>) over the head's d channels.

The reference is computed twice in float64 (on the device, chunked over heads and query blocks so that a 9216-token level fits):
O64 on the exact fp32 inputs, and O64r on the operands as the kernel's planes represent them -- fp16 hi + lo of x * 2^e at the
exponent of the operand's range slot (split_h16 of gemm_epilogue_oracle, with the device's h16_exp_of), the hi plane alone for
the one-term kernel (mma mode 5), or TF32 hi + lo (rn_tf32(x), rn_tf32(x - hi)).  |O64r - O64| is the representation error itself
(three-term: <= 2^-22 relative per operand element plus the split floor 2^-25 2^-e of the shared slot; one-term: 2^-11 relative
plus the floor); the bound adds to it what the kernel's arithmetic on those represented operands can cost.  With u = 2^-24,
w the float64 weights of O64r, A_ic = sum_j w_ij |v_jc|, l_i = sum_j exp(s_ij - max_j s_ij) >= 1 and nb the key blocks of 64:

Scores.  S = Q K^T as hi.hi + hi.lo + lo.hi wgmma products: the dropped lo.lo term is <= 2^-22 |q||k| per channel, and the
tensor core's fp32 accumulation truncates (see kernels_tc.cu), one truncation <= 2u of the running sum per instruction: 3 (one-term
1) instructions per 16 (TF32 8) channels, with two more for the instruction's own alignment.  So
    dS_i <= scale (2^-22 + (n_qk + 2) 2u) max_j sum_c |q_ic| |k_jc|.
Exponents.  p = ex2.approx.ftz(fma(s, scale log2e 2^-(eq+ek), 10 - m)): the argument carries scale log2e's two roundings and the fma's,
<= 4u (|s|max log2e + 10) in log2 units with m <= |s|max log2e; ex2.approx is within 2^-22 relative (taken as 2^-21); every block's
corr = ex2(m_old - m_new) adds the same again, and the key split's merge two more.  All these move a weight by a factor in e^{+-D_i}:
    D_i = dS_i + (nb + 3) (2^-21 + ln2 4u (2 |s|max log2e + 10)).
Softmax perturbation.  Weights moved by factors within e^{+-D} move the output by at most (e^{2D} - 1) sum_j w_j |v_j - O_i|, which
is <= (e^{2D} - 1) (A_ic + |O_ic|).
P split.  P enters P.V as fp16(p 2^10) hi + lo (three-term: <= 2^-22 relative while lo is normal; one-term: hi alone, 2^-11
relative), or TF32 hi + lo left to the tensor core's truncation (2^-21).  Below fp16's normal range the spacing is 2^-24: half of it,
2^-25 2^-10 = 2^-35, absolute per p (p <= 1 relative to the running max, and the later rescale only shrinks it).  The row sum l
takes the unsplit p, so this is not a weight perturbation: it costs rho_P A_ic + 2^-35 sum_j |v_jc| / l_i.
Output.  Per key block one m64nNV accumulation of 3 (one-term 1) instructions per 16 keys (TF32: per 8), 2u each, plus the dropped
lo.lo term 2^-22; nb round-to-nearest O corr + O_j (<= 2u each, the multiply and the add); the merge 2u; all <= Sum |terms| <= A_ic.
l sums 16 values per thread, adds over nb blocks, merges and sums the quad: relative (nb + 24) u, carried into O / l as |O_ic| (nb +
24) u, and the final oscale / l and the product 2u |O_ic|.  The accumulating launch adds u |out|.

Generic route (attention(): two FFMA contractions around softmax_rows, fp32 round-to-nearest): dS_i = scale (d + 4) u max_j sum_c
|q_ic||k_jc|, D_i = dS_i + 2^-21 + 2u |s|max, the row sum relative (L + 4) u and the P.V sum (L + 4) u A_ic.
"""
import math

import numpy as np
import torch

U = 2.0 ** -24
LN2, LOG2E = math.log(2.0), 1.0 / math.log(2.0)
AKV = 64


# ---------------------------------------------------------------------------------------------------- plane representations
def h16_exp_dev(amax):
    """the exponent the kernels derive from a range slot (tc_common.cuh h16_exp_of): 0 for a zero / non-finite slot and for
    2^2 <= amax < 2^15 (no rescale), else e with amax 2^e in [2^14, 2^15) clamped to [-100, 100]"""
    amax = float(np.float32(amax))
    if not (amax > 0.0) or not math.isfinite(amax):
        return 0
    be = math.frexp(amax)[1] - 1
    if 2 <= be <= 14:
        return 0
    return min(max(14 - be, -100), 100)


def exp2i(e):
    """fp32 2^e clamped to the normal range, as the kernels' exp2i"""
    return 2.0 ** min(max(e, -126), 127)


def rep_h16(x, e, lo=True):
    """float64 value of the fp16 planes of float32 x at exponent e: (hi + lo) 2^-e, or hi 2^-e alone (one-term)"""
    sc = exp2i(e)
    xs = x.float() * sc
    hi = xs.half().float()
    if not lo:
        return hi.double() / sc
    return (hi.double() + (xs - hi).half().double()) / sc


def rn_tf32(x):
    """the kernels' TF32 rounding (bits + 0x1000) & 0xFFFFE000 of a float32 tensor, as float32"""
    b = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = ((b + 0x1000) & 0xFFFFE000) & 0xFFFFFFFF
    r = torch.where(r >= 2 ** 31, r - 2 ** 32, r)
    return r.to(torch.int32).view(torch.float32)


def rep_tf32(x):
    """float64 value of the TF32 planes hi = rn_tf32(x), lo = rn_tf32(x - hi)"""
    x = x.float()
    hi = rn_tf32(x)
    return hi.double() + rn_tf32(x - hi).double()


# ---------------------------------------------------------------------------------------------------- reference + bound
FORMATS = ('h16', 'one', 'tf32', 'generic')


def _consts(fmt, d, nb, L, ksplit):
    """(score accumulation factor, weight-factor slack per row w/o the |s|max term, P relative, P absolute, output relative to A,
    output relative to |O|) of the module docstring"""
    if fmt == 'generic':
        return (d + 4) * U, 2.0 ** -21, 2.0 ** -21 + (L + 4) * U, 0.0, (L + 4) * U, (L + 8) * U
    kstep = 8 if fmt == 'tf32' else 16
    terms = 1 if fmt == 'one' else 3
    n_qk = terms * -(-d // kstep)
    dropped = 0.0 if fmt == 'one' else 2.0 ** -22
    ds = dropped + (n_qk + 2) * 2 * U
    rho_p = {'h16': 2.0 ** -22, 'one': 2.0 ** -11, 'tf32': 2.0 ** -21}[fmt]
    abs_p = 2.0 ** -126 if fmt == 'tf32' else 2.0 ** -35
    n_pv = terms * (AKV // kstep) + 2
    out_a = dropped + n_pv * 2 * U + nb * 2 * U + (2 * U if ksplit else 0.0)
    out_o = (nb + 24 + (2 if ksplit else 0)) * U + 2 * U
    return ds, nb + 3, rho_p, abs_p, out_a, out_o


def reference(q, k, v, heads, scale, fmt, causal=False, qchunk=None):
    """float64 attention of q [B, N, C] over k, v [B, L, C] (already the represented operands, float64) and its bound's pieces.
    Returns (O [B, N, C], bound_arith [B, N, C]): the bound of the module docstring without the representation term."""
    B, N, C = q.shape
    L = k.shape[1]
    d = C // heads
    scale = float(np.float32(scale))
    nb = -(-L // AKV)
    ksplit = fmt in ('h16', 'one') and d > 80
    ds_f, n_corr, rho_p, abs_p, out_a, out_o = _consts(fmt, d, nb, L, ksplit)
    O = torch.empty(B, N, C, dtype=torch.float64, device=q.device)
    bnd = torch.empty_like(O)
    if qchunk is None:
        qchunk = max(1, min(N, (1 << 25) // max(1, B * L * 2)))
    for h in range(heads):
        cs = slice(h * d, (h + 1) * d)
        kh, vh = k[:, :, cs], v[:, :, cs]
        kabs, vabs = kh.abs(), vh.abs()
        for i0 in range(0, N, qchunk):
            qh = q[:, i0:i0 + qchunk, cs]
            s = scale * (qh @ kh.transpose(1, 2))                         # [B, n, L]
            t = qh.abs() @ kabs.transpose(1, 2)
            if causal:
                jj = torch.arange(L, device=q.device)
                ii = torch.arange(i0, i0 + qh.shape[1], device=q.device)
                mask = jj[None, :] > ii[:, None]
                s = s.masked_fill(mask, -math.inf)
                t = t.masked_fill(mask, 0.0)
            m = s.max(dim=-1, keepdim=True).values
            w = torch.exp(s - m)
            l = w.sum(dim=-1, keepdim=True)
            o = (w @ vh) / l
            A = (w @ vabs) / l
            F = vabs.sum(dim=1, keepdim=True) / l if abs_p else 0.0
            smax = s.masked_fill(torch.isinf(s), 0.0).abs().max(dim=-1, keepdim=True).values
            ds = scale * ds_f * t.max(dim=-1, keepdim=True).values
            if fmt == 'generic':
                D = ds + n_corr + 2 * U * smax
            else:
                D = ds + n_corr * (2.0 ** -21 + LN2 * 4 * U * (2 * smax * LOG2E + 10))
            b = torch.expm1(2 * D) * (A + o.abs()) + rho_p * A + abs_p * F + out_a * A + out_o * o.abs()
            O[:, i0:i0 + qh.shape[1], cs] = o
            bnd[:, i0:i0 + qh.shape[1], cs] = b
    return O, bnd


def represent(x, fmt, slot=None):
    """x (float32) as the planes of format fmt represent it (float64); slot: the range slot value its exponent comes from"""
    if fmt == 'tf32':
        return rep_tf32(x)
    if fmt == 'generic':
        return x.double()
    return rep_h16(x, h16_exp_dev(slot), lo=fmt == 'h16')


def bound(q, k, v, heads, scale, fmt, q_slot=None, kv_slot=None, causal=False):
    """(O64, O64r, bound) for float32 q [B, N, C], k, v [B, L, C]: bound = |O64r - O64| + the arithmetic bound on the represented
    operands (module docstring).  q_slot / kv_slot: the range slots whose exponents the fp16 planes of q and of k, v take."""
    O64, _ = reference(q.double(), k.double(), v.double(), heads, scale, 'generic', causal)
    qr, kr, vr = represent(q, fmt, q_slot), represent(k, fmt, kv_slot), represent(v, fmt, kv_slot)
    O64r, b = reference(qr, kr, vr, heads, scale, fmt, causal)
    return O64, O64r, (O64r - O64).abs() + b


# ---------------------------------------------------------------------------------------------------- CPU emulation
def emulate_online(q, k, v, heads, scale, fmt, ksplit=False, prescale=True):
    """float32 numpy emulation of the fused kernel's online algorithm on represented operands (float64 arrays q [N, C], k, v [L, C],
    one image): blocks of 64 keys, p = exp2(fma(s, scale log2e, 10 - m)), P split as fp16(p 2^10) hi + lo (one-term: hi) or TF32,
    O = O corr + P V_j, l = l corr + sum p; ksplit: even / odd blocks in two states merged at the end; prescale = False: P without the
    2^10.  Returns float64 [N, C]."""
    f32 = np.float32
    N, C = q.shape
    L = k.shape[0]
    d = C // heads
    nb = -(-L // AKV)
    sl = f32(f32(scale) * f32(LOG2E))
    pexp = f32(0.0 if fmt == 'tf32' or not prescale else 10.0)
    out = np.zeros((N, C))
    for h in range(heads):
        cs = slice(h * d, (h + 1) * d)
        qh, kh, vh = (a[:, cs].astype(f32) for a in (q, k, v))
        states = []
        for part in ((0, 1) if ksplit else (None,)):
            m = np.full((N, 1), -np.inf, f32)
            l = np.zeros((N, 1), f32)
            o = np.zeros((N, d), f32)
            for j in range(nb):
                if part is not None and j % 2 != part:
                    continue
                kb, vb = kh[j * AKV:(j + 1) * AKV], vh[j * AKV:(j + 1) * AKV]
                s = qh @ kb.T
                mx = (s.max(axis=1, keepdims=True) * sl).astype(f32)
                mn = np.maximum(m, mx)
                corr = np.exp2(m - mn).astype(f32)
                arg = (s.astype(np.float64) * sl + (pexp - mn)).astype(f32)
                p = np.exp2(arg).astype(f32)
                l = (l * corr + p.sum(axis=1, keepdims=True, dtype=f32)).astype(f32)
                m = mn
                if fmt == 'tf32':
                    ph = rn_tf32(torch.from_numpy(p)).numpy()
                    pl = (p - ph).astype(f32)
                    pr = ph + pl
                else:
                    ph = p.astype(np.float16).astype(f32)
                    pr = ph if fmt == 'one' else ph + (p - ph).astype(np.float16).astype(f32)
                o = (o * corr + pr @ vb).astype(f32)
            states.append((m, l, o))
        if ksplit:
            (m0, l0, o0), (m1, l1, o1) = states
            mm = np.maximum(m0, m1)
            c0, c1 = np.exp2(m0 - mm).astype(f32), np.exp2(m1 - mm).astype(f32)
            l, o = (l0 * c0 + l1 * c1).astype(f32), (o0 * c0 + o1 * c1).astype(f32)
        else:
            _, l, o = states[0]
        out[:, cs] = (o * (f32(1.0) / l)).astype(f32)
    return out
