"""CPU restatements and the float64 reference for the conv3x3 gather suite (tests/test_conv_gather_gpu.py), pinned on the CPU by
tests/test_conv_oracle_cpu.py.

Restatements of the host code in kernels_tc.cu / kernels_gemm.cu:
  conv_box     the pixel box {bw, bh, bn} (bw bh bn = 128) of one M tile of the tensor-core conv: the power-of-two rule when both
               output sides are powers of two, else conv_ragged_tile (fewest tiles, then the smallest halo, then the wider box), and
               the refusal of a box past TMA's 256-element limit (bw stride, bh stride, bn);
  tc_eligible  whether gemm_tc takes a conv3x3 (mode 1) or leaves it to the FFMA tiles;
  plan         gemm_tc's work partition (tile width w, split-K factor S) from its cost model, in 64-K blocks for the fp16-split
               operands and 32-K blocks otherwise;
  ffma_tile    the FFMA tiles' side (128 when the 128-tiles fill two waves and N > 64, else 64).

Reference.  conv64 is the conv in float64 of x [B, Hin, Win, Cin] (NHWC, as the engine holds it) with w [N, Cin, 3, 3]: the input
upsampled nearest-2x when up == 2, padded by `pad` pixels on the low sides and by one pixel on the high sides (OAI's symmetric pad 1;
pad 0 is the VAE's (0, 1, 0, 1) pad followed by an unpadded stride-2 conv), output [B, Hout, Wout] with Hout = (Hin up + pad - 2) //
stride + 1 unless given.  Input pixels outside [0, Hin up) x [0, Win up) read as zero.  It returns y [M, N] and
S[m, n] = sum_k |A(m, k)| |W(n, k)|, the same conv on |x| and |w|.

Error bound.  With u = 2^-24 and S as above, every kind below adds its parts, each a multiple of u S, plus the fp16-split floor.

  Operands.  fp16 split ('h16'): x' = x 2^e (e_a from A's range slot by the device rule h16_exp_dev, b_exp from the weights' range
  by the host rule), hi = fp16(x'), lo = fp16(x' - hi).  x' - hi is exact in fp32 and |x' - hi| <= 2^-11 |x'|; rounding it to fp16
  costs 2^-11 of that while lo is normal, so hi + lo keeps 22 bits: |x - (hi + lo) 2^-e| <= 2^-22 |x|.  The three terms
  lo.hi + hi.lo + hi.hi are the represented product minus lo.lo, and |lo_a lo_w| <= 2^-22 |a'| |w'|: 3 2^-22 |a| |w| per product.
  Once lo (or, one-term, hi) falls below fp16's normal range its error is half the subnormal spacing, 2^-25 absolute in the scaled
  space, which over the dot product is split_floor of gemm_epilogue_oracle.py (2^-25 (2^-e_a sum |w| + 2^-b_exp sum |a|)).
  One term ('h16_fast'): hi alone, 2^-11 per operand, (2^-10 + 2^-22) |a| |w| per product, and the same floor.
  TF32 ('ts'): hi = rn_tf32(x) (2^-11), lo = rn_tf32(x - hi) (2^-11 of |x - hi|): 3 2^-22 as for the fp16 split, no floor (the
  operands are not rescaled and fp32's subnormal spacing is negligible).
  Accumulation.  Products of fp16 (or TF32) planes are exact in fp32.  The tensor core adds each instruction's products into its
  fp32 accumulator with truncation: <= 2u of the running sum per instruction, plus two for the instruction's own alignment (the model
  of attention_oracle.py).  The accumulator restarts every chunk of 256 K (one chunk when the work item's K is <= 512), so a chunk of
  n instructions costs (n + 2) 2u of its own sum |terms|, and the chunks together (n_max + 2) 2u S.  An instruction covers 16 K
  (fp16, 3 or 1 terms) or 8 K (TF32, 3 terms): n_max = 48, 16 or 96 per 256-K chunk, twice that in a single 512-K chunk.  Each
  chunk's total is added to the fp32 sum with round-to-nearest, u of the running sum (<= S) per add.
  Split-K.  The partials are summed in fixed order in fp32, u S per add (S - 1 adds), then scaled by a power of two (exact).
  FFMA ('ffma'): one fp32 fma per K in order, the classic gamma_K = K u / (1 - K u) of S.

So |y_gpu - y| <= rel S + floor with rel = rep + (n_max + 2) 2u + (chunks per work item + splits - 1) u, padded by 2^-10 of itself
for the second-order terms.  It is far below the error of a dropped lo.hi term on operands whose lo planes have one sign (~2^-12 S)
and of a tap read one pixel off (a ninth of the terms replaced), which test_conv_oracle_cpu.py checks on the suite's shapes.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from tests.attention_oracle import h16_exp_dev, rn_tf32
from tests.gemm_epilogue_oracle import h16_exp, split_floor

U = 2.0 ** -24
TBM = 128
KINDS = ('h16', 'h16_fast', 'ts', 'ss')


def cdiv(a, b):
    return -(-a // b)


def pow2(v):
    return v > 0 and (v & (v - 1)) == 0


# ------------------------------------------------------------------------------------------------------------- restatements
def conv_ragged_tile(Wo, Ho, B, stride):
    """kernels_tc.cu conv_ragged_tile: (bw, bh, bn)"""
    best, box = None, None
    bw = TBM
    while bw >= 1:
        bh = TBM // bw
        while bh >= 1:
            bn = TBM // (bw * bh)
            if not (bw * stride > 256 or bh * stride > 256):
                tiles = cdiv(Wo, bw) * cdiv(Ho, bh) * cdiv(B, bn)
                halo = bn * (bw + 2) * (bh + 2)
                if best is None or (tiles, halo) < best:
                    best, box = (tiles, halo), (bw, bh, bn)
            bh //= 2
        bw //= 2
    return box


def conv_box(Ho, Wo, B, stride):
    """the M tile's pixel box and tile count: (bw, bh, bn, tiles_m), or None when gemm_tc refuses the box"""
    if pow2(Ho) and pow2(Wo):
        bw = Wo if Wo < 16 else 16
        bh = Ho if Ho < TBM // bw else TBM // bw
        bn = TBM // (bw * bh)
    else:
        bw, bh, bn = conv_ragged_tile(Wo, Ho, B, stride)
    if bn > 256 or bw * stride > 256 or bh * stride > 256:
        return None
    return bw, bh, bn, cdiv(Wo, bw) * cdiv(Ho, bh) * cdiv(B, bn)


def tc_eligible(M, N, Cin, Hin, Win, Hout, Wout, stride, up=1, lda=None, ldc=None, out_nchw=False):
    """gemm_tc's conditions for a conv3x3 (mode 1) with 16-byte aligned buffers; False: the FFMA tiles run it"""
    lda = Cin if lda is None else lda
    ldc = N if ldc is None else ldc
    if not out_nchw and (N % 4 or ldc % 4):
        return False
    if lda % 4 or M < 64 or (N < 32 and M < 2048):
        return False
    if stride not in (1, 2) or up != 1 or Cin % 32:
        return False
    if Hin != Hout * stride or Win != Wout * stride:
        return False
    return conv_box(Hout, Wout, M // (Hout * Wout), stride) is not None


def plan(M, N, K, tiles_m, kind, flags=0, sms=132):
    """gemm_tc's (tile width, split-K factor).  kind: 'h16' / 'h16_fast' (fp16 planes, 64-K blocks), 'ts' (TF32 planes) or 'ss'
    (raw fp32 B, 128-wide only); flags: 1 GEGLU / transposed planes, 2 NCHW store (no split-K for either)"""
    h16 = kind in ('h16', 'h16_fast')
    bk = 64 if h16 else 32
    num_kb = cdiv(K, bk)
    kc0, kc1 = (700.0, 6.0) if h16 else (400.0, 3.0)
    min_kbs = 4 if h16 else 8
    only128 = bool(flags & 1) or kind == 'ss'
    best, bw, bs = 1e30, 128, 1
    for w in (128, 64):
        if w == 64 and only128:
            break
        tn = cdiv(N, w)
        base = 0.0
        for S in range(1, 9):
            kbs = cdiv(num_kb, S)
            if S > 1 and (cdiv(num_kb, kbs) != S or kbs < min_kbs or flags or tiles_m * tn >= 4 * sms):
                continue
            cost = cdiv(tiles_m * tn * S, sms) * (kbs * (kc0 + kc1 * w) + 3000.0)
            if S == 1:
                base = cost
            else:
                cost += 4000.0 + (2.0 * S + 1.0) * M * N * 4.0 / 3e12 * 1.8e9
            if cost < best - 1e-9 and (S == 1 or cost < 0.9 * base):
                best, bw, bs = cost, w, S
    return bw, bs


def ffma_tile(M, N, sms=132):
    """the FFMA tiles' side"""
    return 128 if cdiv(M, 128) * cdiv(N, 128) >= 2 * sms and N > 64 else 64


def work_items(K, kind, splits):
    """K of each split's work item (32-K stages: the kernel's kb_per_split), in split order"""
    bk = 64 if kind in ('h16', 'h16_fast') else 32
    kbs = cdiv(cdiv(K, bk), splits) * bk
    return [min(kbs, K - s * kbs) for s in range(splits)]


def chunks(k_item):
    """K of each accumulation chunk of one work item: one chunk up to 512 K, else 256-K chunks"""
    if k_item <= 512:
        return [k_item]
    return [min(256, k_item - c) for c in range(0, k_item, 256)]


# ------------------------------------------------------------------------------------------------------------- reference
def out_size(Hin, stride, pad, up=1):
    return (Hin * up + pad - 2) // stride + 1


def im2col64(x, stride=1, pad=1, up=1, Hout=None, Wout=None):
    """[B, Hin, Win, C] -> float64 [B * Hout * Wout, 9 C], column k = tap * C + c (the kernels' K order), tap = 3 dy + dx"""
    x = x.double()
    if up != 1:
        x = x.repeat_interleave(up, 1).repeat_interleave(up, 2)
    B, Hl, Wl, C = x.shape
    Hout = out_size(Hl, stride, pad) if Hout is None else Hout
    Wout = out_size(Wl, stride, pad) if Wout is None else Wout
    hi_y = max(0, (Hout - 1) * stride + 3 - pad - Hl)
    hi_x = max(0, (Wout - 1) * stride + 3 - pad - Wl)
    xp = F.pad(x, (0, 0, pad, hi_x, pad, hi_y))
    cols = []
    for dy in range(3):
        for dx in range(3):
            cols.append(xp[:, dy:dy + (Hout - 1) * stride + 1:stride, dx:dx + (Wout - 1) * stride + 1:stride, :])
    return torch.cat(cols, -1).reshape(B * Hout * Wout, 9 * C)


def wmat(w):
    """OIHW [N, C, 3, 3] -> [N, 9 C] in the kernels' K order"""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)


def conv64(x, w, stride=1, pad=1, up=1, Hout=None, Wout=None):
    """(y, S) as float64 [M, N]: the conv and the same conv on |x|, |w| (module docstring)"""
    A = im2col64(x, stride, pad, up, Hout, Wout)
    W = wmat(w).double()
    return A @ W.t(), A.abs() @ W.abs().t()


# ------------------------------------------------------------------------------------------------------------- bound
def rel_bound(K, kind, splits=1):
    """the multiple of u S (as a plain factor of S) of the module docstring"""
    if kind == 'ffma':
        return K * U / (1 - K * U) * (1 + 2.0 ** -10)
    rep = {'h16': 3 * 2.0 ** -22, 'ts': 3 * 2.0 ** -22, 'h16_fast': 2.0 ** -10 + 2.0 ** -22}[kind]
    per16 = {'h16': 3, 'h16_fast': 1, 'ts': 6}[kind]                 # instructions per 16 K
    items = work_items(K, kind, splits)
    n_max = max(per16 * cdiv(c, 16) for k in items for c in chunks(k))
    adds = max(len(chunks(k)) for k in items)
    return (rep + (n_max + 2) * 2 * U + (adds + splits - 1) * U) * (1 + 2.0 ** -10)


def exponents(x, w, a_slot=None, w_range=0.0):
    """(e_a, b_exp) the fp16 planes take: A from its range slot (default: its true range) by the device rule, the weights by the
    host rule from max(w_range, max |w|)"""
    e_a = h16_exp_dev(float(x.abs().max()) if a_slot is None else a_slot)
    b_exp = h16_exp(max(w_range, float(w.abs().max())))
    return e_a, b_exp


def bound(S, a_abs_sum, w_abs_sum, K, kind, splits=1, e_a=0, b_exp=0):
    """elementwise bound [M, N] (float64): rel_bound S plus, for the fp16 kinds, the split floor"""
    b = rel_bound(K, kind, splits) * S
    if kind in ('h16', 'h16_fast'):
        b = b + split_floor(a_abs_sum, w_abs_sum, e_a, b_exp) * (1 + 2.0 ** -10)
    return b


# ------------------------------------------------------------------------------------------------------------- simulation
def planes(x, kind, e=0):
    """float64 (hi, lo) planes of float32 x as the kernels form them, in the scaled space (x 2^e for the fp16 kinds)"""
    x = x.float()
    if kind == 'ts':
        hi = rn_tf32(x)
        return hi.double(), rn_tf32(x - hi).double()
    xs = x * 2.0 ** e
    hi = xs.half().float()
    lo = (xs - hi).half().double() if kind == 'h16' else torch.zeros_like(xs, dtype=torch.float64)
    return hi.double(), lo


def rz32(v):
    """float64 -> the float32 value nearest to it towards zero (the tensor core's truncating add), as float64"""
    n = v.numpy()
    f = n.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(n)
    f = np.where(over, np.nextafter(f, np.float32(0)), f)
    return torch.from_numpy(f.astype(np.float64))


def rn32(v):
    return v.float().double()


def simulate(A, W, kind, splits=1, e_a=0, b_exp=0, drop=None):
    """float64 value of the fp32 result the tensor-core kernel computes for A [M, K] @ W [N, K]^T (float32): the kind's planes,
    three (one) product terms per K step in the kernel's order (lo.hi, hi.lo, hi.hi), each instruction's exact sum truncated into
    the chunk accumulator, chunks added to the total with round-to-nearest, split partials summed in order, then the exact
    power-of-two rescale.  drop='lohi' leaves out the hi_a.lo_w term (a broken kernel, to show the bound sees it)."""
    K = A.shape[1]
    if kind == 'ts':
        e_a = b_exp = 0
    ah, al = planes(A, kind, e_a)
    wh, wl = planes(W, kind, b_exp)
    step = 8 if kind == 'ts' else 16
    terms = [(ah, wh)] if kind == 'h16_fast' else [(al, wh), (ah, wl), (ah, wh)]
    if drop == 'lohi':
        terms = [t for t in terms if not (t[0] is ah and t[1] is wl)]
    parts = []
    k0 = 0
    for k_item in work_items(K, kind, splits):
        tot = torch.zeros(A.shape[0], W.shape[0], dtype=torch.float64)
        for c in chunks(k_item):
            acc = torch.zeros_like(tot)
            for k in range(k0, k0 + c, step):
                for a, w in terms:
                    acc = rz32(acc + a[:, k:k + step] @ w[:, k:k + step].t())
            tot = rn32(tot + acc)
            k0 += c
        parts.append(tot)
    y = parts[0]
    for p in parts[1:]:
        y = rn32(y + p)
    return y * 2.0 ** -(e_a + b_exp)


# ------------------------------------------------------------------------------------------------------------- operands
def lo_biased(x, e, g):
    """x moved onto fp16 grid value + 0.1 .. 0.45 of its fp16 spacing at exponent e (one sign for every lo plane), float32"""
    xs = x.double() * 2.0 ** e
    q = xs.float().half().double()
    mag = q.abs().clamp_min(2.0 ** -14)
    ulp = 2.0 ** (torch.floor(torch.log2(mag)) - 10)
    frac = 0.1 + 0.35 * torch.rand(x.shape, generator=g, dtype=torch.float64)
    return ((q + torch.sign(q) * frac * ulp) * 2.0 ** -e).float()


def operands(seed, B, Hin, Win, Cin, N, data='randn', a_scale=1.0, w_scale=1.0):
    """(x [B, Hin, Win, Cin], w [N, Cin, 3, 3]) float32.  data: 'randn' (signed); 'pos' (non-negative, every lo plane of one sign:
    constant-sign operands whose dropped lo.hi term adds up instead of cancelling); 'outlier' (randn with one input element 2^12
    larger)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Hin, Win, Cin, generator=g) * a_scale
    w = torch.randn(N, Cin, 3, 3, generator=g) * (w_scale / math.sqrt(9 * Cin))
    if data == 'pos':
        x, w = x.abs(), w.abs()
        x = lo_biased(x, h16_exp_dev(float(x.abs().max())), g)
        w = lo_biased(w, h16_exp(float(w.abs().max())), g)
    elif data == 'outlier':
        x[B // 2, Hin // 2, Win // 2, Cin // 2] = 4096.0 * a_scale
    return x, w


# ------------------------------------------------------------------------------------------------------------- the suite's geometries
class Case:
    """one conv of the GPU suite: x [B, Hin, Win, Cin] -> [B, Hout, Wout, N] (or NCHW), its operands from `operands`"""

    def __init__(self, name, B, Hin, Win, Cin, N, stride=1, pad=1, up=1, data='randn', nchw=False):
        self.name, self.B, self.Hin, self.Win, self.Cin, self.N = name, B, Hin, Win, Cin, N
        self.stride, self.pad, self.up, self.data, self.nchw = stride, pad, up, data, nchw
        self.Hout, self.Wout = out_size(Hin, stride, pad, up), out_size(Win, stride, pad, up)
        self.M, self.K = B * self.Hout * self.Wout, 9 * Cin

    def seed(self):
        return sum(map(ord, self.name)) * 7919

    def operands(self, **kw):
        return operands(self.seed(), self.B, self.Hin, self.Win, self.Cin, self.N, self.data, **kw)

    def tc(self, lda=None, ldc=None):
        return tc_eligible(self.M, self.N, self.Cin, self.Hin, self.Win, self.Hout, self.Wout, self.stride, self.up, lda, ldc, self.nchw)

    def box(self):
        return conv_box(self.Hout, self.Wout, self.B, self.stride)

    def plan(self, kind, sms=132):
        return plan(self.M, self.N, self.K, self.box()[3], kind, 2 if self.nchw else 0, sms)


SUITE = [
    # power-of-two maps (box by the pow2 rule), B a multiple of bn and not
    Case('1x1_b130', 130, 1, 1, 32, 36), Case('1x1_b128', 128, 1, 1, 64, 100),
    Case('1x2_b100', 100, 1, 2, 32, 36), Case('1x8_b24', 24, 1, 8, 32, 36),
    Case('2x2_b20', 20, 2, 2, 32, 36), Case('2x2_b32', 32, 2, 2, 96, 100),
    Case('4x4_b9', 9, 4, 4, 32, 100), Case('4x4_b16', 16, 4, 4, 64, 36),
    Case('8x8_b3', 3, 8, 8, 96, 100), Case('8x8_b4', 4, 8, 8, 32, 36),
    Case('16x16_b1', 1, 16, 16, 64, 100), Case('16x16_b3', 3, 16, 16, 32, 36),
    Case('4x64_b3', 3, 4, 64, 32, 36), Case('4x64_b2', 2, 4, 64, 64, 100), Case('64x4_b3', 3, 64, 4, 32, 36),
    # ragged maps (conv_ragged_tile): tiles overhang x and y, and the batch with them
    Case('3x5_b5', 5, 3, 5, 32, 36), Case('7x7_b3', 3, 7, 7, 64, 100), Case('6x10_b2', 2, 6, 10, 96, 36),
    Case('9x15_b1', 1, 9, 15, 32, 36), Case('12x20_b2', 2, 12, 20, 32, 100), Case('24x40_b1', 1, 24, 40, 64, 36),
    Case('40x24_b1', 1, 40, 24, 32, 36), Case('10x80_b1', 1, 10, 80, 32, 36), Case('1x40_b5', 5, 1, 40, 32, 36),
    Case('40x1_b5', 5, 40, 1, 32, 36), Case('1x100_b3', 3, 1, 100, 32, 36), Case('96x96_b1', 1, 96, 96, 32, 36),
    # stride 2, pad 1 (OAI Downsample) and pad 0 (the VAE's (0, 1, 0, 1) pad): every box side, up to bw 2 = 256 and bh 2 = 256
    Case('s2_1x1_b70', 70, 2, 2, 32, 36, 2), Case('s2_1x2_b40', 40, 2, 4, 32, 36, 2, 0), Case('s2_1x8_b12', 12, 2, 16, 32, 36, 2),
    Case('s2_2x2_b20', 20, 4, 4, 32, 36, 2, 0), Case('s2_4x4_b5', 5, 8, 8, 32, 100, 2), Case('s2_4x8_b3', 3, 8, 16, 32, 36, 2, 0),
    Case('s2_8x8_b2', 2, 16, 16, 32, 36, 2), Case('s2_8x8_b3_p0', 3, 16, 16, 64, 100, 2, 0), Case('s2_16x16_b1', 1, 32, 32, 32, 36, 2),
    Case('s2_4x100_b3', 3, 8, 200, 32, 36, 2), Case('s2_1x40_b3', 3, 2, 80, 32, 36, 2, 0), Case('s2_1x80_b9', 9, 2, 160, 32, 36, 2),
    Case('s2_80x1_b9', 9, 160, 2, 32, 36, 2, 0), Case('s2_48x80', 1, 96, 160, 32, 36, 2), Case('s2_48x80_p0', 1, 96, 160, 32, 36, 2, 0),
    Case('s2_24x40_b2', 2, 48, 80, 64, 36, 2), Case('s2_24x40_b2_p0', 2, 48, 80, 64, 100, 2, 0),
    # wide N, both tile widths, and split-K S = 2 .. 8; Cin 320 / 1280 / 1920 (K 11520 / 17280), odd multiples of 32
    Case('n4_m2304', 1, 48, 48, 32, 4), Case('n320_16x16_b4', 4, 16, 16, 64, 320), Case('n640_7x7_b4', 4, 7, 7, 96, 640),
    Case('n1280_3x5_b33', 33, 3, 5, 96, 1280), Case('k3_n1280_3x5_b5', 5, 3, 5, 96, 1280, data='pos'),
    Case('k2_16x16_b23', 23, 16, 16, 320, 36, data='pos'), Case('k4_2x2_b16', 16, 2, 2, 96, 36), Case('k5_6x10_b33', 33, 6, 10, 320, 36, data='pos'),
    Case('k6_3x5_b5', 5, 3, 5, 320, 640, data='pos'), Case('k7_3x5_b33', 33, 3, 5, 320, 100, data='pos'),
    Case('k8_2x2_b16', 16, 2, 2, 320, 36, data='pos'), Case('k_c1280_2x2_b16', 16, 2, 2, 1280, 36, data='pos'),
    Case('k_c1920_4x4_b4', 4, 4, 4, 1920, 100, data='pos'), Case('k_c1920_3x5_b9', 9, 3, 5, 1920, 320, data='pos'),
    Case('outlier_12x20_b2', 2, 12, 20, 320, 100, data='outlier'),
    # NCHW final store (any N) on the tensor cores (M >= 2048) and the FFMA tiles
    Case('nchw_n3', 2, 32, 32, 32, 3, nchw=True), Case('nchw_n4', 2, 32, 32, 32, 4, nchw=True), Case('nchw_n6_24x40', 3, 24, 40, 32, 6, nchw=True),
    Case('nchw_n3_small', 1, 12, 20, 32, 3, nchw=True),
    # FFMA-only gathers: few-channel inputs (scalar gather), stride 2 with Hin != 2 Hout, the nearest-2x fold
    Case('c3_16x16_b2', 2, 16, 16, 3, 36), Case('c4_12x20_b2', 2, 12, 20, 4, 100), Case('c20_7x7_b3', 3, 7, 7, 20, 36),
    Case('s2_odd_9x15', 2, 9, 15, 32, 36, 2), Case('s2_odd_9x15_p0', 2, 9, 15, 64, 36, 2, 0),
    Case('up2_8x8_b2', 2, 8, 8, 32, 36, up=2), Case('up2_6x10', 1, 6, 10, 64, 100, up=2), Case('up2_c4_5x3', 3, 5, 3, 4, 36, up=2),
]
