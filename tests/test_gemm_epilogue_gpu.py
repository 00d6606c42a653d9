"""The GEMM epilogue, term by term, on every route and work partition, through the production gemm() (cdx_op_gemm).

Epilogue isolation.  The planner's cache key and cost model do not look at the bias, the row vector, the residual, the range and
statistics slots or the split of A into two sources, so a "plain" run (no epilogue term) and a "full" run of the same M, N, K, data
and operand exponents run the same plan -- each case asserts that from the plan the hook reports -- and produce bitwise-equal
accumulators (the mainloop and the split-K reduce are deterministic).  Every epilogue then adds in fp32 in a fixed order
(tensor-core epilogue: alpha * tot + bias, + row vector, + residual; split-K reduce: the fixed-order split sum, * alpha, + bias, ...;
FFMA tiles: alpha * acc, + bias, ...).  alpha is a power of two here (the fp16 rescale 2^-e_a 2^-b_exp included), so whether or not
the first step is contracted into an FMA, the full run equals ((plain + bias) + rowvec) + residual evaluated in fp32 on the CPU,
exactly.  The same argument gives the other exact identities: a two-source A equals the one-source GEMM over the materialised concat;
TF32 planes are rn_tf32 of the plain values; V^T planes are their transpose; the NCHW store is a permutation; the range slot is the
max |stored value|.  GEGLU is checked against v * gelu(g) of the plain run's columns with the bound derived in
tests/gemm_epilogue_oracle.py.

Every plain run is also checked against a float64 reference of the whole operation under the per-op budget of
test_gemm_ring_gpu.py (2e-5 of the result's range for the faithful modes, 5e-3 for the one-term fp16 mode 4), plus the fp16-split
floor of the oracle's docstring in the fp16 modes.  Every output buffer sits inside guard rows, guard columns and the padding
between N and its stride, all filled with a NaN sentinel that must come back bitwise untouched, and every call runs twice with
bitwise-equal outputs and slots.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.gemm_epilogue_oracle import geglu_bound, geglu_ref, h16_exp, split_floor, tf32_planes

pytestmark = pytest.mark.gpu

MODES = (0, 1, 3, 4)
KIND = {0: 'ffma', 1: 'h16', 3: 'ts', 4: 'h16_fast'}
BUDGET = {0: 2e-5, 1: 2e-5, 3: 2e-5, 4: 5e-3}
SENTINEL = 0x7FC0BEEF         # a quiet NaN with a payload no kernel writes
GUARD_ROWS = 2


@pytest.fixture(scope='module')
def engines():
    from cycle_diffusion_b200.engine import Engine
    es = {}
    for m in MODES:
        es[m] = Engine(0)
        es[m].set_mma_mode(m)
    return es


# ------------------------------------------------------------------------------------------------------------- buffers
class Out:
    """an output of `rows` x `cols` at row stride ld inside guard rows and the [cols, ld) padding, all NaN-sentinel filled"""

    def __init__(self, rows, cols, ld, dtype=torch.float32):
        assert ld >= cols
        self.rows, self.cols, self.ld = rows, cols, ld
        self.pre = GUARD_ROWS * ld - GUARD_ROWS * ld % 4       # at least one guard row; the view stays 16-byte aligned
        self.store = torch.empty(self.pre + rows * ld + GUARD_ROWS * ld + 4, dtype=dtype, device='cuda')
        inside = torch.zeros(self.store.numel(), dtype=torch.bool)
        idx = self.pre + torch.arange(rows)[:, None] * ld + torch.arange(cols)[None, :]
        inside[idx.reshape(-1)] = True
        self.outside = ~inside
        self.view = self.store[self.pre:self.pre + rows * ld].view(rows, ld)[:, :cols]

    def fill(self):
        self.store.view(torch.int32).fill_(SENTINEL)

    def guards_ok(self):
        return bool((self.store.view(torch.int32).cpu()[self.outside] == SENTINEL).all())

    def get(self):
        return self.view.cpu().clone()


class Slot:
    """a device float range slot (c_amax), starting at 0, between two sentinel neighbours"""

    def __init__(self, init=0.0):
        self.init = init
        self.store = torch.empty(3, dtype=torch.float32, device='cuda')
        self.view = self.store[1:2]

    def fill(self):
        self.store.view(torch.int32).fill_(SENTINEL)
        self.view.fill_(self.init)

    def guards_ok(self):
        s = self.store.view(torch.int32).cpu()
        return int(s[0]) == SENTINEL and int(s[2]) == SENTINEL

    def get(self):
        return float(self.view.cpu())


def run(eng, outs, **fields):
    """op_gemm twice with the outputs `outs` (name -> Out / Slot); guards intact, both runs bitwise equal.  -> ({name: cpu}, plan)"""
    results = []
    for _ in range(2):
        for o in outs.values():
            o.fill()
        plan = eng.op_gemm(**fields, **{k: o.view for k, o in outs.items()})
        torch.cuda.synchronize()
        for k, o in outs.items():
            assert o.guards_ok(), f'{k}: a write landed outside the output'
        results.append(({k: o.get() for k, o in outs.items()}, plan))
    (r1, p1), (r2, p2) = results
    assert p1 == p2
    for k in r1:
        a, b = r1[k], r2[k]
        same = a == b if isinstance(a, float) else torch.equal(a.view(torch.int32), b.view(torch.int32))
        assert same, f'{k}: two runs of the same call differ'
    return r1, p1


def plan_key(p):
    return (p['kind'], p['width'], p['splits'])


def check_plan(p, mode, want):
    """the route this case claims: the mode's operand kind (or the FFMA tiles) and a (width, split?) from `want`"""
    kind = want.get('kind', KIND[mode])
    assert p['kind'] == kind, f'expected the {kind} route, ran {p}'
    if 'wS' in want:
        assert (p['width'], p['splits'] > 1) in want['wS'], f'expected one of {want["wS"]} (width, split), ran {p}'
    print(f'plan mode {mode}: {p["kind"]} w{p["width"]} S{p["splits"]}')


def bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def gen(seed):
    return torch.Generator().manual_seed(seed)


def amax_of(x):
    return float(x.abs().max()) if x.numel() else 0.0


# ------------------------------------------------------------------------------------------------------------- operands
class Problem:
    """A dense ([M, K] rows, optional second source) or conv3x3 (NHWC) contraction with CPU copies of everything and the float64
    product.  Device copies of A sit in wider row buffers when lda > K (A a column slice)."""

    def __init__(self, seed, M=None, K=None, N=None, conv=None, C2=0, lda_pad=0, a_scale=1.0, a2_scale=1.0, w=None):
        g = gen(seed)
        self.conv = conv
        if conv:
            B, H, W, Cin, stride = conv
            self.B, self.H, self.W, self.Cin, self.stride = B, H, W, Cin, stride
            self.Ho, self.Wo = H // stride, W // stride
            self.M, self.K, self.N = B * self.Ho * self.Wo, 9 * Cin, N
            self.C1, self.C2 = Cin, 0
            self.lda = Cin + lda_pad
            self.x = torch.randn(B, H, W, Cin, generator=g) * a_scale
            self.w = torch.randn(N, Cin, 3, 3, generator=g) / math.sqrt(9 * Cin) if w is None else w
            xb = torch.zeros(B, H, W, self.lda)
            xb[..., :Cin] = self.x
            self.A_dev = xb.cuda()
            self.A2_dev = None
            x64 = self.x.double().permute(0, 3, 1, 2)
            y = F.conv2d(x64, self.w.double(), stride=stride, padding=1)
            self.y64 = y.permute(0, 2, 3, 1).reshape(self.M, N)
            asum = F.conv2d(x64.abs(), torch.ones(1, Cin, 3, 3, dtype=torch.float64), stride=stride, padding=1)
            self.a_abs_sum = asum.permute(0, 2, 3, 1).reshape(self.M)
            self.w_abs_sum = self.w.double().abs().reshape(N, -1).sum(1)
            self.a_amax = amax_of(self.x)
            self.rows_per_img = self.Ho * self.Wo
        else:
            self.M, self.K, self.N = M, K, N
            self.C1, self.C2 = K - C2, C2
            self.lda = self.C1 + lda_pad
            a1 = torch.randn(M, self.C1, generator=g) * a_scale
            a2 = torch.randn(M, C2, generator=g) * a2_scale if C2 else torch.zeros(M, 0)
            self.a = torch.cat([a1, a2], 1)
            self.w = torch.randn(N, K, generator=g) / math.sqrt(K) if w is None else w
            ab = torch.zeros(M, self.lda)
            ab[:, :self.C1] = a1
            self.A_dev = ab.cuda()
            self.A2_dev = a2.cuda() if C2 else None
            self.y64 = self.a.double() @ self.w.double().t()
            self.a_abs_sum = self.a.double().abs().sum(1)
            self.w_abs_sum = self.w.double().abs().sum(1)
            self.a_amax = amax_of(self.a)
            self.a1_amax, self.a2_amax = amax_of(a1), amax_of(a2)
        self.w_dev = self.w.cuda()

    def fields(self):
        f = dict(M=self.M, N=self.N, K=self.K, A=self.A_dev, lda=self.lda, C1=self.C1, w=self.w_dev)
        if self.conv:
            f.update(mode=1, Hin=self.H, Win=self.W, Hout=self.Ho, Wout=self.Wo, stride=self.stride, pad=1)
        else:
            f.update(mode=0, ldb=self.K)
            if self.C2:
                f.update(A2=self.A2_dev, lda2=self.C2, C2=self.C2)
        return f

    def check_whole(self, y, mode, extra=None, a_range=None, w_range=None, alpha=1.0):
        """the plain result against float64: per-op budget of the result's range, plus the fp16-split floor in the fp16 modes"""
        ref = alpha * self.y64 + (extra if extra is not None else 0.0)
        err = (y.double() - ref).abs()
        bound = BUDGET[mode] * float(ref.abs().max())
        if mode in (1, 4):
            e_a = h16_exp(a_range if a_range is not None else self.a_amax)
            b_exp = h16_exp(max(w_range or 0.0, float(self.w.abs().max())))
            bound = bound + alpha * split_floor(self.a_abs_sum, self.w_abs_sum, e_a, b_exp)
        ratio = float((err / bound).max())
        print(f'  whole result vs float64: worst error / bound {ratio:.3f}')
        assert ratio <= 1.0
        return ratio


def f32_add(*terms):
    """left-to-right fp32 sum"""
    out = terms[0].float().clone()
    for t in terms[1:]:
        out = out + t.float()
    return out


# ------------------------------------------------------------------------------------------------------------- 1. bias / rowvec / residual
# (name, problem kwargs, ldc pad, ldr pad, images (rows per image), plan wanted per mode); several images per tile and ragged M / N
DENSE = [
    ('hw81_w64', dict(M=81 * 5, K=320, N=200, lda_pad=12), 4, 8, 81, {1: {(64, False)}, 3: {(64, False)}, 4: {(64, False)}, 0: {(64, False)}}),
    ('hw200_w64', dict(M=200 * 9, K=256, N=324, lda_pad=4), 8, 4, 200, {1: {(64, False)}, 3: {(64, False)}, 4: {(64, False)}, 0: {(64, False)}}),
    ('hw576_w128', dict(M=576 * 8, K=320, N=1152), 4, 12, 576, {1: {(128, False)}, 3: {(128, False)}, 4: {(128, False)}, 0: {(128, False)}}),
    ('splitk_w64', dict(M=200, K=6400, N=324, lda_pad=4), 4, 8, 81, {1: {(64, True)}, 3: {(64, True)}, 4: {(64, True)}, 0: {(64, False)}}),
    ('splitk_w128', dict(M=256, K=5120, N=2560), 0, 4, 81, {1: {(128, True)}, 3: {(128, True)}, 4: {(128, True)}, 0: {(64, False)}}),
]
# conv: (name, (B, H, W, Cin, stride), Cout, ldc pad, ldr pad, plan wanted)
CONV = [
    ('8x8_b5', (5, 8, 8, 64, 1), 96, 4, 8, {1: {(64, False)}, 3: {(64, False)}, 4: {(64, False)}, 0: {(64, False)}}),
    ('24x40', (3, 24, 40, 64, 1), 100, 0, 4, {1: {(64, False)}, 3: {(64, False)}, 4: {(64, False)}, 0: {(64, False)}}),
    ('8x8_splitk', (6, 8, 8, 320, 1), 320, 4, 0, {1: {(64, True)}, 3: {(64, True)}, 4: {(64, True)}, 0: {(64, False)}}),
    ('8x8_splitk_w128', (9, 8, 8, 640, 1), 640, 0, 4, {1: {(128, True)}, 3: {(128, True)}, 4: {(128, True)}, 0: {(64, False)}}),
    ('16x16_s2_splitk', (3, 16, 16, 96, 2), 160, 4, 4, {1: {(64, True)}, 3: {(64, True)}, 4: {(64, True)}, 0: {(64, False)}}),
]
TERMS = ['bias', 'rowvec', 'residual', 'all', 'cancel']


def epilogue_terms(p, seed, rows_per_img, ldr_pad, which):
    """bias per column, a distinct row vector per image far from the bias, a residual at another scale; 'cancel': bias and a
    residual of -(A W^T + bias) rounded to fp32, so the outputs cancel to near zero"""
    g = gen(seed + 1)
    imgs = -(-p.M // rows_per_img)
    bias = torch.randn(p.N, generator=g) * 3.0
    rowvec = (torch.arange(imgs, dtype=torch.float32)[:, None] + 1.0) * 100.0 + torch.randn(imgs, p.N, generator=g)
    residual = torch.randn(p.M, p.N + ldr_pad, generator=g) * 1e-3
    if which == 'cancel':
        residual[:, :p.N] = (-(p.y64 + bias.double()[None, :])).float()
    t = {}
    if which in ('bias', 'all', 'cancel'):
        t['bias'] = bias
    if which in ('rowvec', 'all'):
        t['rowvec'] = rowvec
    if which in ('residual', 'all', 'cancel'):
        t['residual'] = residual
    return t


def identity_case(eng, mode, p, rows_per_img, ldc_pad, ldr_pad, which, want, seed):
    ldc = p.N + ldc_pad
    slot = Slot()
    plain, pp = run(eng, {'C': Out(p.M, p.N, ldc), 'c_amax': slot}, **p.fields(), ldc=ldc)
    check_plan(pp, mode, want)
    p.check_whole(plain['C'], mode)
    assert plain['c_amax'] == float(plain['C'].abs().max())
    t = epilogue_terms(p, seed, rows_per_img, ldr_pad, which)
    f = p.fields()
    f.update(ldc=ldc, rows_per_batch=rows_per_img)
    if 'bias' in t:
        f['bias'] = t['bias'].cuda()
    if 'rowvec' in t:
        f.update(rowvec=t['rowvec'].cuda(), ld_rowvec=p.N)
    if 'residual' in t:
        f.update(residual=t['residual'].cuda(), ldr=p.N + ldr_pad)
    full, pf = run(eng, {'C': Out(p.M, p.N, ldc), 'c_amax': Slot()}, **f)
    assert plan_key(pf) == plan_key(pp), f'plain and full runs took different plans: {pp} vs {pf}'
    img = torch.arange(p.M) // rows_per_img
    exp = [plain['C']]
    if 'bias' in t:
        exp.append(t['bias'][None, :].expand(p.M, p.N))
    if 'rowvec' in t:
        exp.append(t['rowvec'][img])
    if 'residual' in t:
        exp.append(t['residual'][:, :p.N])
    want_c = f32_add(*exp)
    assert bits_equal(full['C'], want_c), f'{which}: {int((full["C"] != want_c).sum())} elements differ from the plain run + terms'
    assert full['c_amax'] == float(want_c.abs().max())


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('which', TERMS)
@pytest.mark.parametrize('case', DENSE, ids=[c[0] for c in DENSE])
def test_dense_epilogue_identity(engines, mode, which, case):
    name, kw, ldc_pad, ldr_pad, hw, want = case
    seed = sum(map(ord, name + which))
    p = Problem(seed, **kw)
    identity_case(engines[mode], mode, p, hw, ldc_pad, ldr_pad, which, {'wS': want[mode]}, seed)


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('which', ['all', 'rowvec', 'cancel'])
@pytest.mark.parametrize('case', CONV, ids=[c[0] for c in CONV])
def test_conv_epilogue_identity(engines, mode, which, case):
    name, geo, N, ldc_pad, ldr_pad, want = case
    seed = sum(map(ord, name + which))
    p = Problem(seed, conv=geo, N=N)
    identity_case(engines[mode], mode, p, p.rows_per_img, ldc_pad, ldr_pad, which, {'wS': want[mode]}, seed)


# mode-1 shapes the tensor cores do not take: M < 64, N % 4 != 0, N < 32 with small M, lda % 4 != 0
FALLBACKS = [('m_lt_64', dict(M=48, K=320, N=128), 0), ('n_mod4', dict(M=512, K=320, N=130), 2), ('n_lt_32', dict(M=512, K=256, N=24), 0),
             ('lda_mod4', dict(M=512, K=320, N=128, lda_pad=2), 0)]


@pytest.mark.parametrize('case', FALLBACKS, ids=[c[0] for c in FALLBACKS])
@pytest.mark.parametrize('which', ['all', 'cancel'])
def test_mode1_fallback_identity(engines, case, which):
    name, kw, ldc_pad = case
    seed = sum(map(ord, name + which))
    p = Problem(seed, **kw)
    identity_case(engines[1], 1, p, 81, ldc_pad, 4, which, {'kind': 'ffma'}, seed)


def test_splitk_bias_any_alignment(engines):
    """A bias at a 4-byte offset on a split-K shape: it runs (the reduce loads the bias by scalar) and matches the aligned bias."""
    eng = engines[1]
    p = Problem(77, M=200, K=6400, N=324)
    bias = torch.randn(p.N, generator=gen(78))
    aligned = bias.cuda()
    store = torch.empty(p.N + 4, device='cuda')
    store[1:1 + p.N] = aligned
    off = store[1:1 + p.N]
    assert off.data_ptr() % 16 == 4
    ra, pa = run(eng, {'C': Out(p.M, p.N, p.N), 'c_amax': Slot()}, **p.fields(), ldc=p.N, bias=aligned)
    ro, po = run(eng, {'C': Out(p.M, p.N, p.N), 'c_amax': Slot()}, **p.fields(), ldc=p.N, bias=off)
    check_plan(pa, 1, {'wS': {(64, True)}})
    assert plan_key(pa) == plan_key(po)
    assert bits_equal(ra['C'], ro['C']) and ra['c_amax'] == ro['c_amax']


# ------------------------------------------------------------------------------------------------------------- 2. two sources
# (name, M, C1, C2, N, modes): C1 an odd multiple of 32 (the source boundary inside a 64-K planner block), the 1920-channel skip
# conv (1280 + 640), and for the FFMA tiles C1 % 4 == 0 but not a multiple of 32
TWO_SOURCE = [('c1_96', 512, 96, 224, 320, (1, 3, 4, 0)), ('c1_160', 1024, 160, 160, 320, (1, 3, 4, 0)),
              ('skip1920', 256, 1280, 640, 640, (1, 3, 4, 0)), ('c1_36_ffma', 512, 36, 92, 200, (0,))]


@pytest.mark.parametrize('case', TWO_SOURCE, ids=[c[0] for c in TWO_SOURCE])
@pytest.mark.parametrize('tracked', [False, True])
def test_two_source_equals_concat(engines, case, tracked):
    name, M, C1, C2, N, modes = case
    for mode in modes:
        eng = engines[mode]
        p = Problem(C1 + C2, M=M, K=C1 + C2, N=N, C2=C2, a_scale=1e-3, a2_scale=1e2)      # ranges 1e5 apart
        f = p.fields()
        bias = torch.randn(N, generator=gen(5)).cuda()
        slots = {}
        if tracked:
            slots = dict(a_amax=torch.tensor([p.a1_amax], device='cuda'), a2_amax=torch.tensor([p.a2_amax], device='cuda'))
        two, pt = run(eng, {'C': Out(M, N, N), 'c_amax': Slot()}, **f, ldc=N, bias=bias, **slots)
        cat = Problem(C1 + C2, M=M, K=C1 + C2, N=N, w=p.w)
        cat.A_dev = p.a.cuda()
        cat.a = p.a
        fc = cat.fields()
        one_slot = dict(a_amax=torch.tensor([p.a_amax], device='cuda')) if tracked else {}
        one, po = run(eng, {'C': Out(M, N, N), 'c_amax': Slot()}, **fc, ldc=N, bias=bias, **one_slot)
        check_plan(pt, mode, {})
        assert plan_key(pt) == plan_key(po), f'two-source and concat took different plans: {pt} vs {po}'
        assert bits_equal(two['C'], one['C']), f'mode {mode}: two-source result differs from the concat'
        assert two['c_amax'] == one['c_amax'] == float(one['C'].abs().max())
        p.check_whole(one['C'], mode, extra=bias.cpu().double()[None, :])


# ------------------------------------------------------------------------------------------------------------- 3. GEGLU
def interleaved_weights(N, K, seed):
    return torch.randn(N, K, generator=gen(seed)) / math.sqrt(K)


# (name, mode, M, K, N, ldc pad, route wanted): the tensor-core epilogue (its own plan: 128-wide, no split, which the plain run
# must share), the mode-0 fallback (a temporary + geglu_kernel) and a mode-1 shape the tensor cores do not take (M < 64)
GEGLU = [('tc_1152', 1, 4608, 320, 1152, 0, 'h16'), ('tc_1152_ldc', 1, 4608, 320, 1152, 8, 'h16'), ('tc_ts', 3, 4608, 320, 1152, 4, 'ts'),
         ('tc_fast', 4, 4608, 320, 1152, 0, 'h16_fast'), ('ffma_1280', 0, 300, 160, 1280, 0, 'ffma'), ('mode1_m48', 1, 48, 320, 256, 0, 'ffma')]


@pytest.mark.parametrize('case', GEGLU, ids=[c[0] for c in GEGLU])
def test_geglu(engines, case):
    name, mode, M, K, N, ldc_pad, kind = case
    eng = engines[mode]
    p = Problem(N + M, M=M, K=K, N=N, w=interleaved_weights(N, K, N))
    bias = torch.randn(N, generator=gen(3)).cuda()
    plain, pp = run(eng, {'C': Out(M, N, N)}, **p.fields(), ldc=N, bias=bias)
    p.check_whole(plain['C'], mode, extra=bias.cpu().double()[None, :])
    ldc = N // 2 + ldc_pad
    full, pf = run(eng, {'C': Out(M, N // 2, ldc), 'c_amax': Slot()}, **p.fields(), ldc=ldc, bias=bias, geglu=1)
    check_plan(pf, mode, {'kind': kind})
    if kind != 'ffma':
        assert plan_key(pf) == plan_key(pp) == (kind, 128, 1), f'GEGLU and its plain run: {pf} vs {pp}'
    o64, v, g = geglu_ref(plain['C'])
    ratio = float(((full['C'].double() - o64).abs() / (geglu_bound(v, g) + 1e-300)).max())
    print(f'  GEGLU vs v * gelu(g) of the plain run: worst error / bound {ratio:.3f}')
    assert ratio <= 1.0
    assert full['c_amax'] == float(full['C'].abs().max())


def test_geglu_fallback_rejects_strided_output(engines):
    eng = engines[0]
    p = Problem(9, M=256, K=160, N=256, w=interleaved_weights(256, 160, 9))
    out = Out(256, 128, 136)
    out.fill()
    with pytest.raises(AssertionError, match='GEGLU output must be dense'):
        eng.op_gemm(**p.fields(), C=out.view, ldc=136, geglu=1)
    assert out.guards_ok()


def test_geglu_n_not_128_multiple_is_rejected(engines):
    """GEGLU is fused on the tensor cores for N % 128 == 0 only, and its fallback needs the same: anything else is an error"""
    p = Problem(10, M=512, K=320, N=192, w=interleaved_weights(192, 320, 10))
    with pytest.raises(AssertionError, match='bad GEGLU problem'):
        engines[1].op_gemm(**p.fields(), C=Out(512, 96, 96).view, ldc=96, geglu=1)


# ------------------------------------------------------------------------------------------------------------- 4. planes
PLANES = [('tc_w64', 1, dict(M=648, K=320, N=200)), ('tc_w128', 1, dict(M=4608, K=320, N=1152)), ('splitk', 1, dict(M=200, K=6400, N=324)),
          ('ts', 3, dict(M=648, K=320, N=200)), ('ts_splitk', 3, dict(M=256, K=5120, N=2560)), ('fast', 4, dict(M=648, K=320, N=200)),
          ('ffma_split_planes', 0, dict(M=300, K=160, N=200)), ('mode1_m48', 1, dict(M=48, K=320, N=128))]


@pytest.mark.parametrize('case', PLANES, ids=[c[0] for c in PLANES])
def test_tf32_planes(engines, case):
    name, mode, kw = case
    eng = engines[mode]
    p = Problem(kw['M'] + kw['N'], **kw)
    bias = torch.randn(p.N, generator=gen(4)).cuda()
    plain, pp = run(eng, {'C': Out(p.M, p.N, p.N)}, **p.fields(), ldc=p.N, bias=bias)
    p.check_whole(plain['C'], mode, extra=bias.cpu().double()[None, :])
    full, pf = run(eng, {'C': Out(p.M, p.N, p.N), 'C_lo': Out(p.M, p.N, p.N), 'c_amax': Slot()}, **p.fields(), ldc=p.N, bias=bias)
    assert plan_key(pf) == plan_key(pp)
    check_plan(pf, mode, {'kind': 'ffma'} if name == 'mode1_m48' else {})
    hi, lo = tf32_planes(plain['C'])
    assert bits_equal(full['C'], hi) and bits_equal(full['C_lo'], lo)
    assert full['c_amax'] == float(hi.abs().max())


# q|k|v in one call: q|k columns as TF32 planes, v columns (n >= t_col0) transposed to Ct[(n - t_col0) * ldt + m], ldt > M
QKV = [('qkv_320', 1, 4096, 320, 960, 640, 64), ('qkv_ts', 3, 4096, 320, 960, 640, 36), ('qkv_fast', 4, 2048, 640, 1920, 1280, 8)]


@pytest.mark.parametrize('case', QKV, ids=[c[0] for c in QKV])
def test_transposed_planes(engines, case):
    name, mode, M, K, N, t0, ldt_pad = case
    eng = engines[mode]
    p = Problem(M + N, M=M, K=K, N=N)
    plain, pp = run(eng, {'C': Out(M, N, N)}, **p.fields(), ldc=N)
    p.check_whole(plain['C'], mode)
    ldt = M + ldt_pad
    outs = {'C': Out(M, t0, N), 'C_lo': Out(M, t0, N), 'Ct_hi': Out(N - t0, M, ldt), 'Ct_lo': Out(N - t0, M, ldt), 'c_amax': Slot()}
    full, pf = run(eng, outs, **p.fields(), ldc=N, t_col0=t0, ldt=ldt)
    check_plan(pf, mode, {})
    assert plan_key(pf) == plan_key(pp) and pf['width'] == 128 and pf['splits'] == 1, f'{pf} vs {pp}'
    hi, lo = tf32_planes(plain['C'][:, :t0])
    assert bits_equal(full['C'], hi) and bits_equal(full['C_lo'], lo)
    thi, tlo = tf32_planes(plain['C'][:, t0:].t().contiguous())
    assert bits_equal(full['Ct_hi'], thi) and bits_equal(full['Ct_lo'], tlo)
    # the slot: the q|k columns as stored (hi), the V^T columns before rounding -- which the plain run shows
    assert full['c_amax'] == max(float(hi.abs().max()), float(plain['C'][:, t0:].abs().max()))


# ------------------------------------------------------------------------------------------------------------- 5. NCHW
# (name, mode, conv geometry or dense M, N): any N (the NCHW store is scalar), stride 2; the plain run pads N to a multiple of 4 with
# zero weight rows (one column's dot product does not depend on the others) so that it can take the same plan
NCHW = [('conv_n3', 1, (2, 32, 32, 32, 1), 3), ('conv_n4', 1, (2, 32, 32, 32, 1), 4), ('conv_n6_s2', 1, (2, 64, 64, 32, 2), 6),
        ('conv_n3_ts', 3, (2, 32, 32, 32, 1), 3), ('conv_n3_ffma', 0, (2, 16, 16, 64, 1), 3), ('dense_n36', 1, 2304, 36),
        ('dense_n36_fast', 4, 2304, 36), ('dense_n6_ffma', 0, 600, 6)]


@pytest.mark.parametrize('case', NCHW, ids=[c[0] for c in NCHW])
def test_nchw_output(engines, case):
    name, mode, geo, N = case
    eng = engines[mode]
    Np = -(-N // 4) * 4
    if isinstance(geo, tuple):
        p = Problem(N + 1, conv=geo, N=N)
        rpi = p.rows_per_img
        wp = torch.cat([p.w, torch.zeros(Np - N, *p.w.shape[1:])])
        pp_ = Problem(N + 1, conv=geo, N=Np, w=wp)
    else:
        p = Problem(N + 1, M=geo, K=256, N=N)
        rpi = geo // 4
        wp = torch.cat([p.w, torch.zeros(Np - N, p.K)])
        pp_ = Problem(N + 1, M=geo, K=256, N=Np, w=wp)
    bias = torch.randn(N, generator=gen(6))
    biasp = torch.cat([bias, torch.zeros(Np - N)])
    plain, pp = run(eng, {'C': Out(p.M, Np, Np)}, **pp_.fields(), ldc=Np, bias=biasp.cuda())
    imgs = p.M // rpi
    slot = Slot(init=0.0)
    full, pf = run(eng, {'C': Out(imgs * N, rpi, rpi), 'c_amax': slot}, **p.fields(), ldc=N, bias=bias.cuda(), out_nchw=1, rows_per_img=rpi)
    check_plan(pf, mode, {})
    assert plan_key(pf) == plan_key(pp), f'{pf} vs {pp}'
    want = plain['C'][:, :N].reshape(imgs, rpi, N).permute(0, 2, 1).reshape(imgs * N, rpi)
    assert bits_equal(full['C'], want)
    assert full['c_amax'] == 0.0, 'no range is fused for an NCHW result: the slot must be left as it was'
    p.check_whole(plain['C'][:, :N], mode, extra=bias.double()[None, :])


# ------------------------------------------------------------------------------------------------------------- 7. operand exponents
# dense M=512 K=640 N=320 (and a split-K shape) in the fp16-split modes: the A exponent from a tracked slot, the weight exponent from
# a net-wide range above the weight's own
EXP_SHAPES = [dict(M=512, K=640, N=320), dict(M=200, K=6400, N=324)]


@pytest.mark.parametrize('mode', [1, 4])
@pytest.mark.parametrize('shape', EXP_SHAPES, ids=['tile', 'splitk'])
def test_tracked_slot_equal_to_true_range(engines, mode, shape):
    """a slot holding exactly max |A| gives the exponent the hook measures itself: bitwise the same result"""
    eng = engines[mode]
    p = Problem(11, **shape)
    a, pa = run(eng, {'C': Out(p.M, p.N, p.N)}, **p.fields(), ldc=p.N)
    b, pb = run(eng, {'C': Out(p.M, p.N, p.N)}, **p.fields(), ldc=p.N, a_amax=torch.tensor([p.a_amax], device='cuda'))
    check_plan(pa, mode, {})
    assert plan_key(pa) == plan_key(pb) and bits_equal(a['C'], b['C'])


@pytest.mark.parametrize('mode', [1, 4])
@pytest.mark.parametrize('shape', EXP_SHAPES, ids=['tile', 'splitk'])
@pytest.mark.parametrize('slot_scale,w_scale', [(2.0 ** 8, None), (1.0, 2.0 ** 10), (1.0, 2.0 ** 20), (2.0 ** 8, 2.0 ** 20)])
def test_operand_exponents(engines, mode, shape, slot_scale, w_scale):
    eng = engines[mode]
    p = Problem(12, **shape)
    a_range = p.a_amax * slot_scale
    w_range = float(p.w.abs().max()) * w_scale if w_scale else 0.0
    r, pl = run(eng, {'C': Out(p.M, p.N, p.N)}, **p.fields(), ldc=p.N, a_amax=torch.tensor([a_range], device='cuda'), w_range=w_range)
    check_plan(pl, mode, {})
    print(f'  slot x{slot_scale:g}, w_range x{w_scale or 1:g}')
    p.check_whole(r['C'], mode, a_range=a_range, w_range=w_range)


# ------------------------------------------------------------------------------------------------------------- 8. batched FFMA
# the FFMA attention's two contractions: S = scale * Q K^T (b_kn 0) and O = P V (b_kn 1), heads along the columns (head_stride d)
ATTN = [(2, 77, 77, 4, 40), (2, 64, 77, 8, 64), (1, 256, 256, 2, 160), (3, 16, 300, 5, 80)]


@pytest.mark.parametrize('B,Nq,Nk,heads,d', ATTN)
def test_batched_ffma(engines, B, Nq, Nk, heads, d):
    eng = engines[0]
    g = gen(B * Nq + Nk + heads + d)
    C = heads * d
    q, k, v = (torch.randn(B, n, C, generator=g) for n in (Nq, Nk, Nk))
    scale = d ** -0.5
    S = Out(B * heads * Nq, Nk, Nk)
    r, pl = run(eng, {'C': S}, mode=0, M=Nq, N=Nk, K=d, A=q.cuda(), lda=C, C1=d, w=k.cuda(), ldb=C, ldc=Nk, alpha=scale, batch=B, heads=heads,
                sA_b=Nq * C, sA_h=d, sB_b=Nk * C, sB_h=d, sC_b=heads * Nq * Nk, sC_h=Nq * Nk)
    check_plan(pl, 0, {})
    qh = q.double().reshape(B, Nq, heads, d).permute(0, 2, 1, 3)
    kh = k.double().reshape(B, Nk, heads, d).permute(0, 2, 1, 3)
    s64 = scale * qh @ kh.transpose(-1, -2)
    ratio_s = float((r['C'].double().reshape(B, heads, Nq, Nk) - s64).abs().max() / (BUDGET[0] * s64.abs().max()))
    P = torch.softmax(r['C'].reshape(B, heads, Nq, Nk), -1)
    O = Out(B * Nq, C, C)
    ro, plo = run(eng, {'C': O}, mode=0, M=Nq, N=d, K=Nk, A=P.reshape(-1).cuda(), lda=Nk, C1=Nk, w=v.cuda(), ldb=C, ldc=C, b_kn=1, batch=B, heads=heads,
                  sA_b=heads * Nq * Nk, sA_h=Nq * Nk, sB_b=Nk * C, sB_h=d, sC_b=Nq * C, sC_h=d)
    vh = v.double().reshape(B, Nk, heads, d).permute(0, 2, 1, 3)
    o64 = (P.double() @ vh).permute(0, 2, 1, 3).reshape(B * Nq, C)
    ratio_o = float((ro['C'].double() - o64).abs().max() / (BUDGET[0] * o64.abs().max()))
    print(f'  batched FFMA: worst error / bound QK^T {ratio_s:.3f}, PV {ratio_o:.3f}')
    assert ratio_s <= 1.0 and ratio_o <= 1.0
