"""The conv3x3 gather against float64, through the production gemm() (cdx_op_gemm, mode 1), on every pixel box, stride, padding and
route: the tensor-core conv (modes 1, 3 and 4: the fp16 split, 3xTF32 and the one-term fp16 term of autocast) and the FFMA tiles
(mode 0, and whatever the tensor cores refuse).  The geometries, restatements, reference and elementwise bound are in
tests/conv_oracle.py, pinned on the CPU by tests/test_conv_oracle_cpu.py.

Every case:
  * the input sits inside one allocation at pixel stride lda = Cin + pad, with a guard image before and after it; the pad columns
    and the guards hold a NaN sentinel, so a read outside [B, Hin, Win, Cin] makes a NaN.  (The weights are repacked by the call, so
    their row padding is not the caller's to poison.)  The output sits inside the epilogue suite's Out: NaN guard rows and ldc
    padding that must come back untouched;
  * the route (tensor cores or FFMA tiles) is the one tc_eligible restates, and the work partition the one plan / ffma_tile do;
  * the result is within the oracle's elementwise bound and within the per-op budget of test_gemm_epilogue_gpu.py;
  * two runs are bitwise equal.
The worst error / bound per mode is printed at the end, with the file's time.
"""
import time

import pytest
import torch

from tests import conv_oracle as O
from tests.gemm_epilogue_oracle import split_floor
from tests.test_gemm_epilogue_gpu import BUDGET, KIND, MODES, SENTINEL, Out, engines, run  # noqa: F401  (engines: the module's fixture)

pytestmark = pytest.mark.gpu

WORST = {}


@pytest.fixture(scope='module', autouse=True)
def report():
    t0 = time.time()
    yield
    print(f'\nconv gather suite: {time.time() - t0:.1f} s; worst error / bound per mode: '
          + ', '.join(f'{m}: {r:.3f}' for m, r in sorted(WORST.items())))


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Input:
    """x [B, Hin, Win, Cin] at pixel stride lda (a multiple of 4 above Cin) between two guard images, pads and guards NaN"""

    def __init__(self, x):
        B, H, W, C = x.shape
        self.lda = C + 4 + (-C) % 4
        img = H * W * self.lda
        store = torch.empty((B + 2) * img, dtype=torch.float32)
        store.view(torch.int32).fill_(SENTINEL)
        store[img:(B + 1) * img].view(B, H, W, self.lda)[..., :C] = x
        self.store = store.cuda()
        self.view = self.store[img:]


class Ref:
    """a case's operands on the device and its float64 reference"""

    def __init__(self, c, **kw):
        self.c = c
        self.x, self.w = c.operands(**kw)
        self.inp = Input(self.x)
        self.w_dev = self.w.cuda()
        self.y, self.S = O.conv64(self.x, self.w, c.stride, c.pad, c.up)
        self.asum = O.im2col64(self.x.abs(), c.stride, c.pad, c.up).sum(1)
        self.wsum = O.wmat(self.w).double().abs().sum(1)

    def fields(self):
        c = self.c
        return dict(mode=1, M=c.M, N=c.N, K=c.K, A=self.inp.view, lda=self.inp.lda, C1=c.Cin, w=self.w_dev, Hin=c.Hin, Win=c.Win,
                    Hout=c.Hout, Wout=c.Wout, stride=c.stride, pad=c.pad, up=c.up)


def conv_run(eng, mode, ref, a_slot=None):
    """one case in one mode: route and partition as restated, guards intact, bitwise repeatable, within the bound and the budget.
    -> (worst error / bound, worst error / S)"""
    c = ref.c
    hw = c.Hout * c.Wout
    if c.nchw:
        out, ldc, extra = Out(c.B * c.N, hw, hw), c.N, dict(out_nchw=1, rows_per_img=hw)
    else:
        out, ldc, extra = Out(c.M, c.N, c.N + 4), c.N + 4, {}
    if a_slot is not None:
        extra['a_amax'] = torch.tensor([a_slot], device='cuda')
    r, p = run(eng, {'C': out}, **ref.fields(), ldc=ldc, **extra)
    y = r['C'].reshape(c.B, c.N, hw).permute(0, 2, 1).reshape(c.M, c.N) if c.nchw else r['C']
    tc = mode != 0 and c.tc(lda=ref.inp.lda, ldc=ldc)
    kind = KIND[mode] if tc else 'ffma'
    assert p['kind'] == kind, f'{c.name} mode {mode}: expected the {kind} route, ran {p}'
    if tc:
        want = c.plan(kind, sms())
        assert (p['width'], p['splits']) == want, f'{c.name} mode {mode}: planned {want}, ran {p}'
    else:
        assert (p['width'], p['splits']) == (O.ffma_tile(c.M, c.N, sms()), 1), f'{c.name} mode {mode}: {p}'
    assert bool(torch.isfinite(y).all()), f'{c.name} mode {mode}: a NaN came back (a read outside the input)'
    e_a, b_exp = O.exponents(ref.x, ref.w, a_slot)
    bnd = O.bound(ref.S, ref.asum, ref.wsum, c.K, kind, p['splits'], e_a, b_exp)
    err = (y.double() - ref.y).abs()
    ratio = float((err / bnd).max())
    budget = BUDGET[mode] * float(ref.y.abs().max())
    if kind in ('h16', 'h16_fast'):
        budget = budget + split_floor(ref.asum, ref.wsum, e_a, b_exp)
    b_ratio = float((err / budget).max())
    print(f'{c.name} mode {mode}: {p["kind"]} w{p["width"]} S{p["splits"]}  error / bound {ratio:.3f}, / budget {b_ratio:.3f}')
    WORST[mode] = max(WORST.get(mode, 0.0), ratio)
    assert ratio <= 1.0, f'{c.name} mode {mode}: error {ratio:.2f}x the bound'
    assert b_ratio <= 1.0, f'{c.name} mode {mode}: error {b_ratio:.2f}x the per-op budget'
    return ratio, float((err / ref.S.clamp_min(1e-300)).max())


# ------------------------------------------------------------------------------------------------------------- planning
def test_each_shape_plans_on_its_own(engines):
    """two shapes of one 128-row band (one plan-cache band before M was in the key) plan differently: each runs its own plan, in
    either order.  Shapes no other test plans: the plan cache lives for the whole process."""
    eng = engines[1]
    g = torch.Generator().manual_seed(31)
    for M in (513, 521):                              # dense N=128, K=640: (w64, S3) then (w64, S1)
        A, w = torch.randn(M, 640, generator=g).cuda(), torch.randn(128, 640, generator=g).cuda()
        p = eng.op_gemm(mode=0, M=M, N=128, K=640, A=A, lda=640, C1=640, w=w, ldb=640, C=torch.empty(M, 128, device='cuda'), ldc=128)
        assert (p['width'], p['splits']) == O.plan(M, 128, 640, O.cdiv(M, 128), 'h16', sms=sms()), f'dense M={M}: {p}'
    for B in (8, 7):                                  # conv 7x7, Cin 96, N 640, the same four tiles: (w64, S1) then (w64, S3)
        c = O.Case(f'plan_7x7_b{B}', B, 7, 7, 96, 640)
        ref = Ref(c)
        p = eng.op_gemm(**ref.fields(), C=torch.empty(c.M, c.N, device='cuda'), ldc=c.N)
        assert (p['width'], p['splits']) == c.plan('h16', sms()), f'conv B={B}: {p}'
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------------- the suite
@pytest.mark.parametrize('c', O.SUITE, ids=[c.name for c in O.SUITE])
def test_conv_gather(engines, c):
    ref = Ref(c)
    for mode in MODES:
        conv_run(engines[mode], mode, ref)


# ------------------------------------------------------------------------------------------------------------- range slots
SLOT_CASE = O.Case('slot_7x7_b3', 3, 7, 7, 64, 100)


def test_conservative_slot(engines):
    """an A slot 2^8 above the true range: 8 bits fewer for A, which the split floor accounts for.  (A range of 2^-10: both it and
    the slot lie below the [4, 2^15) window in which the device rule does not rescale.)"""
    ref = Ref(SLOT_CASE, a_scale=2.0 ** -12)
    amax = float(ref.x.abs().max())
    assert O.exponents(ref.x, ref.w, amax * 2.0 ** 8)[0] == O.exponents(ref.x, ref.w)[0] - 8
    conv_run(engines[1], 1, ref, a_slot=amax * 2.0 ** 8)


def test_exact_slot_equals_measured_range(engines):
    ref = Ref(SLOT_CASE)
    out = {}
    for slot in (None, float(ref.x.abs().max())):
        o = Out(SLOT_CASE.M, SLOT_CASE.N, SLOT_CASE.N)
        extra = {} if slot is None else dict(a_amax=torch.tensor([slot], device='cuda'))
        out[slot is None], _ = run(engines[1], {'C': o}, **ref.fields(), ldc=SLOT_CASE.N, **extra)
    assert torch.equal(out[True]['C'].view(torch.int32), out[False]['C'].view(torch.int32))


@pytest.mark.parametrize('scale', [1e-6, 3e4])
def test_operand_scale(engines, scale):
    """operands far from 1: the tracked exponents keep the relative error of unit-scale operands (the relative part of the bound,
    without the floor)"""
    ref = Ref(SLOT_CASE, a_scale=scale)
    _, rel = conv_run(engines[1], 1, ref)
    assert rel <= O.rel_bound(SLOT_CASE.K, 'h16'), f'scale {scale}: relative error {rel:.3g}'
