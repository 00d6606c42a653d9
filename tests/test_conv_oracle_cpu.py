"""CPU checks of the conv3x3 gather suite's restatements, reference and error bound (tests/conv_oracle.py)."""
import pytest
import torch

from tests import conv_oracle as O

torch.set_num_threads(8)


# ------------------------------------------------------------------------------------------------------------- box rules
# (Ho, Wo, B, stride) -> (bw, bh, bn, tiles_m), worked by hand from the rules in conv_oracle's docstring
BOXES = [
    ((8, 8, 5, 1), (8, 8, 2, 3)),             # pow2: bw = Wo, bh = Ho, two images per tile, B odd
    ((16, 16, 3, 1), (16, 8, 1, 6)),          # pow2: bw capped at 16, bh = 128 / 16
    ((64, 4, 1, 1), (4, 32, 1, 2)),           # pow2, tall: bh capped at 128 / bw
    ((1, 1, 130, 1), (1, 1, 128, 2)),         # pow2 1x1: 128 images per tile
    ((1, 2, 40, 2), (2, 1, 64, 1)),
    ((3, 5, 5, 1), (8, 4, 4, 2)),             # ragged: two tiles is the fewest (bn >= 5 leaves bw bh <= 16 < 8 x 3); 8x4x4 the smallest halo
    ((40, 1, 5, 1), (1, 64, 2, 3)),           # ragged column: 1x64x2 covers 40 rows of two images in one tile
    ((1, 100, 3, 1), (128, 1, 1, 3)),         # ragged row: one 128-wide tile per image
    ((1, 80, 9, 2), (128, 1, 1, 9)),          # stride 2: bw 2 = 256, TMA's box limit, still allowed
    ((80, 1, 9, 2), (1, 128, 1, 9)),          # bh 2 = 256
    ((6, 10, 33, 1), (2, 8, 8, 25)),          # ragged, many images: 5 x 1 x 5 tiles beat any wider box
    ((24, 40, 1, 1), (16, 8, 1, 9)),
    ((48, 80, 1, 2), (16, 8, 1, 30)),
]


@pytest.mark.parametrize('geo,want', BOXES)
def test_box_table(geo, want):
    assert O.conv_box(*geo) == want


def test_box_refusal_and_product():
    """every box is 128 pixels; the TMA limit refuses a box side past 256 elements"""
    for stride in (1, 2):
        for Ho in range(1, 70):
            for Wo in (1, 2, 3, 5, 8, 13, 40, 64, 100, 130):
                b = O.conv_box(Ho, Wo, 3, stride)
                assert b is not None and b[0] * b[1] * b[2] == 128
                assert b[0] * stride <= 256 and b[1] * stride <= 256
    # stride 4 (not a conv the engine runs): the ragged rule skips 128-wide boxes, whose TMA box would be 512 elements
    assert O.conv_ragged_tile(100, 1, 1, 4)[0] == 64


def reachable(stride):
    bws, bns = set(), set()
    for Ho in range(1, 160):
        for Wo in range(1, 160):
            for B in (1, 2, 3, 5, 9, 17, 33, 65, 129):
                b = O.conv_box(Ho, Wo, B, stride)
                bws.add(b[0])
                bns.add(b[2])
    return bws, bns


def test_suite_covers_every_box():
    tc = [c for c in O.SUITE if c.tc()]
    for stride in (1, 2):
        bws, bns = reachable(stride)
        assert bws == bns == {1 << i for i in range(8)}, f'stride {stride}: reachable bw {sorted(bws)}, bn {sorted(bns)}'
        boxes = [c.box() for c in tc if c.stride == stride]
        assert {b[0] for b in boxes} == bws, f'stride {stride}: bw {sorted(bws - {b[0] for b in boxes})} never runs'
        assert {b[2] for b in boxes} == bns, f'stride {stride}: bn {sorted(bns - {b[2] for b in boxes})} never runs'
    s2 = [c.box() for c in tc if c.stride == 2]
    assert any(b[0] * 2 == 256 for b in s2) and any(b[1] * 2 == 256 for b in s2)
    # a tile that overhangs the batch and the map's x or y edge at once
    assert any(c.B % c.box()[2] and (c.Wout % c.box()[0] or c.Hout % c.box()[1]) for c in tc)
    assert {c.stride for c in tc} == {1, 2} and {c.pad for c in tc if c.stride == 2} == {0, 1}
    kinds = ('h16', 'ts', 'h16_fast')
    assert {c.plan(k)[0] for c in tc for k in kinds} == {64, 128}
    assert {c.plan('h16')[1] for c in tc} >= set(range(1, 9))
    assert {c.Cin for c in tc} >= {32, 64, 96, 320, 1280, 1920}
    assert {c.N for c in tc} >= {4, 36, 100, 320, 640, 1280} and any(c.N == 4 and c.M >= 2048 for c in tc)
    ffma = [c for c in O.SUITE if not c.tc()]
    assert {c.Cin for c in ffma} >= {3, 4, 20} and any(c.up == 2 for c in ffma)
    assert any(c.stride == 2 and c.Hin != 2 * c.Hout for c in ffma)
    assert {c.N for c in O.SUITE if c.nchw} == {3, 4, 6}


def test_eligibility():
    assert O.tc_eligible(80, 36, 32, 4, 4, 2, 2, 2)
    assert not O.tc_eligible(80, 36, 20, 4, 4, 2, 2, 2)                     # Cin % 32
    assert not O.tc_eligible(80, 36, 32, 9, 15, 5, 8, 2)                    # Hin != 2 Hout
    assert not O.tc_eligible(512, 36, 32, 8, 8, 16, 16, 1, up=2)            # nearest-2x fold
    assert not O.tc_eligible(48, 36, 32, 4, 4, 4, 4, 1)                     # M < 64
    assert not O.tc_eligible(1024, 4, 32, 32, 32, 32, 32, 1)                # thin N, small M
    assert O.tc_eligible(2048, 4, 32, 32, 32, 32, 32, 1)                    # thin N, large M
    assert O.tc_eligible(2048, 3, 32, 32, 32, 32, 32, 1, out_nchw=True)     # the NCHW store takes any N
    assert not O.tc_eligible(2048, 36, 32, 32, 32, 32, 32, 1, lda=34)       # lda % 4


def test_plan_table():
    """hand-checked partitions (132 SMs): the cost model's tie-breaks and its split-K refusals"""
    assert O.plan(513, 128, 640, 5, 'h16') == (64, 3)
    assert O.plan(521, 128, 640, 5, 'h16') == (64, 1)        # the M term of the split traffic tips it
    assert O.plan(64, 36, 17280, 1, 'h16') == (64, 8)
    assert O.plan(64, 36, 17280, 1, 'h16', flags=2) == (64, 1)   # NCHW: never split
    assert O.plan(64, 36, 17280, 1, 'ss') == (128, 8)             # raw fp32 B: 128 wide only
    # 45 k-blocks; w 128: 3 waves of 384 items x (45 (700 + 768) + 3000) = 207180 < w 64: 5 waves x (45 (700 + 384) + 3000) = 258900
    assert O.plan(16384, 320, 2880, 128, 'h16') == (128, 1)


# ------------------------------------------------------------------------------------------------------------- reference
def test_conv64_matches_torch():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 7, 9, 5, generator=g)
    w = torch.randn(4, 5, 3, 3, generator=g)
    xc = x.double().permute(0, 3, 1, 2)
    for stride, pad, up in ((1, 1, 1), (2, 1, 1), (2, 0, 1), (1, 1, 2)):
        y, S = O.conv64(x, w, stride, pad, up)
        xi = xc.repeat_interleave(up, 2).repeat_interleave(up, 3)
        ref = torch.nn.functional.conv2d(torch.nn.functional.pad(xi, (pad, 1, pad, 1)), w.double(), stride=stride)
        Ho, Wo = O.out_size(7, stride, pad, up), O.out_size(9, stride, pad, up)
        assert ref.shape[2:] == (Ho, Wo)
        assert torch.allclose(y, ref.permute(0, 2, 3, 1).reshape(-1, 4), rtol=0, atol=1e-12)
        refa = torch.nn.functional.conv2d(torch.nn.functional.pad(xi.abs(), (pad, 1, pad, 1)), w.double().abs(), stride=stride)
        assert torch.allclose(S, refa.permute(0, 2, 3, 1).reshape(-1, 4), rtol=0, atol=1e-12)


# ------------------------------------------------------------------------------------------------------------- bound vs simulation
SIM = [O.Case('sim_5x7', 2, 5, 7, 32, 24), O.Case('sim_5x7_pos', 2, 5, 7, 64, 24, data='pos'),
       O.Case('sim_3x4_outlier', 3, 3, 4, 96, 16, data='outlier'), O.Case('sim_4x4_k1152', 2, 4, 4, 128, 16)]


def represented_sums(c, x, w):
    A = O.im2col64(x, c.stride, c.pad, c.up)
    return A, O.wmat(w).double(), A.abs().sum(1), O.wmat(w).double().abs().sum(1)


@pytest.mark.parametrize('c', SIM, ids=[c.name for c in SIM])
@pytest.mark.parametrize('kind', ['h16', 'h16_fast', 'ts'])
@pytest.mark.parametrize('splits', [1, 3])
def test_bound_holds_on_simulated_kernel(c, kind, splits):
    x, w = c.operands()
    y, S = O.conv64(x, w)
    A, W, asum, wsum = represented_sums(c, x, w)
    e_a, b_exp = O.exponents(x, w)
    got = O.simulate(A.float(), W.float(), kind, splits, e_a, b_exp)
    bnd = O.bound(S, asum, wsum, c.K, kind, splits, e_a, b_exp)
    ratio = float(((got - y).abs() / bnd).max())
    print(f'{c.name} {kind} S{splits}: worst error / bound {ratio:.3f}')
    assert 0.0 < ratio <= 1.0


def test_bound_holds_for_sequential_fma():
    c = SIM[1]
    x, w = c.operands()
    y, S = O.conv64(x, w)
    A, W, _, _ = represented_sums(c, x, w)
    acc = torch.zeros(A.shape[0], W.shape[0], dtype=torch.float64)
    for k in range(c.K):
        acc = (acc + A[:, k:k + 1] * W[:, k][None, :]).float().double()
    assert float(((acc - y).abs() / O.bound(S, None, None, c.K, 'ffma')).max()) <= 1.0


def test_floor_grows_with_a_conservative_slot():
    """a slot 2^8 above the true range costs A 8 bits: the simulated error grows past the unscaled bound's reach only by the floor"""
    c = SIM[0]
    x, w = c.operands(a_scale=2.0 ** -12)
    y, S = O.conv64(x, w)
    A, W, asum, wsum = represented_sums(c, x, w)
    e_a, b_exp = O.exponents(x, w, a_slot=float(x.abs().max()) * 2.0 ** 8)
    got = O.simulate(A.float(), W.float(), 'h16', 1, e_a, b_exp)
    assert float(((got - y).abs() / O.bound(S, asum, wsum, c.K, 'h16', 1, e_a, b_exp)).max()) <= 1.0
    assert e_a == O.exponents(x, w)[0] - 8


# ------------------------------------------------------------------------------------------------------------- bound vs broken kernels
def fault_ratios(c):
    """worst |fault error| / bound over the case's outputs for (a) the hi_a lo_w term dropped, (b) the centre tap read one pixel to
    the right, with the bound of the kind the case runs in mode 1"""
    x, w = c.operands()
    y, S = O.conv64(x, w, c.stride, c.pad, c.up)
    A = O.im2col64(x, c.stride, c.pad, c.up)
    W = O.wmat(w).double()
    kind = 'h16' if c.tc() else 'ffma'
    splits = c.plan('h16')[1] if c.tc() else 1
    e_a, b_exp = O.exponents(x, w)
    bnd = O.bound(S, A.abs().sum(1), W.abs().sum(1), c.K, kind, splits, e_a, b_exp)
    d = torch.zeros_like(w)
    d[:, :, 1, 2] = w[:, :, 1, 1]
    d[:, :, 1, 1] = -w[:, :, 1, 1]
    shift = O.conv64(x, d, c.stride, c.pad, c.up)[0]
    r_shift = float((shift.abs() / bnd).max())
    if kind != 'h16':
        return None, r_shift
    ah = O.planes(x, 'h16', e_a)[0] * 2.0 ** -e_a
    wl = O.planes(w, 'h16', b_exp)[1] * 2.0 ** -b_exp
    drop = O.conv64(ah, wl, c.stride, c.pad, c.up)[0]
    return float((drop.abs() / bnd).max()), r_shift


@pytest.mark.parametrize('c', O.SUITE, ids=[c.name for c in O.SUITE])
def test_bound_sees_broken_kernels(c):
    r_drop, r_shift = fault_ratios(c)
    print(f'{c.name}: dropped lo.hi {r_drop} x bound, shifted tap {r_shift:.1f} x bound')
    assert r_shift > 2.0
    assert r_drop is None or r_drop > 2.0


def test_gemm_desc_takes_up_as_a_trailing_field():
    """cdx_gemm_desc grew `up` at its end (ABI version 2 unchanged): the binding's layout ends with it"""
    import ctypes
    from cycle_diffusion_b200 import _cabi
    assert _cabi.GemmDesc._fields_[-1] == ('up', ctypes.c_int)
    assert _cabi.GemmDesc.up.offset == _cabi.GemmDesc.sC_h.offset + 8
    assert _cabi.lib.cdx_abi_version() == 2
