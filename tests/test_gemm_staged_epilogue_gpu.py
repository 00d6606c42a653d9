"""The tensor-core epilogue that stages its tile in shared memory: geometries it adds, through the identities of
test_gemm_epilogue_gpu.py (the full run equals the plain run plus its terms in fp32, bit for bit; guard rows and padding untouched).

The staged epilogue takes the ring slots after a work item's last stage for the output tile and the residual tile, which TMA loads
there and stores from there, clipping rows and columns outside C.  Cases:
  * work items of one or two 32-K stages, fewer than or as many as the slots the tile needs, at both tile widths;
  * a conv3x3 at both tile widths whose last M tile overhangs the batch (8x8 maps: two images per tile, an odd image count), so
    the residual box reads past the last image and the store clips it.
"""
import pytest

from tests.test_gemm_epilogue_gpu import Problem, engines, identity_case  # noqa: F401  (engines: the module's engine fixture)

pytestmark = pytest.mark.gpu

MODES = (1, 3, 4)
# (name, problem kwargs, ldc pad, ldr pad, rows per image, (width, split) wanted in every mode)
SHORT_K = [
    ('k32_w64', dict(M=4096, K=32, N=256), 0, 0, 512, (64, False)),
    ('k32_w128', dict(M=130 * 128 - 37, K=32, N=200), 4, 8, 256, (128, False)),
    ('k64_w64', dict(M=4096 - 5, K=64, N=196, lda_pad=4), 8, 4, 512, (64, False)),
]
# (name, (B, H, W, Cin, stride), Cout, ldc pad, ldr pad, (width, split) wanted)
CONV_OVERHANG = [
    ('8x8_b7_w64', (7, 8, 8, 64, 1), 256, 4, 8, (64, False)),
    ('8x8_b131_w128', (131, 8, 8, 64, 1), 256, 0, 4, (128, False)),
]


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('which', ['residual', 'all', 'cancel'])
@pytest.mark.parametrize('case', SHORT_K, ids=[c[0] for c in SHORT_K])
def test_short_k_staged_identity(engines, mode, which, case):
    name, kw, ldc_pad, ldr_pad, rows_per_img, want = case
    seed = sum(map(ord, name + which))
    p = Problem(seed, **kw)
    identity_case(engines[mode], mode, p, rows_per_img, ldc_pad, ldr_pad, which, {'wS': {want}}, seed)


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('which', ['all', 'cancel'])
@pytest.mark.parametrize('case', CONV_OVERHANG, ids=[c[0] for c in CONV_OVERHANG])
def test_conv_batch_overhang_staged_identity(engines, mode, which, case):
    name, geo, N, ldc_pad, ldr_pad, want = case
    seed = sum(map(ord, name + which))
    p = Problem(seed, conv=geo, N=N)
    identity_case(engines[mode], mode, p, p.rows_per_img, ldc_pad, ldr_pad, which, {'wS': {want}}, seed)
