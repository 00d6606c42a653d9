"""The persistent tensor-core GEMM (unsplit dense fp16-split work items, one CTA per SM walking the tile raster) against the
one-CTA-per-work-item path, in one process: every output bit for bit.

Each case runs the same call twice on one engine, Engine.set_persist(False) then set_persist(True, max_ctas), on identical inputs:
  * every dense (Linear / 1x1 conv) shape of a 12-row and an 8-row SD v1 512^2 U-Net call, with the terms the U-Net fuses there
    (bias and range slot; residual on the 320 / 640 / 1280-wide outputs; GEGLU on the FF1 shapes; the skip 1x1 convs as two
    sources), plus a per-image row vector and GroupNorm sums on the others;
  * ragged M and N at both tile widths;
  * grids of 1, 3 and 7 CTAs, so one CTA walks many work items and the ring's phases wrap many times.
C and c_amax must match bit for bit; c_stats to 1e-12 of its magnitude (its fp64 atomics are not order-fixed on either path).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

MODES = (1, 5)
# (tokens per image, K, N) of the SD v1-4 U-Net's dense layers at 512^2: Linear layers (tools/bench_ops.py), the cross-attention
# K / V projections of the 77-token context, and the ResBlock skip 1x1 convs (C1 + C2 = K: the decoder's concatenated sources)
LINEARS = [(4096, 320, 320), (4096, 320, 960), (4096, 320, 2560), (4096, 1280, 320), (1024, 640, 640), (1024, 640, 1920),
           (1024, 640, 5120), (1024, 2560, 640), (256, 1280, 1280), (256, 1280, 3840), (256, 1280, 10240), (256, 5120, 1280),
           (64, 1280, 1280), (64, 1280, 3840), (64, 1280, 10240), (64, 5120, 1280), (77, 768, 320), (77, 768, 640), (77, 768, 1280)]
SKIPS = [(4096, 320, 320, 320), (4096, 640, 320, 320), (1024, 320, 320, 640), (1024, 640, 320, 640), (1024, 640, 640, 640),
         (1024, 1280, 640, 640), (256, 640, 640, 1280), (256, 1280, 640, 1280), (256, 1280, 1280, 1280), (64, 1280, 1280, 1280)]


@pytest.fixture(scope='module')
def engines():
    from cycle_diffusion_b200.engine import Engine
    es = {}
    for m in MODES:
        es[m] = Engine(0)
        es[m].set_mma_mode(m)
    return es


def rnd(g, *shape, scale=1.0):
    return torch.randn(*shape, device='cuda', generator=g) * scale


def compare(eng, fields, out_cols, stats_rows=0, grids=(0,)):
    """run `fields` through op_gemm on the old path and on the persistent one with each grid cap; assert identity"""
    M = fields['M']
    ldc = fields.get('ldc', out_cols)

    def run(persist, grid):
        eng.set_persist(persist, grid)
        C = torch.full((M, ldc), float('nan'), device='cuda')
        amax = torch.zeros(1, device='cuda')
        extra = dict(c_amax=amax)
        stats = None
        if stats_rows:
            stats = torch.zeros(stats_rows, fields['N'], 2, dtype=torch.float64, device='cuda')
            extra['c_stats'] = stats
        plan = eng.op_gemm(**fields, C=C, **extra)
        torch.cuda.synchronize()
        return plan, C, amax, stats

    try:
        p0, c0, a0, s0 = run(False, 0)
        for grid in grids:
            p1, c1, a1, s1 = run(True, grid)
            assert (p1['kind'], p1['width'], p1['splits']) == (p0['kind'], p0['width'], p0['splits']), (p0, p1)
            assert p1['kind'] in ('h16', 'h16_fast'), p1
            assert torch.equal(c1[:, :out_cols].view(torch.int32), c0[:, :out_cols].view(torch.int32)), \
                f'grid {grid}: max|d| {(c1[:, :out_cols] - c0[:, :out_cols]).abs().max().item()}'
            assert torch.isnan(c1[:, out_cols:]).all(), 'columns past the output were written'
            assert torch.equal(a1.view(torch.int32), a0.view(torch.int32)), (a0.item(), a1.item())
            if stats_rows:
                assert p1['stats_fused'] == p0['stats_fused']
                tol = 1e-12 * s0.abs().amax(dim=(0, 1), keepdim=True)
                assert ((s1 - s0).abs() <= tol).all(), f'grid {grid}: stats max|d| {(s1 - s0).abs().max().item()}'
    finally:
        eng.set_persist(True, 0)


def dense_fields(g, M, K, N, ldc=None, C2=0):
    C1 = K - C2
    f = dict(mode=0, M=M, N=N, K=K, A=rnd(g, M, C1), lda=C1, C1=C1, w=rnd(g, N, K, scale=K ** -0.5), ldb=K, bias=rnd(g, N),
             ldc=ldc or N)
    if C2:
        f.update(A2=rnd(g, M, C2, scale=2.0), lda2=C2, C2=C2)
    return f


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('rows', [12, 8])
@pytest.mark.parametrize('shape', LINEARS, ids=[f'{t}x{k}x{n}' for t, k, n in LINEARS])
def test_unet_linear_shapes(engines, mode, rows, shape):
    tokens, K, N = shape
    M = tokens * rows
    g = torch.Generator(device='cuda').manual_seed(tokens + K * 3 + N * 7 + rows)
    if N == 8 * K:                                   # FF1: GEGLU, value / gate in [32 | 32] column blocks
        f = dict(dense_fields(g, M, K, N), geglu=1, ldc=N // 2)
        compare(engines[mode], f, N // 2)
        return
    f = dense_fields(g, M, K, N)
    compare(engines[mode], f, N)
    if N in (320, 640, 1280) and tokens % 32 == 0:
        f2 = dict(f, residual=rnd(g, M, N), ldr=N, rows_per_batch=tokens)
        compare(engines[mode], f2, N, stats_rows=rows)


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('rows', [12, 8])
@pytest.mark.parametrize('shape', SKIPS, ids=[f'{t}x{a}+{b}x{n}' for t, a, b, n in SKIPS])
def test_unet_skip_convs_two_sources(engines, mode, rows, shape):
    tokens, C1, C2, N = shape
    M = tokens * rows
    g = torch.Generator(device='cuda').manual_seed(tokens + C1 * 3 + C2 * 5 + N * 7 + rows)
    f = dict(dense_fields(g, M, C1 + C2, N, C2=C2), residual=rnd(g, M, N), ldr=N)
    compare(engines[mode], f, N)


# (M, K, N, ldc): ragged M and N, at the widths the planner picks for them
RAGGED = [(130 * 128 - 37, 320, 200, 204), (4096 - 5, 64, 196, 200), (12288 + 77, 640, 644, 648), (3000, 32, 256, 256),
          (49152 - 1, 1280, 324, 324)]


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('case', RAGGED, ids=[f'{m}x{k}x{n}' for m, k, n, _ in RAGGED])
def test_ragged_all_terms(engines, mode, case):
    M, K, N, ldc = case
    g = torch.Generator(device='cuda').manual_seed(M + K + N)
    rows_per_batch = 64
    nb = -(-M // rows_per_batch)
    f = dict(dense_fields(g, M, K, N, ldc=ldc), residual=rnd(g, M, N + 4), ldr=N + 4, rowvec=rnd(g, nb, N), ld_rowvec=N,
             rows_per_batch=rows_per_batch)
    compare(engines[mode], f, N, stats_rows=nb if M % rows_per_batch == 0 else 0)


# grids of 1, 3 and 7 CTAs: each walks many work items, the ring's stage counter wraps its phase many times
SMALL_GRID = [('k320_w128', 12288, 320, 640, 0), ('k640_two_src_w128', 4096, 640, 320, 320), ('k64_ragged', 4096 - 5, 64, 196, 0),
              ('k1280_geglu', 2048, 1280, 2048, 0)]


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('case', SMALL_GRID, ids=[c[0] for c in SMALL_GRID])
def test_small_grids(engines, mode, case):
    name, M, K, N, C2 = case
    g = torch.Generator(device='cuda').manual_seed(sum(map(ord, name)))
    if 'geglu' in name:
        f = dict(dense_fields(g, M, K, N), geglu=1, ldc=N // 2)
        compare(engines[mode], f, N // 2, grids=(1, 3, 7))
        return
    f = dict(dense_fields(g, M, K, N, C2=C2), residual=rnd(g, M, N), ldr=N, rows_per_batch=256)
    compare(engines[mode], f, N, stats_rows=M // 256 if M % 256 == 0 else 0, grids=(1, 3, 7))
