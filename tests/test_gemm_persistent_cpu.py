"""The persistent tensor-core GEMM's tile walk, restated on the host: CTA c of a grid of G takes work items t = c, c + G, ... and maps
each through tile_coord's band raster (kernels_tc.cu).  For every grid from 1 to the H100's 132 SMs, every output tile of the
dense shapes the persistent path serves is computed exactly once."""
import pytest

RASTER_M = 8      # kernels_tc.cu: M tiles per band of the raster
NUM_SMS = 132


def tile_coord(t, tiles_m, tiles_n):
    """(tm, tn) of work item t of one unsplit dense launch (tile_coord with splits == 1, one z)"""
    m_lo = t // (RASTER_M * tiles_n) * RASTER_M
    bm = min(RASTER_M, tiles_m - m_lo)
    u = t - m_lo * tiles_n
    return m_lo + u % bm, u // bm


def walk(grid, total):
    for c in range(min(grid, total)):
        yield from range(c, total, grid)


# (tiles_m, tiles_n): 12-row SD v1 shapes at BN 128 / 64, and ragged bands (tiles_m not a multiple of RASTER_M)
SHAPES = [(384, 3), (384, 5), (96, 5), (96, 20), (24, 10), (6, 10), (1, 1), (1, 7), (130, 2), (33, 4), (7, 3), (9, 1)]


@pytest.mark.parametrize('tiles', SHAPES, ids=[f'{m}x{n}' for m, n in SHAPES])
def test_walk_covers_every_tile_once(tiles):
    tiles_m, tiles_n = tiles
    total = tiles_m * tiles_n
    for grid in range(1, NUM_SMS + 1):
        seen = {}
        for t in walk(grid, total):
            tm, tn = tile_coord(t, tiles_m, tiles_n)
            assert 0 <= tm < tiles_m and 0 <= tn < tiles_n
            seen[(tm, tn)] = seen.get((tm, tn), 0) + 1
        assert len(seen) == total and set(seen.values()) == {1}, f'grid {grid}'
