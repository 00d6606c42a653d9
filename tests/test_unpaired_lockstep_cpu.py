"""CPU checks for lock-step unpaired translation: the new C entry points, the chunked draw order, the schedule-compatibility check."""
import pytest
import torch

from cycle_diffusion_b200 import _cabi
from cycle_diffusion_b200.schedule import DDIMSchedule, PixelSchedule, same_schedule
from cycle_diffusion_b200.wrappers import lockstep_noise_chunks


def test_lockstep_symbols_exported_and_bound():
    for s in ('cdx_pixel_cycle_lockstep', 'cdx_latent_cycle_pair'):
        assert hasattr(_cabi.lib, s), f'{s} not exported by libcdx.so'
        assert s in _cabi.SIGNATURES
    assert _cabi.lib.cdx_abi_version() == 2


@pytest.mark.parametrize('n_rec,chunk,buffered', [(0, 4, True), (1, 1, True), (7, 3, True), (7, 1, False), (7, 7, True), (7, 32, True),
                                                  (9, 4, False)])
def test_chunked_draws_match_two_phase_order(n_rec, chunk, buffered):
    """encode's x_T + n_rec draws, then generate's `last` and two refine iterations (q_sample draw + 3 steps each): the chunked
    helper yields the same tensors and leaves the CPU generator where the two-phase path leaves it."""
    shape = (2, 3, 8, 8)

    def tail():
        return [torch.randn(shape)] + [torch.randn(shape) for _ in range(2 * (1 + 3))]

    torch.manual_seed(123)
    ref = list(torch.stack([torch.randn(shape) for _ in range(n_rec + 1)])) + tail()
    torch.manual_seed(123)
    bufs = [torch.empty((min(chunk, n_rec) + 1,) + shape) for _ in range(2)] if buffered else None
    got, ranges = [], []
    for i0, i1, nz in lockstep_noise_chunks(shape, n_rec, chunk, bufs):
        assert nz.shape == (i1 - i0 + (i0 == 0),) + shape
        ranges.append((i0, i1))
        got += [t.clone() for t in nz]
    got += tail()
    assert ranges[0][0] == 0 and ranges[-1][1] == n_rec
    assert all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
    assert all(i1 - i0 <= chunk for i0, i1 in ranges)
    assert len(got) == len(ref)
    assert all(torch.equal(a, b) for a, b in zip(got, ref))


def test_same_schedule_accepts_identical_and_rejects_mismatches():
    a = PixelSchedule('ddim', 100, 20, 0.1)
    assert same_schedule(a, PixelSchedule('ddim', 100, 20, 0.1))
    for other in (PixelSchedule('ddim', 100, 21, 0.1), PixelSchedule('ddim', 100, 20, 0.2), PixelSchedule('ddpm', 100, 20),
                  PixelSchedule('ddim', 50, 20, 0.1)):
        assert not same_schedule(a, other)
    p = PixelSchedule('ddpm', 100, 20)
    assert same_schedule(p, PixelSchedule('ddpm', 100, 20)) and not same_schedule(p, PixelSchedule('ddpm', 100, 20, var_type='fixedlarge'))
    d = DDIMSchedule(50, 0.1)
    assert same_schedule(d, DDIMSchedule(50, 0.1))
    for other in (DDIMSchedule(50, 0.2), DDIMSchedule(40, 0.1), DDIMSchedule(50, 0.1, skip_steps=5)):
        assert not same_schedule(d, other)
    assert not same_schedule(a, d)
