"""CPU checks for the lock-step ensemble search: the planner's order, chunks and U-Net row counts, the replayed random draws, the
selection rule, and the new C entry points."""
import random

import pytest
import torch

from cycle_diffusion_b200 import _cabi
from cycle_diffusion_b200.ensemble import EnsemblePlan, MemberNoise, guidance_rows, select_better
from cycle_diffusion_b200.schedule import DDIMSchedule
from cycle_diffusion_b200.wrappers import _StochasticTextWrapperBase

# [gan] section of translate_text2img256_stable_diffusion_stochastic_1.cfg (the 16 published text configurations share it)
PUBLISHED = dict(custom_steps=99, white_box_steps=100, eta=0.1, encoder_unconditional_guidance_scales=[1],
                 decoder_unconditional_guidance_scales=[1, 1.5, 2, 3, 4, 5], n_trials=15, skip_steps=[15, 20, 25, 30, 40, 50])


def _plan(n_trials, enc, skips, dec, bsz, budget, steps=99):
    return EnsemblePlan(n_trials, enc, skips, dec, bsz, {s: DDIMSchedule(steps, 0.1, s).refine_steps for s in skips}, budget)


def test_member_and_candidate_order_follow_the_reference_loops():
    enc, skips, dec = [1.0, 3.0], [2, 3, 5], [1.0, 0.0, 3.0]
    p = _plan(2, enc, skips, dec, 1, 100, steps=8)
    ref = [(t, e, s) for t in range(2) for e in enc for s in skips]                    # SDW:189-191, skip innermost
    assert p.members == ref
    cands = [(m, k) for m in range(len(ref)) for k in range(len(dec))]                 # SDW:146-165: each z, then each decoder scale
    assert [p.candidate(m, k) for m, k in cands] == list(range(len(cands))) == list(range(p.n_candidates))
    # SDW:237-247 recovers (encoder scale, decoder scale, skip) of a best index with skip varying fastest over the member index
    for idx in range(p.n_candidates):
        m, k = divmod(idx, len(dec))
        assert p.members[m][2] == skips[m % len(skips)] and p.dec_scales[k] == dec[k]


@pytest.mark.parametrize('bsz,budget', [(1, 1), (1, 12), (2, 20), (3, 48), (2, 1000)])
def test_every_chain_in_exactly_one_chunk_within_budget(bsz, budget):
    p = _plan(3, [1, 2.5], [10, 20, 30], [1, 0, 3, 5], bsz, budget)
    seen = []
    for c in p.chunks:
        assert c.chains and len({p.members[m][2] for m, _ in c.chains}) == 1 and p.members[c.chains[0][0]][2] == c.skip
        assert c.rows == sum(p.chain_rows(m) for m, _ in c.chains)
        assert c.rows <= budget or len(c.chains) == 1
        seen += c.chains
    assert sorted(seen) == sorted((m, b) for m in range(len(p.members)) for b in range(bsz))
    assert len(seen) == len(set(seen))


def test_guidance_rows():
    assert [guidance_rows(s) for s in (1, 1.0, 0, 0.0, 1.5, 3, -1)] == [1, 1, 1, 1, 2, 2, 2]


def test_published_configuration_counts():
    """SURVEY 8f-2: 74,520 U-Net sample-forwards per image for the lock-step search, 86,940 for encode + forward as the engine
    runs it (both CFG segments for every batched chain)."""
    g = PUBLISHED
    p = _plan(g['n_trials'], g['encoder_unconditional_guidance_scales'], g['skip_steps'], g['decoder_unconditional_guidance_scales'], 1, 48,
              steps=g['custom_steps'])
    assert all(g['white_box_steps'] - s - 1 >= DDIMSchedule(g['custom_steps'], g['eta'], s).refine_steps for s in g['skip_steps'])
    assert p.n_candidates == 540
    assert p.sample_forwards() == 74520
    assert p.two_phase_sample_forwards() == 86940


def test_replayed_draws_equal_encode_batched():
    """MemberNoise's per-chunk noise equals the draws _encode_batched makes (same calls, same order), and the CPU generator ends
    where encode() leaves it."""
    enc, skips, dec, bsz, shape = [1.0, 3.0], [2, 3], [1.0, 0.0, 3.0], 2, (2, 4, 3, 3)
    S = 6
    scheds = {s: DDIMSchedule(S, 0.1, s) for s in skips}
    draw = lambda skip: _StochasticTextWrapperBase._encode_noise(None, scheds[skip], scheds[skip].refine_steps, shape)
    torch.manual_seed(5)
    ref = []
    for _trial in range(2):                                   # _encode_batched's loop
        for _e in enc:
            for skip in skips:
                ref.append(draw(skip))
    after = torch.randn(4)
    p = EnsemblePlan(2, enc, skips, dec, bsz, {s: sc.refine_steps for s, sc in scheds.items()}, 7)
    torch.manual_seed(5)
    mn = MemberNoise(p, draw)
    chunks = list(p.chunks)
    random.Random(0).shuffle(chunks)
    for c in chunks:
        nz = mn.chunk(c)
        assert nz.shape == (scheds[c.skip].refine_steps + 1, len(c.chains)) + shape[1:]
        for j, (m, b) in enumerate(c.chains):
            assert torch.equal(nz[:, j], ref[m][:, b])
    assert torch.equal(torch.randn(4), after)


def _argmax_by_rule(chunks, B, n):
    best = [(0.0, -1)] * B
    for scores, cand, samp in chunks:
        for s, c, b in zip(scores, cand, samp):
            if select_better(s, c, *best[b]):
                best[b] = (s, c)
    return [i for _, i in best]


def test_selection_rule_equals_torch_argmax():
    nan = float('nan')
    rows = [[0.5, 0.9, 0.9, 0.1, nan, 0.9, nan],      # tie and NaNs: the first NaN
            [0.2, 0.7, 0.1, 0.7, 0.7, -1.0, 0.3],     # ties: the lowest index
            [-float('inf')] * 7,                      # all equal
            [nan] * 7,
            [0.1, 0.2, 0.3, 0.4, 0.5, 0.6, float('inf')]]
    mat = torch.tensor(rows)
    B, n = mat.shape
    entries = [(mat[b, c].item(), c, b) for b in range(B) for c in range(n)]
    for seed in range(20):
        random.Random(seed).shuffle(entries)
        cut = sorted(random.Random(100 + seed).sample(range(1, len(entries)), 2))
        parts = [entries[:cut[0]], entries[cut[0]:cut[1]], entries[cut[1]:]]
        chunks = [([s for s, _, _ in p], [c for _, c, _ in p], [b for _, _, b in p]) for p in parts]
        assert _argmax_by_rule(chunks, B, n) == torch.argmax(mat, dim=1).tolist()


def test_new_symbols_exported_and_bound():
    for s in ('cdx_latent_cycle_fan', 'cdx_ensemble_select'):
        assert hasattr(_cabi.lib, s), f'{s} not exported by libcdx.so'
        assert s in _cabi.SIGNATURES
    assert _cabi.lib.cdx_abi_version() == 2
