"""Host-side plan of the lock-step ensemble search of the text wrappers (SURVEY 8f-2).  Free of the engine: it only decides the
order, the U-Net rows and the chunks, and replays the random draws.

  member order      SDW:189-204: for trial, for encoder scale, for skip (skip innermost) -- the order of encode()'s z list
  candidate index   SDW:146-165, 219-249: member * n_dec + k for decoder scale k -- the column of the [B, candidates] score matrix
  source chain      one (member, sample) pair's DPM-Encoder chain; it drives the K = n_dec decoder chains of that pair
  rows per chain    guidance_rows(encoder scale) + sum_k guidance_rows(decoder scale k)
  chunk             source chains of one skip (one schedule), in member then sample order, filled up to ``row_budget`` U-Net rows
                    per call; at least one chain
"""
import torch


def guidance_rows(scale):
    """U-Net rows a chain needs per step: scale 1 runs the cond row only, scale 0 the uncond row only (the reference's single-forward
    branches, ddim.py:550-551), any other scale both (ddim.py:555-559)."""
    return 1 if float(scale) in (0.0, 1.0) else 2


class Chunk:
    def __init__(self, skip):
        self.skip, self.chains, self.rows = skip, [], 0          # chains: [(member, sample)]


class EnsemblePlan:
    def __init__(self, n_trials, enc_scales, skips, dec_scales, bsz, refine_steps, row_budget):
        """refine_steps: {skip: steps of that skip's loop}.  row_budget: U-Net rows per call a chunk may fill."""
        self.members = [(t, float(es), int(sk)) for t in range(n_trials) for es in enc_scales for sk in skips]
        self.dec_scales = [float(s) for s in dec_scales]
        self.n_dec = len(self.dec_scales)
        self.n_candidates = len(self.members) * self.n_dec
        self.bsz = bsz
        self.refine_steps = {int(k): int(v) for k, v in refine_steps.items()}
        self.chunks = []
        for skip in dict.fromkeys(int(s) for s in skips):
            chunk = None
            for m, (_, _, sk) in enumerate(self.members):
                if sk != skip:
                    continue
                r = self.chain_rows(m)
                for b in range(bsz):
                    if chunk is None or (chunk.chains and chunk.rows + r > row_budget):
                        chunk = Chunk(skip)
                        self.chunks.append(chunk)
                    chunk.chains.append((m, b))
                    chunk.rows += r

    def chain_rows(self, m):
        return guidance_rows(self.members[m][1]) + sum(guidance_rows(s) for s in self.dec_scales)

    def candidate(self, m, k):
        return m * self.n_dec + k

    def sample_forwards(self):
        """U-Net sample-forwards of the lock-step search for the whole batch."""
        return sum(c.rows * self.refine_steps[c.skip] for c in self.chunks)

    def two_phase_sample_forwards(self):
        """The same for encode() + forward() with batched members: cdx_latent_loop_ens runs both CFG segments for every chain."""
        return sum(self.bsz * self.refine_steps[sk] * 2 * (1 + self.n_dec) for _, _, sk in self.members)


class MemberNoise:
    """The DPM-Encoder draws of every member, made with the calls and in the order encode() makes them (``draw(skip)`` -> [n+1, B,
    C,h,w], member order), then replayed per chunk from the generator state saved before each member, so only one chunk's noise
    exists at a time.  The CPU generator is left where encode() leaves it."""

    def __init__(self, plan, draw):
        self.plan, self.draw, self.states = plan, draw, []
        for _, _, skip in plan.members:
            self.states.append(torch.get_rng_state())
            draw(skip)
        self.end = torch.get_rng_state()

    def chunk(self, chunk):
        """-> noise [n+1, n_src, C,h,w] of the chunk's source chains."""
        cols, member, nz = [], None, None
        for m, b in chunk.chains:
            if m != member:
                torch.set_rng_state(self.states[m])
                member, nz = m, self.draw(chunk.skip)
            cols.append(nz[:, b])
        torch.set_rng_state(self.end)
        return torch.stack(cols, dim=1)


def select_better(sa, ia, sb, ib):
    """The rule of ensemble_select_kernel: does candidate (score sa, index ia) beat (sb, ib) under torch.argmax?  Larger wins, NaN
    beats any number, ties and NaN pairs go to the lower index; ib < 0 is an empty slot."""
    if ia < 0:
        return False
    if ib < 0:
        return True
    na, nb = sa != sa, sb != sb
    if na or nb:
        return na and (not nb or ia < ib)
    return sa > sb or (sa == sb and ia < ib)
