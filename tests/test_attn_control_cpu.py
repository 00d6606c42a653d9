"""CPU checks of Prompt-to-Prompt attention control: the token-map helper against a transcription of its rule, the pipeline's
cross_attention_kwargs parsing, and the P2P oracle with no controlled step against the masked oracle's plain lock-step cycle."""
import pytest
import torch

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.attn_control import AttentionControl, replace_token_map
from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
from tests.common import NARROW, maxdiff


def _rule(p, ns, nt, L):
    """The mapper for prompts with a common prefix of p tokens, then a run of ns source / nt target tokens, then a common rest."""
    A = torch.zeros(L, L)
    for i in range(L):
        if i < p:
            A[i, i] = 1.0
        elif i < p + ns:
            if ns == nt:
                A[i, i] = 1.0
            else:
                for j in range(p, min(p + nt, L)):
                    A[i, j] = 1.0 / nt
        elif i + nt - ns < L:
            A[i, i + nt - ns] = 1.0
    return A


@pytest.mark.parametrize('prefix,src_run,tgt_run,rest,L', [
    ([49406, 320], [2368], [1929], [530, 518, 2870, 49407], 12),            # equal runs: one-to-one (a cat -> a dog)
    ([49406, 320], [2368], [1929, 4558], [530, 49407], 12),                 # one token -> two
    ([49406, 320], [2368, 4558, 911], [1929], [530, 49407], 12),            # three tokens -> one: the rest shifts left
    ([49406, 320, 530], [2368], [1929, 4558, 911], [49407], 8),             # run near the end: positions pushed past L dropped
    ([49406, 320, 530], [2368, 911], [1929], [], 6),                        # run at the very end of the prompt
    ([49406, 320, 530], [], [], [49407], 6),                                # identical prompts: the identity
])
def test_replace_token_map_follows_the_rule(prefix, src_run, tgt_run, rest, L):
    A = replace_token_map(prefix + src_run + rest, prefix + tgt_run + rest, L)
    assert A.shape == (L, L) and A.dtype == torch.float32
    assert torch.equal(A, _rule(len(prefix), len(src_run), len(tgt_run), L))


def test_attention_control_steps_and_validation():
    ctl = AttentionControl(0.8, 0.4)
    assert ctl.steps(5) == (4, 2) and ctl.steps(50) == (40, 20) and ctl.self_max_tokens == 256
    for bad in (dict(cross_steps=1.5, self_steps=0.2), dict(cross_steps=0.5, self_steps=-0.1), dict(cross_steps='0.5', self_steps=0.1),
                dict(cross_steps=0.5, self_steps=0.1, self_max_tokens=-1), dict(cross_steps=0.5, self_steps=0.1, token_map=[[1.0]])):
        with pytest.raises(ValueError):
            AttentionControl(**bad)
    with pytest.raises(ValueError):
        AttentionControl(0.5, 0.5, token_map=torch.eye(4)).device_map(2, 5, 'cpu')
    A = AttentionControl(0.5, 0.5, token_map=torch.eye(4)).device_map(3, 4, 'cpu')
    assert A.shape == (3, 4, 4) and A.is_contiguous()


def test_pipeline_kwargs_map_to_the_control():
    parse = CycleDiffusionPipeline._attn_control
    assert parse(None, 1.0, False) is None and parse({'scale': 1.0}, 1.0, False) is None     # no edit_type: today's behaviour
    L = 6
    swap = torch.eye(L)[[0, 2, 1, 3, 4, 5]]
    eq = torch.tensor([1.0, 1.0, 2.0, 1.0, 1.0, 1.0])
    ctl = parse({'edit_type': 'reweight', 'cross_replace_steps': 0.8, 'self_replace_steps': 0.4, 'self_replace_max_tokens': 64,
                 'token_map': swap, 'equalizer': eq}, 1.0, False)
    assert (ctl.cross_steps, ctl.self_steps, ctl.self_max_tokens) == (0.8, 0.4, 64)
    assert torch.equal(ctl.token_map, swap @ torch.diag(eq))
    ctl = parse({'edit_type': 'replace', 'cross_replace_steps': 1.0, 'self_replace_steps': 0.0, 'equalizer': eq.expand(2, L)}, 3.0, False)
    assert torch.equal(ctl.token_map, torch.diag(eq).expand(2, L, L))
    ok = {'edit_type': 'replace', 'cross_replace_steps': 0.5, 'self_replace_steps': 0.5}
    assert parse(ok, 1.0, False).token_map is None
    bad = [({**ok, 'edit_type': 'refine'}, 1.0, False), (ok, 1.0, True), (ok, 0.0, False),
           ({**ok, 'cross_replace_steps': 1.2}, 1.0, False), ({'edit_type': 'replace', 'cross_replace_steps': 0.5}, 1.0, False),
           ({**ok, 'token_map': torch.eye(L)[:4]}, 1.0, False), ({**ok, 'token_map': swap, 'equalizer': torch.ones(L + 1)}, 1.0, False),
           ({**ok, 'local_blend': object()}, 1.0, False), ({**ok, 'edit_type': 'blend'}, 1.0, False)]
    for kw, src_scale, two_phase in bad:
        with pytest.raises(ValueError):
            parse(kw, src_scale, two_phase)


def test_p2p_oracle_at_zero_steps_is_the_plain_cycle():
    """With no controlled step the oracle's one-call-per-step loop is masked_cycle(mask=None), up to the batching of the CPU
    contractions: masked_cycle calls the U-Net once per chain, and fp32 CPU sums depend on the batch (1e-6 .. 2e-6 relative seen).
    A random token map changes nothing when no step is controlled."""
    from oracle import unet_openai
    from tests.masked_oracle import masked_cycle
    from tests.p2p_oracle import p2p_cycle
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    g = torch.Generator().manual_seed(7)
    x0 = torch.randn(2, 4, 8, 8, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(2, 77, 48, generator=g) for _ in range(3))
    with torch.no_grad():
        torch.manual_seed(3)
        y, z = p2p_cycle(usd, NARROW, x0, c_src, c_tgt, uc, 6, 0.1, 3, 1.0, 3.0, 0, 0, token_map=torch.rand(2, 77, 77, generator=g))
        torch.manual_seed(3)
        (y_ref,), z_ref = masked_cycle(lambda x, t, c: unet_openai.unet_forward(usd, NARROW, x, t, c), x0, c_src, c_tgt, uc, 6, 0.1, 3,
                                       1.0, [3.0], None)
    z, z_ref = torch.stack(z, dim=1), torch.stack(z_ref, dim=1)
    rz, ry = maxdiff(z, z_ref) / float(z_ref.abs().max()), maxdiff(y, y_ref) / float(y_ref.abs().max())
    print(f'p2p oracle at zero steps vs masked_cycle: rel|dz| {rz:.2e}  rel|dy| {ry:.2e}')
    assert rz < 5e-6 and ry < 5e-6
