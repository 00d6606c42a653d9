"""CPU checks of Prompt-to-Prompt's refine edit: the alignment mapper on worked examples, the pipeline's cross_attention_kwargs for
refine, AttentionControl's own_weight, and the refine oracle against the replace oracle and the plain cycle."""
import pytest
import torch

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.attn_control import AttentionControl, refine_token_map
from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
from tests.common import NARROW, maxdiff

BOS, EOS = 49406, 49407
A_, CAT, DOG, FLUFFY, ON, GRASS, SNOW = 320, 2368, 1929, 21416, 525, 3321, 2583


def _src_of(A, n):
    """m(j) for target positions j < n from a 0/1 map: the source row of column j's one, -1 for an empty column."""
    return [int(A[:, j].argmax()) if float(A[:, j].sum()) > 0 else -1 for j in range(n)]


@pytest.mark.parametrize('src,tgt,expect', [
    ([BOS, A_, CAT, EOS], [BOS, A_, FLUFFY, CAT, EOS], [0, 1, -1, 2, 3]),                       # insertion
    ([BOS, A_, CAT, EOS], [BOS, A_, DOG, EOS], [0, 1, -1, 3]),                                  # substitution: drop + insertion
    ([BOS, A_, FLUFFY, CAT, EOS], [BOS, A_, CAT, EOS], [0, 1, 3, 4]),                           # deletion
    ([BOS, A_, CAT, ON, GRASS, EOS], [BOS, A_, DOG, ON, SNOW, EOS], [0, 1, -1, 3, -1, 5]),      # two substitutions
    ([BOS, A_, CAT, EOS], [BOS, A_, CAT, EOS], [0, 1, 2, 3]),                                   # identical prompts
])
def test_refine_token_map_aligns_the_examples(src, tgt, expect):
    L = 12
    A = refine_token_map(src, tgt, L)
    assert A.shape == (L, L) and A.dtype == torch.float32
    assert set(A.unique().tolist()) <= {0.0, 1.0} and bool((A.sum(dim=0) <= 1).all())
    assert _src_of(A, len(tgt)) == expect
    for j in range(len(tgt), L):                   # padding to padding
        assert _src_of(A, L)[j] == j
    if src == tgt:
        assert torch.equal(A, torch.eye(L))


def test_refine_token_map_bos_eos_and_truncation():
    # BOS and EOS align with each other even when every word differs
    A = refine_token_map([BOS, CAT, EOS], [BOS, DOG, GRASS, EOS], 8)
    assert _src_of(A, 4) == [0, -1, -1, 2]
    # L shorter than the prompts: positions past L are dropped, on either side
    A = refine_token_map([BOS, A_, FLUFFY, CAT, EOS], [BOS, A_, CAT, EOS], 3)
    assert A.shape == (3, 3) and _src_of(A, 3) == [0, 1, -1]        # target 2 ("cat") aligns to source 3, past L
    A = refine_token_map([BOS, A_, CAT, EOS], [BOS, A_, FLUFFY, CAT, EOS], 4)
    assert _src_of(A, 4) == [0, 1, -1, 2]
    # L == len(tgt): no padding column
    A = refine_token_map([BOS, CAT, EOS], [BOS, A_, CAT, EOS], 4)
    assert _src_of(A, 4) == [0, -1, 1, 2]


def test_own_weight_validation():
    L = 5
    ctl = AttentionControl(0.5, 0.2, token_map=torch.eye(L), own_weight=torch.zeros(L))
    w = ctl.device_weight(3, L, 'cpu')
    assert w.shape == (3, L) and w.is_contiguous() and w.dtype == torch.float32
    assert AttentionControl(0.5, 0.2).device_weight(3, L, 'cpu') is None
    with pytest.raises(ValueError):
        AttentionControl(0.5, 0.2, own_weight=[1.0] * L)
    for bad in (torch.ones(L + 1), torch.ones(2, L), torch.ones(3, L, 1), torch.tensor([1.0, -0.5, 0, 0, 0]),
                torch.tensor([1.0, float('inf'), 0, 0, 0])):
        with pytest.raises(ValueError):
            AttentionControl(0.5, 0.2, own_weight=bad).device_weight(3, L, 'cpu')
    _, A, w = AttentionControl(0.5, 0.2, token_map=torch.eye(L), own_weight=torch.ones(L)).c_struct(4, 3, L, 'cpu')
    assert A.shape == (3, L, L) and w.shape == (3, L)


def test_pipeline_refine_kwargs():
    parse = CycleDiffusionPipeline._attn_control
    L = 6
    A = refine_token_map([BOS, A_, CAT, EOS], [BOS, A_, FLUFFY, CAT, EOS], L)
    base = {'edit_type': 'refine', 'cross_replace_steps': 0.8, 'self_replace_steps': 0.4}
    ctl = parse({**base, 'token_map': A}, 1.0, False)
    assert torch.equal(ctl.token_map, A)
    assert torch.equal(ctl.own_weight, torch.tensor([0.0, 0.0, 1.0, 0.0, 0.0, 0.0]))
    # the equalizer scales both terms: A . diag(eq) and w = (1 - colsum(A)) . eq
    eq = torch.tensor([1.0, 1.0, 2.5, 0.5, 1.0, 1.0])
    ctl = parse({**base, 'token_map': A, 'equalizer': eq, 'self_replace_max_tokens': 64}, 1.0, False)
    assert torch.equal(ctl.token_map, A @ torch.diag(eq)) and ctl.self_max_tokens == 64
    assert torch.equal(ctl.own_weight, (1 - A.sum(0)) * eq)
    # [B, L, L] maps and [B, L] equalizers give [B, L] weights; a fractional map keeps the rest of each column
    Ab = torch.stack([A, torch.eye(L) * 0.25])
    eqb = torch.stack([eq, torch.ones(L) * 2])
    ctl = parse({**base, 'token_map': Ab, 'equalizer': eqb}, 3.0, False)
    assert torch.equal(ctl.token_map, Ab * eqb.unsqueeze(-2))
    assert torch.equal(ctl.own_weight, torch.stack([(1 - A.sum(0)) * eq, torch.full((L,), 1.5)]))
    ctl = parse({**base, 'token_map': A, 'equalizer': eqb}, 1.0, False)
    assert ctl.token_map.shape == (2, L, L) and ctl.own_weight.shape == (2, L)
    # replace and reweight carry no own weight
    assert parse({**base, 'edit_type': 'replace', 'token_map': A}, 1.0, False).own_weight is None
    assert parse({**base, 'edit_type': 'reweight', 'token_map': A, 'equalizer': eq}, 1.0, False).own_weight is None
    # rejections: no map, column sums outside [0, 1], and replace's own
    over = A.clone()
    over[1, 3] = 0.5                                   # column 3 sums to 1.5
    neg = torch.eye(L)
    neg[2, 2] = -0.25                                  # column 2 sums to -0.25
    bad = [({**base}, 1.0, False), ({**base, 'token_map': over}, 1.0, False), ({**base, 'token_map': neg}, 1.0, False),
           ({**base, 'token_map': A}, 1.0, True), ({**base, 'token_map': A}, 0.0, False),
           ({**base, 'token_map': A, 'local_blend': object()}, 1.0, False), ({**base, 'token_map': A[:4]}, 1.0, False),
           ({**base, 'token_map': A, 'equalizer': torch.ones(L + 1)}, 1.0, False),
           ({**base, 'token_map': A, 'equalizer': -torch.ones(L)}, 1.0, False)]
    for kw, src_scale, two_phase in bad:
        with pytest.raises(ValueError):
            parse(kw, src_scale, two_phase)
    # within 1e-6 of the bounds is accepted
    near = torch.eye(L) * (1 + 5e-7)
    assert parse({**base, 'token_map': near}, 1.0, False).own_weight is not None


def _case(seed=7):
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(2, 4, 8, 8, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(2, 77, 48, generator=g) for _ in range(3))
    return usd, g, x0, c_src, c_tgt, uc


def test_refine_oracle_at_zero_weight_is_the_replace_oracle():
    """own_weight == 0 adds attn_own * 0 to the replace oracle's probabilities: the same loop, bit for bit."""
    from tests.p2p_oracle import p2p_cycle
    from tests.p2p_refine_oracle import p2p_refine_cycle
    usd, g, x0, c_src, c_tgt, uc = _case()
    A = torch.rand(2, 77, 77, generator=g) / 77
    with torch.no_grad():
        torch.manual_seed(3)
        y, z = p2p_refine_cycle(usd, NARROW, x0, c_src, c_tgt, uc, 6, 0.1, 3, 1.0, 3.0, 2, 1, 16, A, torch.zeros(2, 77))
        torch.manual_seed(3)
        y_ref, z_ref = p2p_cycle(usd, NARROW, x0, c_src, c_tgt, uc, 6, 0.1, 3, 1.0, 3.0, 2, 1, 16, A)
    assert torch.equal(y, y_ref) and all(torch.equal(a, b) for a, b in zip(z, z_ref))


def test_refine_oracle_without_source_term_is_the_plain_cycle():
    """A == 0 and own_weight == 1 on cross-attention only is the uncontrolled attention: the masked oracle's plain cycle, within
    test_p2p_oracle_at_zero_steps_is_the_plain_cycle's bound (fp32 CPU sums depend on the batching)."""
    from oracle import unet_openai
    from tests.masked_oracle import masked_cycle
    from tests.p2p_refine_oracle import p2p_refine_cycle
    usd, g, x0, c_src, c_tgt, uc = _case(8)
    with torch.no_grad():
        torch.manual_seed(4)
        y, z = p2p_refine_cycle(usd, NARROW, x0, c_src, c_tgt, uc, 6, 0.1, 3, 1.0, 3.0, 3, 0, token_map=torch.zeros(2, 77, 77),
                                own_weight=torch.ones(2, 77))
        torch.manual_seed(4)
        (y_ref,), z_ref = masked_cycle(lambda x, t, c: unet_openai.unet_forward(usd, NARROW, x, t, c), x0, c_src, c_tgt, uc, 6, 0.1, 3,
                                       1.0, [3.0], None)
    z, z_ref = torch.stack(z, dim=1), torch.stack(z_ref, dim=1)
    rz, ry = maxdiff(z, z_ref) / float(z_ref.abs().max()), maxdiff(y, y_ref) / float(y_ref.abs().max())
    print(f'refine oracle with A = 0, w = 1 vs masked_cycle: rel|dz| {rz:.2e}  rel|dy| {ry:.2e}')
    assert rz < 5e-6 and ry < 5e-6
