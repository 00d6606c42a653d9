"""CPU checks of Plug-and-Play injection: PnPControl's validation, the pipeline's cross_attention_kwargs parsing for edit_type='pnp',
the oracle's row pairs, and the PnP oracle with no controlled step against the masked oracle's plain cycle."""
import pytest
import torch

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.attn_control import AttentionControl, MutualSelfControl, PnPControl
from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
from tests.common import NARROW, maxdiff


def test_pnp_control_defaults_and_validation():
    ctl = PnPControl()
    assert (ctl.feature_steps, ctl.attention_steps, ctl.feature_blocks, ctl.attention_start_layer) == (0.8, 0.5, (4,), 8)
    assert PnPControl(0, 1, [3, 4], 0) == PnPControl(feature_steps=0, attention_steps=1, feature_blocks=(3, 4), attention_start_layer=0)
    assert PnPControl(feature_blocks=()).feature_blocks == ()
    assert ctl.steps(10) == (8, 5) and ctl.steps(7) == (5, 3)                      # int(f * n), as Prompt-to-Prompt's fractions
    for bad in (dict(feature_steps=-0.1), dict(feature_steps=1.5), dict(attention_steps=2), dict(attention_steps=True),
                dict(feature_steps=None), dict(feature_blocks=(-1,)), dict(feature_blocks=(4, 4)), dict(feature_blocks=(True,)),
                dict(feature_blocks=(4.0,)), dict(feature_blocks=4), dict(feature_blocks='4'), dict(attention_start_layer=-1),
                dict(attention_start_layer=8.0), dict(attention_start_layer=False), dict(attention_start_layer='8')):
        with pytest.raises(ValueError):
            PnPControl(**bad)
    with pytest.raises(AttributeError):                            # frozen
        ctl.feature_steps = 0.5


def test_pipeline_kwargs_map_to_the_pnp_control():
    parse = CycleDiffusionPipeline._attn_control
    assert parse({'edit_type': 'pnp'}, 1.0, False) == PnPControl()
    assert parse({'edit_type': 'pnp'}, 0.0, False) == PnPControl()                 # PnP's unconditional source branch is allowed
    assert parse({'edit_type': 'pnp', 'feature_steps': 0.5, 'attention_steps': 0.25, 'feature_blocks': [3, 5],
                  'attention_start_layer': 10}, 1.0, False) == PnPControl(0.5, 0.25, (3, 5), 10)
    assert parse({'edit_type': 'pnp', 'feature_blocks': ()}, 2.0, False) == PnPControl(feature_blocks=())
    assert isinstance(parse({'edit_type': 'mutual_self'}, 1.0, False), MutualSelfControl)
    assert isinstance(parse({'edit_type': 'replace', 'cross_replace_steps': 0.5, 'self_replace_steps': 0.5}, 1.0, False), AttentionControl)
    ok = {'edit_type': 'pnp', 'feature_steps': 0.8, 'attention_steps': 0.5}
    bad = [({**ok, 'cross_replace_steps': 0.5}, False), ({**ok, 'start_step': 2}, False), ({**ok, 'start_layer': 8}, False),
           ({**ok, 'token_map': torch.eye(4)}, False), ({**ok, 'pnp_f_t': 0.8}, False), (ok, True), ({**ok, 'feature_steps': 1.2}, False),
           ({**ok, 'attention_steps': -0.5}, False), ({**ok, 'feature_blocks': (4, 4)}, False), ({**ok, 'feature_blocks': (-2,)}, False),
           ({**ok, 'attention_start_layer': 2.5}, False), ({**ok, 'attention_start_layer': True}, False), ({'edit_type': 'PnP'}, False)]
    for kw, two_phase in bad:
        with pytest.raises(ValueError):
            parse(kw, 1.0, two_phase)


def test_pnp_pairs_follow_the_row_mapping():
    """Target cond -> source cond; target uncond -> source uncond, or the source's only row when it has no uncond row.  At source
    scale 0 that only row is the source's uncond row, which the oracle runs as a one-row chain."""
    from tests.pnp_oracle import pnp_pairs
    uc = torch.zeros(1)
    assert sorted(pnp_pairs(2, uc, 0.0, 3.0)) == [(2, 0), (3, 1), (4, 0), (5, 1)]      # rows [src u | tgt u | tgt c]
    assert sorted(pnp_pairs(2, uc, 1.0, 3.0)) == [(2, 0), (3, 1), (4, 0), (5, 1)]      # rows [src c | tgt u | tgt c]
    assert sorted(pnp_pairs(2, uc, 2.0, 3.0)) == [(4, 0), (5, 1), (6, 2), (7, 3)]      # rows [src u | src c | tgt u | tgt c]
    assert sorted(pnp_pairs(2, uc, 0.0, 1.0)) == [(2, 0), (3, 1)]                      # rows [src u | tgt c]
    assert sorted(pnp_pairs(2, None, 2.0, 3.0)) == [(2, 0), (3, 1)]                    # no uc: one row per chain


@pytest.mark.parametrize('src_scale', [2.0, 0.0])
def test_pnp_oracle_at_zero_steps_is_the_plain_cycle(src_scale):
    """With no controlled step the oracle is masked_cycle(mask=None) up to the batching of the CPU contractions (the bound of
    test_mutual_oracle_at_n_steps_is_the_plain_cycle); at source scale 0 that pins the oracle's one-row source chain under uc to
    the plain loop's scale-0 source.  One step of either injection changes the edit, and the oracle's hooks are restored."""
    from oracle import unet_openai
    from tests.masked_oracle import masked_cycle
    from tests.pnp_oracle import pnp_cycle
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    g = torch.Generator().manual_seed(7)
    x0 = torch.randn(2, 4, 8, 8, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(2, 77, 48, generator=g) for _ in range(3))
    args = (usd, NARROW, x0, c_src, c_tgt, uc, 6, 0.1, 3, src_scale, 3.0)
    with torch.no_grad():
        torch.manual_seed(3)
        y, z = pnp_cycle(*args, 0, 0, (4,), 0)
        torch.manual_seed(3)
        (y_ref,), z_ref = masked_cycle(lambda x, t, c: unet_openai.unet_forward(usd, NARROW, x, t, c), x0, c_src, c_tgt, uc, 6, 0.1, 3,
                                       src_scale, [3.0], None)
        torch.manual_seed(3)
        y_feat, _ = pnp_cycle(*args, 1, 0, (4,), 0)
        torch.manual_seed(3)
        y_attn, _ = pnp_cycle(*args, 0, 1, (), 8)
    z, z_ref = torch.stack(z, dim=1), torch.stack(z_ref, dim=1)
    rz, ry = maxdiff(z, z_ref) / float(z_ref.abs().max()), maxdiff(y, y_ref) / float(y_ref.abs().max())
    print(f'pnp oracle at zero steps (source scale {src_scale}) vs masked_cycle: rel|dz| {rz:.2e}  rel|dy| {ry:.2e}')
    assert rz < 5e-6 and ry < 5e-6
    assert maxdiff(y_feat, y) > 1e-4 and maxdiff(y_attn, y) > 1e-4
    assert (unet_openai._resblock.__name__, unet_openai._attention.__name__, unet_openai.unet_forward.__name__) == \
        ('_resblock', '_attention', 'unet_forward')
