"""CPU checks of mutual self-attention control (MasaCtrl): MutualSelfControl's validation, the pipeline's cross_attention_kwargs
parsing for edit_type='mutual_self', and the mutual oracle with no controlled step against the masked oracle's plain cycle."""
import pytest
import torch

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.attn_control import AttentionControl, MutualSelfControl
from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
from tests.common import NARROW, maxdiff


def test_mutual_self_control_defaults_and_validation():
    ctl = MutualSelfControl()
    assert (ctl.start_step, ctl.start_layer) == (4, 10)
    assert MutualSelfControl(0, 0) == MutualSelfControl(start_step=0, start_layer=0)
    for bad in (dict(start_step=-1), dict(start_layer=-1), dict(start_step=True), dict(start_layer=False), dict(start_step=1.0),
                dict(start_layer='10'), dict(start_step=None)):
        with pytest.raises(ValueError):
            MutualSelfControl(**bad)
    with pytest.raises(AttributeError):                            # frozen
        ctl.start_step = 2


def test_pipeline_kwargs_map_to_the_mutual_control():
    parse = CycleDiffusionPipeline._attn_control
    assert parse({'edit_type': 'mutual_self'}, 1.0, False) == MutualSelfControl(4, 10)
    assert parse({'edit_type': 'mutual_self', 'start_step': 0, 'start_layer': 3}, 1.0, False) == MutualSelfControl(0, 3)
    assert parse({'edit_type': 'mutual_self', 'start_layer': 16}, 0.0, False) == MutualSelfControl(4, 16)
    assert isinstance(parse({'edit_type': 'replace', 'cross_replace_steps': 0.5, 'self_replace_steps': 0.5}, 1.0, False), AttentionControl)
    ok = {'edit_type': 'mutual_self', 'start_step': 2, 'start_layer': 10}
    bad = [({**ok, 'cross_replace_steps': 0.5}, False), ({**ok, 'self_replace_steps': 0.5}, False), ({**ok, 'token_map': torch.eye(4)}, False),
           ({**ok, 'equalizer': torch.ones(4)}, False), ({**ok, 'start_steps': 3}, False), ({**ok, 'local_blend': object()}, False),
           (ok, True), ({**ok, 'start_step': -1}, False), ({**ok, 'start_layer': 2.5}, False), ({**ok, 'start_step': True}, False),
           ({'edit_type': 'mutual'}, False)]
    for kw, two_phase in bad:
        with pytest.raises(ValueError):
            parse(kw, 1.0, two_phase)


def test_mutual_pairs_follow_the_row_mapping():
    """Target cond -> source cond; target uncond -> source uncond, or the source's cond row when it runs without one."""
    from tests.mutual_oracle import mutual_pairs
    uc = torch.zeros(1)
    assert sorted(mutual_pairs(2, uc, 1.0, 3.0)) == [(2, 0), (3, 1), (4, 0), (5, 1)]      # rows [src c | tgt u | tgt c]
    assert sorted(mutual_pairs(2, uc, 2.0, 3.0)) == [(4, 0), (5, 1), (6, 2), (7, 3)]      # rows [src u | src c | tgt u | tgt c]
    assert sorted(mutual_pairs(2, uc, 2.0, 1.0)) == [(4, 2), (5, 3)]                      # rows [src u | src c | tgt c]
    assert sorted(mutual_pairs(2, None, 2.0, 3.0)) == [(2, 0), (3, 1)]                    # no uc: one row per chain


def test_mutual_oracle_at_n_steps_is_the_plain_cycle():
    """With start_step at the loop's step count nothing is controlled: the oracle is masked_cycle(mask=None) up to the batching of
    the CPU contractions (the bound of test_p2p_oracle_at_zero_steps_is_the_plain_cycle).  Every layer is counted, so a start_layer
    of 0 would control the first call's layers; at step n it does not."""
    from oracle import unet_openai
    from tests.masked_oracle import masked_cycle
    from tests.mutual_oracle import mutual_cycle
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    g = torch.Generator().manual_seed(7)
    x0 = torch.randn(2, 4, 8, 8, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(2, 77, 48, generator=g) for _ in range(3))
    n = 6 - 3
    with torch.no_grad():
        torch.manual_seed(3)
        y, z = mutual_cycle(usd, NARROW, x0, c_src, c_tgt, uc, 6, 0.1, 3, 2.0, 3.0, n, 0)
        torch.manual_seed(3)
        (y_ref,), z_ref = masked_cycle(lambda x, t, c: unet_openai.unet_forward(usd, NARROW, x, t, c), x0, c_src, c_tgt, uc, 6, 0.1, 3,
                                       2.0, [3.0], None)
        torch.manual_seed(3)
        y_ctl, _ = mutual_cycle(usd, NARROW, x0, c_src, c_tgt, uc, 6, 0.1, 3, 2.0, 3.0, n - 1, 0)
    z, z_ref = torch.stack(z, dim=1), torch.stack(z_ref, dim=1)
    rz, ry = maxdiff(z, z_ref) / float(z_ref.abs().max()), maxdiff(y, y_ref) / float(y_ref.abs().max())
    print(f'mutual oracle at n steps vs masked_cycle: rel|dz| {rz:.2e}  rel|dy| {ry:.2e}')
    assert rz < 5e-6 and ry < 5e-6
    assert maxdiff(y_ctl, y) > 1e-4                                  # one controlled step does change the edit
    assert unet_openai._attention.__name__ == '_attention' and unet_openai.unet_forward.__name__ == 'unet_forward'
