"""Masked editing without a GPU: the masked oracle loop is the unmasked oracle loop at a mask of ones (and so matches the
reference-generated ddim_cycle_narrow fixture), it ends at x0 under a mask of zeros, and the new C ABI symbols are exported."""
import pytest
import torch

from cycle_diffusion_b200 import _cabi, specs
from oracle import dpm_encoder, unet_openai
from tests.common import NARROW, golden, maxdiff
from tests.masked_oracle import masked_cycle


def _case(tag):
    g = golden('ddim_cycle_narrow')
    S, skip, wb, enc_scale, dec_scale, seed = [float(v) for v in g[f'cfg_{tag}']]
    S, skip, wb, seed = int(S), int(skip), int(wb), int(seed)
    if wb - skip - 1 < S - skip:
        pytest.skip('the lock-step loop needs every step recovered')
    sd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    unet = lambda x, t, c: unet_openai.unet_forward(sd, NARROW, x, t, c)
    return g, unet, S, skip, wb, enc_scale, dec_scale, seed


@pytest.mark.parametrize('tag', ['a', 'b'])
def test_mask_of_ones_is_the_unmasked_oracle_loop(tag):
    g, unet, S, skip, wb, enc_scale, dec_scale, seed = _case(tag)
    ones = torch.ones(g['x0'].shape[0], 1, *g['x0'].shape[2:])
    with torch.no_grad():
        torch.manual_seed(seed)
        (y,), z_list = masked_cycle(unet, g['x0'], g['c_src'], g['c_tgt'], g['uc'], S, 0.1, skip, enc_scale, [dec_scale], ones)
        torch.manual_seed(seed)
        z_ref = dpm_encoder.latent_encode(unet, g['x0'], g['c_src'], g['uc'], S, 0.1, skip, wb, enc_scale)
        eps = torch.stack(z_ref[1:], dim=1)
        y_ref = dpm_encoder.latent_decode(unet, z_ref[0], eps, g['c_tgt'], g['uc'], S, 0.1, skip, dec_scale)
    assert all(torch.equal(a, b) for a, b in zip(z_list, z_ref)) and len(z_list) == len(z_ref)
    assert torch.equal(y, y_ref)
    assert maxdiff(y, g[f'tgt_{tag}']) <= 1e-4                  # test_oracle_golden.py's bound for the same loop


@pytest.mark.parametrize('tag', ['a', 'b'])
def test_mask_of_zeros_ends_at_x0(tag):
    g, unet, S, skip, _, enc_scale, dec_scale, seed = _case(tag)
    zeros = torch.zeros(g['x0'].shape[0], 1, *g['x0'].shape[2:])
    torch.manual_seed(seed)
    with torch.no_grad():
        ys, _ = masked_cycle(unet, g['x0'], g['c_src'], g['c_tgt'], g['uc'], S, 0.1, skip, enc_scale, [dec_scale, 0.0], zeros)
    assert all(torch.equal(y, g['x0']) for y in ys)


def test_blend_exact_ends_and_soft_values():
    from tests.masked_oracle import blend
    y, x = torch.randn(2, 4, 3, 5), torch.randn(2, 4, 3, 5)
    m = torch.tensor([0.0, 1.0, 0.25, 0.5, 1.0]).view(1, 1, 1, 5).expand(2, 1, 3, 5)
    out = blend(y, x, m)
    assert torch.equal(out[..., 0], x[..., 0]) and torch.equal(out[..., 1], y[..., 1]) and torch.equal(out[..., 4], y[..., 4])
    assert torch.equal(out[..., 2], x[..., 2] + 0.25 * (y[..., 2] - x[..., 2]))


def test_masked_symbols_are_exported():
    for s in ('cdx_cycle_lockstep_masked', 'cdx_latent_cycle_fan_masked', 'cdx_mask_pool', 'cdx_mask_composite'):
        assert s in _cabi.SIGNATURES and hasattr(_cabi.lib, s)
    from cycle_diffusion_b200.engine import Engine, UNet
    import inspect
    assert 'mask' in inspect.signature(UNet.cycle_lockstep).parameters and 'mask' in inspect.signature(UNet.cycle_fan).parameters
    assert hasattr(Engine, 'mask_pool') and hasattr(Engine, 'mask_composite')
