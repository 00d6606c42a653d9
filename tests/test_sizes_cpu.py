"""CPU checks for rectangular images: the oracle restatement against the rectangular reference fixtures
(tests/golden/make_golden_rect.py), and the C ABI's rectangular first-stage entry points."""
import numpy as np
import torch

from cycle_diffusion_b200 import _cabi, specs
from oracle import unet_openai, vae_kl
from tests.common import NARROW, VAE_SMALL, WIDE, golden, maxdiff, wsum

torch.set_num_threads(8)


def test_rect_symbols_exported_and_bound():
    for s in ('cdx_vae_encode_hw', 'cdx_vae_decode_hw'):
        assert hasattr(_cabi.lib, s), f'{s} not exported by libcdx.so'
        assert s in _cabi.SIGNATURES
    assert _cabi.lib.cdx_abi_version() == 2


def test_oracle_unets_rect():
    for name, cfg in (('unet_sd_rect', NARROW), ('unet_sd_wide_rect', WIDE)):
        g = golden(name)
        assert tuple(g['x'].shape[2:]) == (24, 40)
        sd = specs.synth_state_dict(specs.openai_unet_params(cfg), int(g['seed']))
        assert np.allclose(wsum(sd), g['wsum'], rtol=1e-12), 'synthetic weight generator drifted'
        with torch.no_grad():
            y = unet_openai.unet_forward(sd, cfg, g['x'], g['t'], g['ctx'])
        assert maxdiff(y, g['y']) <= 2e-5 * max(1.0, float(g['y'].abs().max())), name


def test_oracle_vae_rect():
    g = golden('vae_rect')
    sd = specs.synth_state_dict(specs.kl_vae_params(VAE_SMALL), int(g['seed']))
    assert np.allclose(wsum(sd), g['wsum'], rtol=1e-12)
    with torch.no_grad():
        m = vae_kl.encode_moments(sd, VAE_SMALL, g['img'])
        r = vae_kl.decode(sd, VAE_SMALL, g['z'])
    assert m.shape == (1, 8, 12, 20) and r.shape == (1, 3, 96, 160)
    assert maxdiff(m, g['moments']) <= 2e-5 * max(1.0, float(g['moments'].abs().max()))
    assert maxdiff(r, g['rec']) <= 2e-5 * max(1.0, float(g['rec'].abs().max()))
