"""The autocast fixtures (tests/golden/make_golden_autocast.py) on the CPU: their fp32 arm is the existing oracle's result on this
project's weights and inputs (same bounds as test_oracle_golden.py), and their autocast arm differs from it by an fp16-sized
amount."""
import numpy as np
import pytest
import torch

from cycle_diffusion_b200 import specs
from oracle import dpm_encoder, unet_openai, vae_kl
from tests.common import NARROW, VAE_SMALL, WIDE, golden, maxdiff, wsum

torch.set_num_threads(8)


def rel(a, b):
    return maxdiff(a, b) / float(b.abs().max())


@pytest.mark.parametrize('tag,cfg', [('wide', WIDE), ('narrow', NARROW)])
def test_unet_fixture(tag, cfg):
    g = golden('unet_sd_autocast')
    sd = specs.synth_state_dict(specs.openai_unet_params(cfg), int(g[f'seed_{tag}']))
    assert np.allclose(wsum(sd), g[f'wsum_{tag}'], rtol=1e-12), 'synthetic weight generator drifted'
    with torch.no_grad():
        y = unet_openai.unet_forward(sd, cfg, g[f'x_{tag}'], g[f't_{tag}'], g[f'ctx_{tag}'])
    y32 = g[f'y32_{tag}']
    assert maxdiff(y, y32) <= 2e-5 * max(1.0, float(y32.abs().max()))
    assert 1e-4 < rel(g[f'yac_{tag}'], y32) < 3e-2


def test_vae_fixture():
    g = golden('vae_autocast')
    sd = specs.synth_state_dict(specs.kl_vae_params(VAE_SMALL), int(g['seed']))
    assert np.allclose(wsum(sd), g['wsum'], rtol=1e-12)
    with torch.no_grad():
        m = vae_kl.encode_moments(sd, VAE_SMALL, g['img'])
        r = vae_kl.decode(sd, VAE_SMALL, g['z'])
    assert maxdiff(m, g['moments32']) <= 2e-5 * max(1.0, float(g['moments32'].abs().max()))
    assert maxdiff(r, g['rec32']) <= 2e-5 * max(1.0, float(g['rec32'].abs().max()))
    assert 1e-4 < rel(g['momentsac'], g['moments32']) < 3e-2
    assert 1e-4 < rel(g['recac'], g['rec32']) < 3e-2


def test_ddim_cycle_fixture():
    g = golden('ddim_cycle_autocast')
    S, skip, wb, enc_scale, dec_scale, seed = [float(v) for v in g['cfg']]
    S, skip, wb, seed = int(S), int(skip), int(wb), int(seed)
    assert wb - skip - 1 >= S - skip, 'every step recovered: the lock-step path accepts this cycle'
    sd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    unet = lambda x, t, c: unet_openai.unet_forward(sd, NARROW, x, t, c)
    B = g['x0'].shape[0]
    torch.manual_seed(seed)
    with torch.no_grad():
        z = torch.stack(dpm_encoder.latent_encode(unet, g['x0'], g['c_src'], g['uc'], S, 0.1, skip, wb, enc_scale), dim=1).view(B, -1)
        assert maxdiff(z, g['z32']) <= 1e-4 * float(g['z32'].abs().max())
        eps_list = g['z32'].view(B, wb - skip, 4, 16, 16)
        tgt = dpm_encoder.latent_decode(unet, eps_list[:, 0], eps_list[:, 1:], g['c_tgt'], g['uc'], S, 0.1, skip, dec_scale)
    assert maxdiff(tgt, g['tgt32']) <= 1e-4
    assert 1e-4 < rel(g['zac'], g['z32']) < 3e-2
    assert 1e-4 < rel(g['tgtac'], g['tgt32']) < 3e-2
