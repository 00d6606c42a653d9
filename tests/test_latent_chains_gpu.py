"""Identities between the latent loop entry points that follow from their sharing one chain driver and one step kernel: the
single-image cycle is the fan-out loop with one target per source, the DPM-Encoder is its source half and the decoder its target
half."""
import pytest
import torch

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.wrappers import encode_noise
from tests.common import NARROW, maxdiff

pytestmark = pytest.mark.gpu

B = 2


@pytest.fixture(scope='module')
def unet():
    from cycle_diffusion_b200.engine import Engine, UNet
    return UNet(Engine(0), NARROW, 'openai').load_state_dict(specs.synth_state_dict(specs.openai_unet_params(NARROW), 11))


@pytest.fixture(scope='module')
def sched():
    from cycle_diffusion_b200.schedule import DDIMSchedule
    return DDIMSchedule(6, 0.1, 2)


@pytest.fixture(scope='module')
def inputs(sched):
    g = torch.Generator().manual_seed(7)
    x0 = torch.randn(B, 4, 16, 16, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(B, 77, 48, generator=g) for _ in range(3))
    torch.manual_seed(8)
    return x0, c_src, c_tgt, uc, encode_noise(sched, sched.refine_steps, x0.shape)


@pytest.mark.parametrize('src_scale,tgt_scale', [(1.0, 3.0), (3.0, 0.0), (2.0, 5.0)])
def test_fan_with_one_target_is_the_lockstep_cycle(unet, sched, inputs, src_scale, tgt_scale):
    """cycle_fan with K = 1 and the same scale on every chain lays out the rows of cycle_lockstep: latent and z are equal."""
    x0, c_src, c_tgt, uc, noise = inputs
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise, return_z=True)
    out_f, z_f = unet.cycle_fan(x0, c_src, c_tgt, uc, [src_scale] * B, [[tgt_scale]] * B, sched, noise, return_z=True)
    assert torch.isfinite(out).all() and torch.isfinite(z).all()
    assert torch.equal(out_f, out) and torch.equal(z_f, z)


def test_fan_is_encode_then_decode_per_target_scale(unet, sched, inputs):
    """The z a fan-out loop returns is latent_encode's for the same noise, and latent_decode of that z under each target scale is
    the fan's latent for it (bounds of test_lockstep_driver_vs_reference_fixture_and_two_phase: the U-Net batch differs)."""
    x0, c_src, c_tgt, uc, noise = inputs
    src_scale, dec = 3.0, [1.0, 0.0, 3.0]
    out, z = unet.cycle_fan(x0, c_src, c_tgt, uc, [src_scale] * B, [dec] * B, sched, noise, return_z=True)
    z2 = unet.latent_encode(x0, c_src, uc, src_scale, sched, sched.refine_steps, noise)
    rz = maxdiff(z.cpu(), z2.cpu()) / float(z2.abs().max())
    out = out.view(B, len(dec), *x0.shape[1:])
    dx = [maxdiff(out[:, k].cpu(), unet.latent_decode(z, c_tgt, uc, s, sched).cpu()) for k, s in enumerate(dec)]
    print(f'fan vs encode / decode: rel|dz| {rz:.2e}  |dx| per target scale {[f"{d:.2e}" for d in dx]}')
    assert rz < 2e-5 and max(dx) < 1e-4
