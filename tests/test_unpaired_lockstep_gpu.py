"""Unpaired translation in lock-step (UnsupervisedTranslation.forward -> wrapper.cycle): bit-identity with the two-phase
``target(source.encode(image))`` on one and on two engines, chunk boundaries, parity with the CPU oracle's two-model restatement,
flat device memory in es_steps, and the fall-back to the two-phase path for mismatched schedules."""
import pytest
import torch

from cycle_diffusion_b200 import specs, wrappers
from cycle_diffusion_b200.engine import Engine, UNet
from cycle_diffusion_b200.models import UnsupervisedTranslation
from cycle_diffusion_b200.wrappers import lockstep_compatible
from tests.common import maxdiff
from tests.test_ldm_uncond_gpu import UNCOND_SMALL, VQ_SMALL
from tests.test_unet_ddpm_gpu import DDPM_SMALL

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def eng():
    return Engine(0)


@pytest.fixture(scope='module')
def eng2():
    return Engine(0)


def _family(family):
    if family == 'iddpm':
        cfg = specs.iddpm_config(64)
        return cfg, specs.iddpm_unet_params(cfg), 'afhqcat64', 'afhqdog64', 64
    return DDPM_SMALL, specs.ddpm_unet_params(DDPM_SMALL), 'celeba_hq_32', 'celeba_hq_32', 32


_NETS = {}


def _net(e, family, seed):
    key = (id(e), family, seed)
    if key not in _NETS:
        cfg, params, _, _, _ = _family(family)
        _NETS[key] = UNet(e, cfg, family).load_state_dict(specs.synth_state_dict(params, seed))
    return _NETS[key]


def _pixel_model(family, kw, e_src, e_tgt, target_kw=None):
    _, _, src_name, tgt_name, R = _family(family)
    gan = dict(gan_type='DDPM_DDIM', source_model_type=src_name, target_model_type=tgt_name, **kw)
    return UnsupervisedTranslation(dict(gan=gan), source_kwargs=dict(unet=_net(e_src, family, 31), image_size=R),
                                   target_kwargs=dict(unet=_net(e_tgt, family, 32), image_size=R, **(target_kw or {}))).eval()


def _translate(m, img, seed):
    torch.manual_seed(seed)
    (_, out), _, _ = m(torch.zeros(img.shape[0]), original_image=img)
    torch.manual_seed(seed)
    ref = m.target_gan_wrapper(z=m.source_gan_wrapper.encode(image=img))
    return out, ref


DDIM = dict(sample_type='ddim', eta=0.1, custom_steps=20, es_steps=8)
DDPM = dict(sample_type='ddpm', eta=None, custom_steps=20, es_steps=6)
REFINE = dict(refine_steps=3, refine_iterations=2)
CASES = [('iddpm', DDIM), ('iddpm', DDPM), ('iddpm', dict(DDIM, **REFINE)), ('iddpm', dict(DDPM, **REFINE)),
         ('ddpm', dict(sample_type='ddim', eta=0.1, custom_steps=10, es_steps=10))]


@pytest.mark.parametrize('engines', ['one', 'two'])
@pytest.mark.parametrize('family,kw', CASES)
def test_pixel_lockstep_equals_two_phase(eng, eng2, monkeypatch, family, kw, engines):
    monkeypatch.setattr(wrappers, 'LOCKSTEP_CHUNK', 3)          # several chunks: both pinned buffers in use
    m = _pixel_model(family, kw, eng, eng if engines == 'one' else eng2)
    assert lockstep_compatible(m.source_gan_wrapper, m.target_gan_wrapper)
    R = m.source_gan_wrapper.resolution
    img = torch.rand(2, 3, R, R, generator=torch.Generator().manual_seed(1))
    out, ref = _translate(m, img, 7)
    assert out.shape == (2, 3, R, R) and torch.isfinite(out).all()
    assert torch.equal(out, ref), f'|d| {maxdiff(out.cpu(), ref.cpu()):.3e}'


def test_pixel_lockstep_first_call_of_a_fresh_target_engine(eng):
    """The target engine's range and statistics pools are created inside its first U-Net call, which here runs on the engine's
    side stream: their zeroing must be complete before that call's kernels use them."""
    fresh = Engine(0)
    cfg, params, _, _, _ = _family('iddpm')
    tgt = UNet(fresh, cfg, 'iddpm').load_state_dict(specs.synth_state_dict(params, 32))
    gan = dict(gan_type='DDPM_DDIM', source_model_type='afhqcat64', target_model_type='afhqdog64', **DDIM)
    m = UnsupervisedTranslation(dict(gan=gan), source_kwargs=dict(unet=_net(eng, 'iddpm', 31), image_size=64),
                                target_kwargs=dict(unet=tgt, image_size=64)).eval()
    img = torch.rand(2, 3, 64, 64, generator=torch.Generator().manual_seed(1))
    out, ref = _translate(m, img, 7)
    assert torch.equal(out, ref), f'|d| {maxdiff(out.cpu(), ref.cpu()):.3e}'


@pytest.mark.parametrize('es_steps', [1, 9])
def test_pixel_chunk_sizes(eng, eng2, monkeypatch, es_steps):
    m = _pixel_model('iddpm', dict(DDIM, es_steps=es_steps), eng, eng2)
    s, t = m.source_gan_wrapper, m.target_gan_wrapper
    img = torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(2))
    torch.manual_seed(3)
    ref = t(s.encode(img))
    for chunk in (1, 3, 64):
        monkeypatch.setattr(wrappers, 'LOCKSTEP_CHUNK', chunk)
        torch.manual_seed(3)
        out = s.cycle(img, t)
        assert torch.equal(out, ref), f'chunk {chunk}: |d| {maxdiff(out.cpu(), ref.cpu()):.3e}'


@pytest.mark.parametrize('kw', [dict(sample_type='ddim', eta=0.1, custom_steps=10, es_steps=10),
                                dict(sample_type='ddpm', eta=None, custom_steps=20, es_steps=6)])
def test_pixel_lockstep_vs_oracle_two_models(eng, eng2, kw):
    from oracle import dpm_encoder, unet_iddpm
    cfg, params, _, _, _ = _family('iddpm')
    sd_s, sd_t = specs.synth_state_dict(params, 31), specs.synth_state_dict(params, 32)
    m = _pixel_model('iddpm', kw, eng, eng2)
    img = torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(4))
    torch.manual_seed(11)
    (_, out), _, _ = m(torch.zeros(1), original_image=img)
    ora_s = dpm_encoder.PixelCycle(lambda x, t: unet_iddpm.unet_forward(sd_s, cfg, x, t), resolution=64, **kw)
    ora_t = dpm_encoder.PixelCycle(lambda x, t: unet_iddpm.unet_forward(sd_t, cfg, x, t), resolution=64, **kw)
    torch.manual_seed(11)
    with torch.no_grad():
        ref = ora_t.forward(ora_s.encode(img))
    d = maxdiff(out.cpu(), ref)
    print(f'two-model pixel lock-step [{kw["sample_type"]}] vs oracle: |d img| {d:.2e}')
    assert d < 1e-3


def test_pixel_lockstep_memory_flat_in_steps(eng, eng2):
    B, R = 2, 64
    img = torch.rand(B, 3, R, R, generator=torch.Generator().manual_seed(5))
    chunk_bytes = (wrappers.LOCKSTEP_CHUNK + 1) * B * 3 * R * R * 4

    def peak(es, lock):
        m = _pixel_model('iddpm', dict(DDIM, custom_steps=200, es_steps=es), eng, eng2)
        s, t = m.source_gan_wrapper, m.target_gan_wrapper
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        torch.manual_seed(0)
        out = s.cycle(img, t) if lock else t(s.encode(img))
        torch.cuda.synchronize()
        del out
        return torch.cuda.max_memory_allocated() - base + eng.workspace_bytes + eng2.workspace_bytes

    lock = [peak(es, True) for es in (40, 160)]
    two = [peak(es, False) for es in (40, 160)]
    print(f'peak device bytes, es_steps 40 / 160: lock-step {lock}, two-phase {two}')
    assert abs(lock[1] - lock[0]) < chunk_bytes
    assert two[1] - two[0] >= 2 * 120 * B * 3 * R * R * 4


@pytest.mark.parametrize('diff', [dict(es_steps=7), dict(eta=0.2), dict(sample_type='ddpm', eta=None)])
def test_mismatched_schedules_fall_back_to_two_phase(eng, eng2, diff):
    m = _pixel_model('iddpm', DDIM, eng, eng2, target_kw=diff)
    assert not lockstep_compatible(m.source_gan_wrapper, m.target_gan_wrapper)
    img = torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(6))
    if 'es_steps' in diff:          # z of 8 steps cannot be viewed as 7: the two-phase path raises, and so does forward
        for call in (lambda: m(torch.zeros(1), original_image=img), lambda: m.target_gan_wrapper(z=m.source_gan_wrapper.encode(image=img))):
            with pytest.raises(RuntimeError):
                call()
        return
    out, ref = _translate(m, img, 8)
    assert torch.equal(out, ref)


@pytest.mark.parametrize('engines', ['one', 'two'])
def test_ldm_pair_lockstep_equals_two_phase(eng, eng2, engines):
    """FFHQ -> CelebA shape: unconditional LDM pair, white_box_steps - 1 < custom_steps (the target chain finishes alone with
    fresh noise) and an eta = 1 refine pass."""
    from cycle_diffusion_b200.schedule import ldm_alphas_cumprod

    def sd(seed):
        d = {'model.diffusion_model.' + k: v for k, v in specs.synth_state_dict(specs.openai_unet_params(UNCOND_SMALL), seed).items()}
        d.update({'first_stage_model.' + k: v for k, v in specs.synth_state_dict(specs.kl_vae_params(VQ_SMALL), seed + 1).items()})
        return d

    gan = dict(gan_type='LatentDiffStochastic', source_model_type='ffhq256', target_model_type='celebahq256', custom_steps=10, eta=0.1,
               white_box_steps=6, refine_steps=2)
    kw = dict(unet_config=UNCOND_SMALL, vae_config=VQ_SMALL, latent_size=16, resolution=64, alphas_cumprod=ldm_alphas_cumprod())
    m = UnsupervisedTranslation(dict(gan=gan), source_kwargs=dict(engine=eng, state_dict=sd(41), **kw),
                                target_kwargs=dict(engine=eng if engines == 'one' else eng2, state_dict=sd(43), **kw)).eval()
    assert lockstep_compatible(m.source_gan_wrapper, m.target_gan_wrapper)
    img = torch.rand(2, 3, 64, 64, generator=torch.Generator().manual_seed(1))
    out, ref = _translate(m, img, 9)
    assert out.shape == (2, 3, 64, 64) and torch.isfinite(out).all()
    assert torch.equal(out, ref), f'|d| {maxdiff(out.cpu(), ref.cpu()):.3e}'
