"""Mask-guided local editing on the lock-step loop (cdx_cycle_lockstep_masked, cdx_latent_cycle_fan_masked, cdx_mask_pool,
cdx_mask_composite) against the unmasked loop, the exact mask-0 / mask-1 properties, the CPU masked oracle, and through the
pipeline and the text wrappers."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.wrappers import encode_noise
from tests.common import NARROW, VAE_SMALL, maxdiff
from tests.masked_oracle import masked_cycle, masked_search

pytestmark = pytest.mark.gpu

B = 2


@pytest.fixture(scope='module')
def eng():
    from cycle_diffusion_b200.engine import Engine
    return Engine(0)


@pytest.fixture(scope='module')
def usd():
    return specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)


@pytest.fixture(scope='module')
def unet(eng, usd):
    from cycle_diffusion_b200.engine import UNet
    return UNet(eng, NARROW, 'openai').load_state_dict(usd)


@pytest.fixture(scope='module')
def sched():
    from cycle_diffusion_b200.schedule import DDIMSchedule
    return DDIMSchedule(6, 0.1, 2)


def _inputs(sched, h=16, w=16, seed=7):
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(B, 4, h, w, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(B, 77, 48, generator=g) for _ in range(3))
    torch.manual_seed(seed + 1)
    return x0, c_src, c_tgt, uc, encode_noise(sched, sched.refine_steps, x0.shape)


def _soft_mask(n, h, w, seed=3):
    """Values in (0, 1) with exact 0 and 1 regions, so all three branches of the blend run."""
    m = torch.rand(n, 1, h, w, generator=torch.Generator().manual_seed(seed))
    m[..., : h // 4, :] = 0.0
    m[..., -(h // 4):, :] = 1.0
    return m


def _box(n, h, w):
    m = torch.zeros(n, 1, h, w)
    m[..., h // 4: 3 * h // 4, w // 4: 3 * w // 4] = 1.0
    return m


@pytest.fixture
def with_prediction(unet):
    def use(pred):
        unet.set_prediction(pred)
    yield use
    unet.set_prediction('eps')


@pytest.mark.parametrize('pred', ['eps', 'v'])
@pytest.mark.parametrize('src_scale,tgt_scale', [(1.0, 3.0), (3.0, 0.0), (2.0, 5.0)])
def test_mask_of_ones_is_the_unmasked_cycle(unet, sched, with_prediction, pred, src_scale, tgt_scale):
    """A mask of ones takes the target value unchanged at every step: latent and z equal cycle_lockstep's bit for bit.  The source
    chain never reads the mask; under another mask its z changes only through the shared U-Net call, whose fp16-split operands take
    one exponent per tensor over all rows (bound of the lock-step vs two-phase comparison, which also changes the batch)."""
    with_prediction(pred)
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise, return_z=True)
    out_1, z_1 = unet.cycle_lockstep(x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise, return_z=True, mask=torch.ones(B, 1, 16, 16))
    out_s, z_s = unet.cycle_lockstep(x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise, return_z=True, mask=_soft_mask(B, 16, 16))
    assert torch.isfinite(out).all()
    assert torch.equal(out_1, out) and torch.equal(z_1, z)
    rz = maxdiff(z_s.cpu(), z.cpu()) / float(z.abs().max())
    print(f'z under a soft mask vs unmasked ({pred}, {src_scale}/{tgt_scale}): rel|dz| {rz:.2e}')
    assert rz < 2e-5 and not torch.equal(out_s, out)


@pytest.mark.parametrize('mode', [1, 5])
def test_mask_of_zeros_returns_x0(eng, unet, sched, mode):
    """Outside the mask the target takes the source chain's x_{t-1}, which on the last step is x0 itself."""
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    try:
        eng.set_mma_mode(mode)
        out = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=torch.zeros(B, 1, 16, 16))
    finally:
        eng.set_mma_mode(1)
    assert torch.equal(out.cpu(), x0)


def test_box_mask_keeps_the_outside_bit_for_bit(unet, sched):
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    m = _box(B, 16, 16)
    out = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, mask=m).cpu()
    inside = m.expand_as(x0) == 1
    assert torch.equal(out[~inside], x0[~inside])
    assert bool((out[inside] != x0[inside]).all())


@pytest.mark.parametrize('h,w', [(16, 16), (16, 24)])
def test_soft_mask_vs_masked_oracle(unet, usd, sched, h, w):
    """Engine against the CPU masked oracle under a soft mask (bounds of test_lockstep_driver_vs_reference_fixture_and_two_phase)."""
    from oracle import unet_openai
    x0, c_src, c_tgt, uc, noise = _inputs(sched, h, w, seed=11)
    m = _soft_mask(B, h, w, seed=5)
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, noise, return_z=True, mask=m)
    torch.manual_seed(12)                                                     # the seed _inputs drew the noise under
    with torch.no_grad():
        (y_ref,), z_ref = masked_cycle(lambda x, t, c: unet_openai.unet_forward(usd, NARROW, x, t, c), x0, c_src, c_tgt, uc,
                                       6, 0.1, 2, 1.0, [3.0], m)                  # the `sched` fixture's S, eta, skip
    z_ref = torch.stack(z_ref, dim=1)
    rz = maxdiff(z.cpu(), z_ref) / float(z_ref.abs().max())
    dx = maxdiff(out.cpu(), y_ref)
    print(f'masked lock-step {h}x{w} vs oracle: rel|dz| {rz:.2e}  |dx| {dx:.2e}')
    assert rz < 2e-4 and dx < 1e-3


def test_fan_with_mask(unet, sched):
    """K = 1: the masked fan is the masked lock-step cycle bit for bit.  K = 3: each target equals its own masked lock-step call
    (bounds of test_fan_is_encode_then_decode_per_target_scale: the U-Net batch differs)."""
    x0, c_src, c_tgt, uc, noise = _inputs(sched)
    m = _soft_mask(B, 16, 16, seed=9)
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 3.0, 5.0, sched, noise, return_z=True, mask=m)
    out_f, z_f = unet.cycle_fan(x0, c_src, c_tgt, uc, [3.0] * B, [[5.0]] * B, sched, noise, return_z=True, mask=m)
    assert torch.equal(out_f, out) and torch.equal(z_f, z)
    dec = [1.0, 0.0, 3.0]
    fan = unet.cycle_fan(x0, c_src, c_tgt, uc, [3.0] * B, [dec] * B, sched, noise, mask=m).view(B, len(dec), *x0.shape[1:])
    dx = [maxdiff(fan[:, k].cpu(), unet.cycle_lockstep(x0, c_src, c_tgt, uc, 3.0, s, sched, noise, mask=m).cpu()) for k, s in enumerate(dec)]
    print(f'masked fan K=3 vs lock-step: |dx| per target scale {[f"{d:.2e}" for d in dx]}')
    assert max(dx) < 1e-4
    with pytest.raises(ValueError):
        unet.cycle_fan(x0, c_src, c_tgt, uc, [3.0] * B, [dec] * B, sched, noise, mask=m[:1])


def test_mask_pool_matches_avg_pool2d(eng):
    for f, (H, W) in ((8, (128, 96)), (4, (64, 80))):
        m = torch.rand(3, 1, H, W, generator=torch.Generator().manual_seed(f))
        got = eng.mask_pool(m, f).cpu()
        ref = F.avg_pool2d(m, f)
        ulp = torch.from_numpy(np.spacing(ref.abs().numpy()))
        assert got.shape == ref.shape and bool(((got - ref).abs() <= ulp).all())
    ones = eng.mask_pool(torch.ones(1, 1, 64, 64), 8)
    assert torch.equal(ones.cpu(), torch.ones(1, 1, 8, 8))


def _sd_wrapper(eng, **over):
    from cycle_diffusion_b200.wrappers import SDStochasticTextWrapper, SyntheticTextEncoder
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    vsd = specs.synth_state_dict(specs.kl_vae_params(VAE_SMALL), 21)
    sd = {'model.diffusion_model.' + k: v for k, v in usd.items()}
    sd.update({'first_stage_model.' + k: v for k, v in vsd.items()})
    kw = dict(custom_steps=4, eta=0.1, white_box_steps=5, skip_steps=[0], encoder_unconditional_guidance_scales=[1],
              decoder_unconditional_guidance_scales=[3.0], n_trials=1)
    kw.update(over)
    return SDStochasticTextWrapper('synthetic', engine=eng, state_dict=sd, cond_stage=SyntheticTextEncoder(48), unet_config=NARROW,
                                   vae_config=VAE_SMALL, latent_size=16, resolution=128, **kw)


@pytest.mark.parametrize('precision,H,W,pred', [('full', 128, 128, 'eps'), ('autocast', 128, 192, 'eps'), ('full', 128, 192, 'v')])
def test_pipeline_mask_image_and_paste_back(eng, precision, H, W, pred):
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    w = _sd_wrapper(eng)
    w.generator.parameterization = pred
    pipe = CycleDiffusionPipeline(w.generator, precision=precision)
    g = w.generator
    image = torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(4))
    box = torch.zeros(1, 1, H, W)
    box[..., 32:96, 64:112] = 1.0                                              # on the 8-pixel latent grid
    kw = dict(strength=0.75, num_inference_steps=8, guidance_scale=3.0, eta=0.1, num_images_per_prompt=2)
    lat = {}

    def run(tag, **extra):
        cb = lambda i, t, x: lat.__setitem__(tag, x.cpu())
        return pipe('a dog', 'a cat', image, generator=torch.Generator().manual_seed(9), callback=cb, **kw, **extra).images.cpu()

    plain = run('plain')
    assert torch.equal(run('none', mask_image=None), plain)
    assert torch.equal(run('ones', mask_image=torch.ones(1, 1, H, W)), plain)
    boxed = run('box', mask_image=box)
    pasted = run('paste', mask_image=box.expand(1, 1, H, W).clone(), paste_back=True)
    # the latent outside the box is x0 bit for bit: the posterior draw is the generator's first
    gen = torch.Generator().manual_seed(9)
    with eng.precision(precision):
        mom = g.encode_first_stage(eng.shift_scale(image.repeat(2, 1, 1, 1), -0.5, 2.0))
        x0 = eng.vae_posterior(mom, torch.randn(2, 4, H // 8, W // 8, generator=gen), 0.18215).cpu()
    inside = F.avg_pool2d(box, 8).expand_as(x0) == 1
    assert torch.equal(lat['box'][~inside], x0[~inside]) and bool((lat['box'][inside] != x0[inside]).all())
    outside_px = (box == 0).expand(2, 3, H, W)
    assert torch.equal(pasted[outside_px], image.repeat(2, 1, 1, 1)[outside_px])
    inside_px = (box == 1).expand(2, 3, H, W)
    assert torch.equal(pasted[inside_px], boxed[inside_px])
    assert pasted.shape == (2, 3, H, W)


def test_pipeline_rejects_bad_masks(eng):
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    pipe = CycleDiffusionPipeline(_sd_wrapper(eng).generator)
    image = torch.rand(2, 3, 128, 128)
    call = lambda **k: pipe('a dog', 'a cat', image, num_inference_steps=4, **k)
    good = torch.ones(2, 1, 128, 128)
    bad = [torch.ones(2, 1, 64, 64), torch.ones(3, 1, 128, 128), torch.ones(2, 3, 128, 128), good * 1.5, good * -0.1,
           good.clone().index_fill_(2, torch.tensor([3]), float('nan')), good.double()]
    for m in bad:
        with pytest.raises(ValueError):
            call(mask_image=m)
    with pytest.raises(ValueError):
        call(mask_image=good, two_phase=True)
    with pytest.raises(ValueError):
        call(paste_back=True)


def test_wrapper_cycle_with_mask(eng):
    w = _sd_wrapper(eng)
    image = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(2))
    torch.manual_seed(5)
    plain = w.cycle(image, ['a', 'b'], ['c', 'd'])
    torch.manual_seed(5)
    ones = w.cycle(image, ['a', 'b'], ['c', 'd'], mask=torch.ones(2, 1, 128, 128))
    assert torch.equal(ones, plain)
    with pytest.raises(ValueError):
        w.cycle(image, ['a', 'b'], ['c', 'd'], mask=torch.ones(2, 1, 16, 16))


def test_cycle_ensemble_with_mask_vs_oracle_search(eng):
    """The masked lock-step ensemble search picks the candidate the oracle's masked member-by-member search picks (n_trials = 1,
    L1 ranker), and its image is that oracle candidate's."""
    from oracle import dpm_encoder, unet_openai, vae_kl
    from cycle_diffusion_b200.wrappers import SyntheticTextEncoder
    kw = dict(custom_steps=6, eta=0.1, white_box_steps=7, skip_steps=[2, 3], encoder_unconditional_guidance_scales=[1.0, 3.0],
              decoder_unconditional_guidance_scales=[1.0, 0.0, 3.0], n_trials=1)
    ranker = lambda img, orig, et, dt: (None, -(img - orig.to(img.device)).flatten(1).abs().mean(1))
    w = _sd_wrapper(eng, ranker=ranker, **kw)
    assert w.lockstep_ensemble()
    image = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(5))
    mask = torch.zeros(2, 1, 128, 128)
    mask[0, :, 16:80, 32:112] = 1.0
    mask[1, :, 48:128, 0:64] = 1.0
    src, tgt = ['a', 'b'], ['c', 'd']
    torch.manual_seed(77)
    img, idx, scores = w.cycle_ensemble(image, src, tgt, mask=mask)
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    vsd = specs.synth_state_dict(specs.kl_vae_params(VAE_SMALL), 21)
    ora = dpm_encoder.LatentCycle(lambda x, t, c: unet_openai.unet_forward(usd, NARROW, x, t, c),
                                  lambda im: vae_kl.encode_moments(vsd, VAE_SMALL, im), lambda zz: vae_kl.decode(vsd, VAE_SMALL, zz),
                                  SyntheticTextEncoder(48), channels=4, latent_size=16, resolution=128, **kw)
    torch.manual_seed(77)
    with torch.no_grad():
        cands = masked_search(ora, image, src, tgt, mask, 8)
    ref_scores = torch.stack([ranker(c, image, None, None)[1] for c in cands], dim=1)
    ref_idx = ref_scores.argmax(1)
    top2 = ref_scores.topk(2, dim=1).values
    gap = top2[:, 0] - top2[:, 1]
    di = max(maxdiff(img[b].cpu(), cands[int(idx[b])][b]) for b in range(2))
    print(f'masked ensemble: index {idx.tolist()} vs oracle {ref_idx.tolist()} (gap {gap.tolist()})  |d score| '
          f'{maxdiff(scores.cpu(), ref_scores):.2e}  |d img| {di:.2e}')
    assert scores.shape == (2, len(cands)) == (2, 12)
    for b in range(2):
        if gap[b] > 1e-3:
            assert int(idx[b]) == int(ref_idx[b])
    assert di < 1e-3
