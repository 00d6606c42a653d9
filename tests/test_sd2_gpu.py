"""SD 2.x on the GPU: the narrow SD 2 U-Net (64-channel-style fixed head width, Linear projections) and the OpenCLIP tower against
their fixtures, the v-prediction loops (two-phase, lock-step, ensemble fan) against the fixture and each other, the full-size U-Net
at latent 64 and 96 x 96 against the CPU restatement, and the wrapper / pipeline surfaces at 768^2.  Bounds are the SD v1 tests'."""
import pytest
import torch

from cycle_diffusion_b200 import specs
from tests import sd2_oracle
from tests.common import VAE_SMALL, golden, maxdiff
from tests.test_sd2_cpu import NARROW2, OPENCLIP_SMALL

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def eng():
    from cycle_diffusion_b200.engine import Engine
    return Engine(0)


def rel(a, b):
    return maxdiff(a.cpu(), b.cpu()) / float(b.abs().max())


def _unet(eng, prediction='eps'):
    from cycle_diffusion_b200.engine import UNet
    return UNet(eng, NARROW2, 'openai').load_state_dict(specs.synth_state_dict(specs.openai_unet_params(NARROW2), 31)).set_prediction(prediction)


def _noise(n, shape, seed):
    noise = torch.randn((n + 1,) + tuple(shape), generator=torch.Generator().manual_seed(seed))
    noise[n] = 0                                                      # index 0 draws nothing (ddim.py:583-584)
    return noise


@pytest.mark.parametrize('mode', [1, 5])
def test_narrow_unet_vs_reference_fixture(eng, mode):
    g = golden('unet_sd2_narrow')
    unet = _unet(eng)
    try:
        eng.set_mma_mode(mode)
        y = unet(g['x'], g['t'], g['ctx']).cpu()
    finally:
        eng.set_mma_mode(1)
    r = rel(y, g['y'])
    print(f'sd2 narrow unet mode {mode}: rel {r:.2e}')
    assert r < (2e-4 if mode == 1 else 4e-3)          # mode 5: the single-term fp16 bound of test_autocast_gpu.py's kernels


def test_openclip_tower_vs_fixture(eng):
    from cycle_diffusion_b200.wrappers import OpenClipTextCondStage
    g = golden('openclip_text')
    sd = specs.synth_state_dict(specs.openclip_text_params(OPENCLIP_SMALL), int(g['seed']), gain=float(g['gain']))
    sd = {'cond_stage_model.model.' + k: v for k, v in sd.items()}
    cond = OpenClipTextCondStage(eng, sd, lambda texts: g['ids'][:len(texts)], cfg=OPENCLIP_SMALL)
    y = cond(['a', 'b', 'c']).cpu()
    r = rel(y, g['out'])
    print(f'openclip tower: rel {r:.2e}')
    assert r < 5e-5


def test_v_cycle_vs_fixture_and_reconstruction(eng):
    from cycle_diffusion_b200.schedule import DDIMSchedule
    g = golden('ddim_cycle_v')
    S, skip, eta, enc, dec = g['cfg'].tolist()
    unet = _unet(eng, 'v')
    sched = DDIMSchedule(int(S), eta, int(skip))
    n = sched.refine_steps
    torch.manual_seed(int(g['noise_seed']))
    shape = g['x0'].shape
    noise = torch.zeros((n + 1,) + tuple(shape))
    noise[0] = torch.randn(shape)
    for i in range(n):
        if n - 1 - i != 0:
            noise[1 + i] = torch.randn(shape)
    z = unet.latent_encode(g['x0'], g['c_src'], g['uc'], enc, sched, n, noise)
    same = unet.latent_decode(z, g['c_src'], g['uc'], enc, sched).cpu()
    tgt = unet.latent_decode(z, g['c_tgt'], g['uc'], dec, sched).cpu()
    rz = rel(z, g['z'])
    print(f'v cycle: rel|dz| {rz:.2e}  |d same| {maxdiff(same, g["same"]):.2e}  |d tgt| {maxdiff(tgt, g["tgt"]):.2e}  '
          f'|same - x0| {maxdiff(same, g["x0"]):.2e}')
    assert rz < 2e-4
    assert maxdiff(same, g['same']) < 1e-3 and maxdiff(tgt, g['tgt']) < 1e-3
    assert maxdiff(same, g['x0']) < 1e-3
    eps = _unet(eng, 'eps')                                            # the parameterisation is honoured: eps reading differs
    assert maxdiff(eps.latent_decode(z, g['c_tgt'], g['uc'], dec, sched).cpu(), tgt) > 1e-2


def test_v_lockstep_and_fan_vs_two_phase(eng):
    from cycle_diffusion_b200.schedule import DDIMSchedule
    unet = _unet(eng, 'v')
    gen = torch.Generator().manual_seed(3)
    x0 = torch.randn(3, 4, 16, 16, generator=gen) * 0.8
    c_src, c_tgt, uc = (torch.randn(3, 77, 40, generator=gen) for _ in range(3))
    sched = DDIMSchedule(6, 0.1, 2)
    n = sched.refine_steps
    noise = _noise(n, x0.shape, 1)
    out, z = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 2.0, 3.0, sched, noise, return_z=True)
    z2 = unet.latent_encode(x0, c_src, uc, 2.0, sched, n, noise)
    out2 = unet.latent_decode(z2, c_tgt, uc, 3.0, sched)
    rz, dx = rel(z, z2), maxdiff(out.cpu(), out2.cpu())
    print(f'v lockstep vs two-phase: rel|dz| {rz:.2e} |dx| {dx:.2e}')
    assert rz < 2e-5 and dx < 1e-4
    src, decs = [1.0, 3.0, 0.0], [1.0, 0.0, 3.0]
    fo, fz = unet.cycle_fan(x0, c_src, c_tgt, uc, src, [decs] * 3, sched, noise, return_z=True)
    fz2 = unet.latent_encode_ens(x0, c_src, uc, src, sched, n, noise)
    rep = lambda t: t.to(eng.device).repeat_interleave(3, dim=0)
    fo2 = unet.latent_decode_ens(rep(fz2), rep(c_tgt), rep(uc), decs * 3, sched)
    print(f'v fan vs two-phase: rel|dz| {rel(fz, fz2):.2e} |dx| {maxdiff(fo.cpu(), fo2.cpu()):.2e}')
    assert rel(fz, fz2) < 2e-5 and maxdiff(fo.cpu(), fo2.cpu()) < 1e-4


def _wrapper(eng, **over):
    from cycle_diffusion_b200.wrappers import SD2StochasticTextWrapper, SyntheticTextEncoder
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW2), 31)
    vsd = specs.synth_state_dict(specs.kl_vae_params(VAE_SMALL), 21)
    sd = {'model.diffusion_model.' + k: v for k, v in usd.items()}
    sd.update({'first_stage_model.' + k: v for k, v in vsd.items()})
    kw = dict(custom_steps=6, eta=0.1, white_box_steps=7, skip_steps=[2, 3], encoder_unconditional_guidance_scales=[1.0, 3.0],
              decoder_unconditional_guidance_scales=[1.0, 0.0, 3.0], n_trials=2)
    kw.update(over)
    return SD2StochasticTextWrapper('synthetic', parameterization='v', engine=eng, state_dict=sd, cond_stage=SyntheticTextEncoder(40),
                                    unet_config=NARROW2, vae_config=VAE_SMALL, resolution=128, **kw)


def test_v_ensemble_lockstep_vs_encode_forward(eng):
    from tests.test_ensemble_lockstep_gpu import SRC, TGT, _dclip
    dclip = _dclip(eng)
    w = _wrapper(eng, ranker=dclip).eval()
    assert w.resolution == 128 and w.generator.image_size == 16 and w.generator.unet.prediction == 'v'
    assert w.lockstep_ensemble() and not w.single_member()
    image = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(5))
    torch.manual_seed(77)
    img, idx, scores = w.cycle_ensemble(image, SRC, TGT)
    torch.manual_seed(77)
    cands = [eng.shift_scale(i, 1.0, 0.5) for i in w.generate(w.encode(image, SRC), TGT)]
    _, idx2, scores2 = dclip.rank(cands, image, SRC, TGT)
    ds = maxdiff(scores.cpu(), scores2.cpu())
    top2 = scores2.cpu().topk(2, dim=1).values
    gap = top2[:, 0] - top2[:, 1]
    print(f'v ensemble: |d score| {ds:.2e}  index {idx.tolist()} vs {idx2.tolist()} (gap {gap.tolist()})')
    assert scores.shape == (2, 2 * 2 * 2 * 3) and ds < 1e-4
    for b in range(2):
        if gap[b] > 1e-3:
            assert int(idx[b]) == int(idx2[b])
            assert maxdiff(img[b].cpu(), cands[int(idx[b])][b].cpu()) < 1e-3


@pytest.mark.parametrize('hw', [64, 96])
def test_fullsize_sd2_unet_vs_oracle(eng, hw):
    from cycle_diffusion_b200.engine import UNet
    cfg = specs.sd2_unet_config()
    sd = specs.synth_state_dict(specs.openai_unet_params(cfg), 7)
    unet = UNet(eng, cfg, 'openai').load_state_dict(sd)
    g = torch.Generator().manual_seed(hw)
    x, ctx = torch.randn(1, 4, hw, hw, generator=g), torch.randn(1, 77, 1024, generator=g)
    t = torch.tensor([601])
    y = unet(x, t, ctx).cpu()
    with torch.no_grad():
        ref = sd2_oracle.unet_forward(sd, cfg, x, t, ctx)
    r = rel(y, ref)
    print(f'sd2 full-size unet {hw}x{hw}: rel {r:.2e}')
    assert r < 2e-4


def test_sd2_v_wrapper_768_translation_and_pipeline(eng):
    """SD2StochasticTextWrapper(parameterization='v', state_dict='synthetic'): full-size U-Net and VAE, a 2 + 2-step translation at
    768^2 through TextUnsupervisedTranslation.forward, and CycleDiffusionPipeline.from_wrapper on the same generator."""
    from cycle_diffusion_b200.models import TextUnsupervisedTranslation
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    m = TextUnsupervisedTranslation(dict(gan=dict(gan_type='SD2StochasticText', source_model_type='v2-1_768-ema-pruned.ckpt', custom_steps=2,
                                                  eta=0.1, white_box_steps=3, skip_steps=[0], encoder_unconditional_guidance_scales=[1.0],
                                                  decoder_unconditional_guidance_scales=[3.0], n_trials=1, parameterization='v')),
                                    engine=eng, state_dict='synthetic').eval()
    w = m.gan_wrapper
    assert (w.resolution, w.generator.image_size, w.generator.parameterization) == (768, 96, 'v')
    image = torch.rand(1, 3, 768, 768, generator=torch.Generator().manual_seed(1))
    torch.manual_seed(3)
    (_, img), _, _ = m(torch.tensor([0]), image, ['a cat'], ['a dog'])
    assert img.shape == (1, 3, 768, 768) and torch.isfinite(img).all()
    pipe = CycleDiffusionPipeline.from_wrapper(w)
    out = pipe('a dog', 'a cat', image, strength=1.0, num_inference_steps=2, guidance_scale=3.0, source_guidance_scale=1.0, eta=0.1,
               generator=torch.Generator().manual_seed(9)).images
    out2 = pipe('a dog', 'a cat', image, strength=1.0, num_inference_steps=2, guidance_scale=3.0, source_guidance_scale=1.0, eta=0.1,
                generator=torch.Generator().manual_seed(9), two_phase=True).images
    print(f'sd2-v 768: wrapper img range [{float(img.min()):.3f}, {float(img.max()):.3f}]  pipeline lock-step vs two-phase {maxdiff(out.cpu(), out2.cpu()):.2e}')
    assert out.shape == (1, 3, 768, 768) and maxdiff(out.cpu(), out2.cpu()) < 1e-4


def test_set_prediction_rejected_on_pixel_net(eng):
    import ctypes as C
    from cycle_diffusion_b200 import _cabi
    from cycle_diffusion_b200.engine import UNet
    from cycle_diffusion_b200.schedule import v_tables
    pix = UNet(eng, specs.iddpm_config(64), 'iddpm')
    sa, s1 = v_tables()
    arr = lambda a: (C.c_float * len(a))(*a.tolist())
    assert _cabi.lib.cdx_unet_set_prediction(pix.h, _cabi.CDX_PRED_V, arr(sa), arr(s1), len(sa)) == -1      # CDX_E_INVALID
    assert _cabi.lib.cdx_unet_set_prediction(_unet(eng).h, 7, None, None, 0) == -1
