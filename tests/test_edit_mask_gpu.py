"""Edit masks from the prompts (DiffEdit: cdx_edit_map, cdx_edit_map_from_eps, cdx_edit_mask) against float64 and the CPU oracle
of tests/edit_mask_oracle.py, independent of how the maps are split over U-Net calls and launches, and through the pipeline
(generate_mask, mask_image='auto')."""
import pytest
import torch

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.schedule import DDIMSchedule, v_tables
from tests.common import NARROW, maxdiff
from tests.edit_mask_oracle import accumulate, edit_map, edit_mask, normalized
from tests.test_masked_edit_gpu import _sd_wrapper

pytestmark = pytest.mark.gpu


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


@pytest.fixture
def with_prediction(unet):
    def use(pred):
        unet.set_prediction(pred)
    yield use
    unet.set_prediction('eps')


def _preds(B=3, n=5, C=4, h=16, w=24, seed=0):
    g = torch.Generator().manual_seed(seed)
    e_src = torch.randn(B, n, C, h, w, generator=g)
    e_tgt = e_src + 0.3 * torch.randn(B, n, C, h, w, generator=g)
    e_tgt[..., : h // 2, : w // 3] += 2.0
    return e_src, e_tgt


@pytest.mark.parametrize('vscale', [1.0, 0.6710])
def test_edit_map_from_eps_vs_float64(eng, vscale):
    e_src, e_tgt = _preds()
    acc = eng.edit_map_from_eps(e_src, e_tgt, vscale).cpu()
    ref = (vscale * (e_tgt.double() - e_src.double())).abs().sum(dim=(1, 2))
    rel = maxdiff(acc, ref) / float(ref.abs().max())
    print(f'edit_map_from_eps vscale {vscale}: rel vs float64 {rel:.2e}')
    assert rel < 1e-6
    assert torch.equal(acc, accumulate(e_src, e_tgt, vscale))             # the oracle's fp32 op order
    for mpl in (1, 2, 3):
        assert torch.equal(eng.edit_map_from_eps(e_src, e_tgt, vscale, maps_per_launch=mpl).cpu(), acc)


def test_edit_mask_vs_oracle(eng):
    e_src, e_tgt = _preds(B=3, n=5, h=16, w=24, seed=1)
    e_tgt[2] = e_src[2]                                                     # image 2: the prompts agree everywhere
    acc = accumulate(e_src, e_tgt)
    for f in (8, 4, None):
        emap, mask, img = eng.edit_mask(acc, 5, 3.0, f=f)
        emap_r, mask_r, img_r = edit_mask(acc, 5, 4, 3.0, f=f)
        _, norm, _ = normalized(acc, 5, 4, 3.0)
        away = (norm - 0.5).abs() > 1e-4
        assert torch.equal(emap.cpu(), emap_r)
        assert torch.equal(mask.cpu()[away], mask_r[away])
        assert 0 < float(mask[:2].sum()) < mask[:2].numel()
        assert torch.equal(mask[2].cpu(), torch.zeros_like(mask_r[2]))
        if f is None:
            assert img is None
            continue
        assert img.shape == (3, 1, 16 * f, 24 * f)
        assert torch.equal(img.cpu(), mask.cpu().repeat_interleave(f, 2).repeat_interleave(f, 3))
        assert torch.equal(eng.mask_pool(img, f), mask)
    with pytest.raises(ValueError):
        eng.edit_mask(acc, 5, 0.0)


def _map_inputs(B=2, n=3, h=16, w=16, seed=5):
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(B, 4, h, w, generator=g) * 0.8
    c_src, c_tgt = torch.randn(B, 77, 48, generator=g), torch.randn(B, 77, 48, generator=g)
    return x0, c_src, c_tgt, torch.randn(B, n, 4, h, w, generator=g)


@pytest.mark.parametrize('pred', ['eps', 'v'])
def test_unet_edit_map_vs_oracle(unet, usd, with_prediction, pred):
    from oracle import unet_openai
    with_prediction(pred)
    sched = DDIMSchedule(6, 0.0, 3)
    t = sched.t_loop[0]
    vscale = float(v_tables()[0][int(t)]) if pred == 'v' else 1.0
    x0, c_src, c_tgt, noise = _map_inputs()
    c_tgt[0] = c_src[0]                                                     # image 0: nothing to edit
    acc = unet.edit_map(x0, c_src, c_tgt, sched, noise).cpu()
    with torch.no_grad():
        ref = edit_map(lambda x, ts, c: unet_openai.unet_forward(usd, NARROW, x, ts, c), x0, c_src, c_tgt, t, sched.sqrt_a_T,
                       sched.sqrt_1ma_T, noise, vscale)
    rel = maxdiff(acc, ref) / float(ref.abs().max())
    print(f'edit_map ({pred}) vs oracle: rel {rel:.2e}, image 0 max {float(acc[0].abs().max()):.1e}')
    assert rel < 1e-4
    _, norm, _ = normalized(ref, 3, 4)
    away = (norm - 0.5).abs() > 1e-4
    eng = unet.engine
    _, mask, _ = eng.edit_mask(acc, 3, 3.0)
    _, mask_r, _ = edit_mask(ref, 3, 4)
    assert torch.equal(mask.cpu()[away], mask_r[away])
    assert float(acc[0].abs().max()) == 0 and float(mask[0].sum()) == 0
    _, loose, _ = eng.edit_mask(acc, 3, 1.0)                                # threshold at half the mean: never empty unless flat
    assert float(loose[0].sum()) == 0 and float(loose[1].sum()) > 0
    print(f'mask coverage of image 1 at ratio 3: {float(mask[1].mean()):.3f}')
    for rows in (2, 6, 7):
        acc_r = unet.edit_map(x0, c_src, c_tgt, sched, noise, rows_per_call=rows).cpu()
        assert maxdiff(acc_r, ref) / float(ref.abs().max()) < 1e-4
        assert torch.equal(eng.edit_mask(acc_r, 3, 3.0)[1].cpu(), mask.cpu())
    with pytest.raises(AssertionError):
        unet.edit_map(x0, c_src, c_tgt, sched, noise, rows_per_call=1)


def test_unet_edit_map_rejects_a_call_beyond_the_statistics_pool(eng, unet):
    """NARROW's GroupNorm statistics come to over 10^4 doubles per row: a 1024-row call would need more than the pool's 8M.  The
    sizing pass rejects it before anything runs, and the engine stays usable."""
    x0, c_src, c_tgt, noise = _map_inputs(B=2, n=512, h=8, w=8)
    with pytest.raises(AssertionError, match='statistics'):
        unet.edit_map(x0, c_src, c_tgt, DDIMSchedule(6, 0.0, 3), noise, rows_per_call=1024)
    assert unet.edit_map(x0[:1], c_src[:1], c_tgt[:1], DDIMSchedule(6, 0.0, 3), noise[:1, :2]).shape == (1, 8, 8)


def _pipe(eng, precision='full'):
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    return CycleDiffusionPipeline(_sd_wrapper(eng).generator, precision=precision)


@pytest.mark.parametrize('H,W', [(128, 128), (128, 192)])
def test_generate_mask_shapes(eng, H, W):
    pipe = _pipe(eng)
    image = torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(3))
    m = pipe.generate_mask(image, 'a cat', ['a dog', 'a fox'], num_maps_per_mask=4, generator=torch.Generator().manual_seed(1))
    assert m.shape == (2, 1, H, W) and m.dtype == torch.float32 and m.is_cuda
    assert bool(((m == 0) | (m == 1)).all())
    lat = pipe.generate_mask(image, 'a cat', ['a dog', 'a fox'], num_maps_per_mask=4, generator=torch.Generator().manual_seed(1),
                             output_type='latent')
    assert lat.shape == (2, 1, H // 8, W // 8) and torch.equal(pipe.engine.mask_pool(m, 8), lat)
    print(f'generate_mask {H}x{W}: coverage {float(m.mean()):.3f}')


def test_generate_mask_rejects_bad_arguments(eng):
    pipe = _pipe(eng)
    image = torch.rand(1, 3, 128, 128)
    call = lambda img=image, **k: pipe.generate_mask(img, 'a cat', 'a dog', **k)
    for kw in (dict(mask_encode_strength=0.0), dict(mask_encode_strength=1.5), dict(mask_encode_strength=0.5, num_inference_steps=1),
               dict(num_maps_per_mask=0), dict(num_maps_per_mask=2.5), dict(mask_thresholding_ratio=0.0),
               dict(mask_thresholding_ratio=-1.0), dict(output_type='np')):
        with pytest.raises(ValueError):
            call(**kw)
    with pytest.raises(ValueError):
        call(torch.rand(1, 3, 120, 128))
    with pytest.raises(ValueError):
        pipe('a dog', 'a cat', image, num_inference_steps=4, mask_image='box')


@pytest.mark.parametrize('paste_back', [False, True])
def test_auto_mask_is_the_two_call_composition(eng, paste_back):
    pipe = _pipe(eng)
    image = torch.rand(2, 3, 128, 192, generator=torch.Generator().manual_seed(6))
    kw = dict(strength=0.75, num_inference_steps=8, guidance_scale=3.0, eta=0.1, num_images_per_prompt=2, paste_back=paste_back)
    tgt, src = ['a dog', 'a fox'], ['a cat', 'a cat']
    auto = pipe(tgt, src, image, generator=torch.Generator().manual_seed(9), mask_image='auto', **kw).images.cpu()
    gen = torch.Generator().manual_seed(9)
    m = pipe.generate_mask(image, src, tgt, generator=gen, num_inference_steps=8)
    two = pipe(tgt, src, image, generator=gen, mask_image=m, **kw).images.cpu()
    assert torch.equal(auto, two)
    print(f'auto mask coverage {float(m.mean()):.3f}')
    if paste_back:
        outside = (m.cpu() == 0).repeat_interleave(2, 0).expand(4, 3, 128, 192)
        assert torch.equal(auto[outside], image.repeat_interleave(2, 0)[outside])


def test_generate_mask_autocast(eng):
    pipe = _pipe(eng, precision='autocast')
    image = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(8))
    m = pipe.generate_mask(image, 'a cat', 'a dog', num_maps_per_mask=3, generator=torch.Generator().manual_seed(2))
    assert m.shape == (2, 1, 128, 128) and bool(((m == 0) | (m == 1)).all())
    assert eng.mma_mode == 1
