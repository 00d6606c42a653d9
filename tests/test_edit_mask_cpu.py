"""The DiffEdit edit-mask oracle without a GPU: per-image normalisation (no image's mask depends on its batch-mates), the empty mask
of an all-zero map, invariance to a scale on the difference (the v scaling and the dropped guidance scale), the > 0.5 threshold,
the nearest upsample that avg_pool2d undoes exactly, the default mask timestep, and the exported symbols."""
import inspect

import torch
import torch.nn.functional as F

from cycle_diffusion_b200 import _cabi, specs
from cycle_diffusion_b200.schedule import DDIMSchedule
from oracle import unet_openai
from tests.common import NARROW
from tests.edit_mask_oracle import accumulate, edit_map, edit_mask, normalized


def _preds(B=3, n=4, C=4, h=8, w=12, seed=0):
    """Random predictions whose target differs strongly in one corner, so that the masks are neither empty nor full."""
    g = torch.Generator().manual_seed(seed)
    e_src = torch.randn(B, n, C, h, w, generator=g)
    e_tgt = e_src + 0.3 * torch.randn(B, n, C, h, w, generator=g)
    e_tgt[..., : h // 2, : w // 3] += 2.0
    return e_src, e_tgt


def test_default_mask_timestep_is_481():
    sched = DDIMSchedule(50, 0.0, 50 - int(50 * 0.5))
    assert sched.t_loop[0] == 481.0
    assert sched.t_loop == DDIMSchedule(50, 0.1, 25).t_loop and sched.sqrt_a_T == DDIMSchedule(50, 0.1, 25).sqrt_a_T


def test_one_image_alone_gets_its_batch_mask():
    sd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    unet = lambda x, t, c: unet_openai.unet_forward(sd, NARROW, x, t, c)
    g = torch.Generator().manual_seed(3)
    x0 = torch.randn(2, 4, 16, 16, generator=g) * 0.8
    c_src, c_tgt = torch.randn(2, 77, 48, generator=g), torch.randn(2, 77, 48, generator=g)
    noise = torch.randn(2, 2, 4, 16, 16, generator=g)
    sched = DDIMSchedule(6, 0.0, 3)
    args = (sched.t_loop[0], sched.sqrt_a_T, sched.sqrt_1ma_T)
    with torch.no_grad():
        acc = edit_map(unet, x0, c_src, c_tgt, *args, noise)
        acc1 = edit_map(unet, x0[1:], c_src[1:], c_tgt[1:], *args, noise[1:])
    assert torch.equal(acc[1:], acc1)
    _, mask, _ = edit_mask(acc, 2, 4)
    _, mask1, _ = edit_mask(acc1, 2, 4)
    assert torch.equal(mask[1:], mask1)
    # a batch-mate with a map 100x larger changes nothing either
    acc_big = acc.clone()
    acc_big[0] *= 100
    assert torch.equal(edit_mask(acc_big, 2, 4)[1][1:], mask1)


def test_zero_map_gives_an_empty_mask():
    e_src, e_tgt = _preds()
    e_tgt[1] = e_src[1]
    emap, mask, img = edit_mask(accumulate(e_src, e_tgt), 4, 4, f=8)
    assert torch.equal(emap[1], torch.zeros_like(emap[1])) and torch.equal(mask[1], torch.zeros_like(mask[1]))
    assert not torch.isnan(mask).any() and img[1].sum() == 0 and mask[0].sum() > 0


def test_a_scale_on_the_difference_leaves_the_mask():
    e_src, e_tgt = _preds(seed=1)
    _, mask, _ = edit_mask(accumulate(e_src, e_tgt), 4, 4)
    for s in (7.5, 0.25, 0.9991):                 # a guidance scale, a power of two, a v scale sa_v[t]
        _, norm_s, _ = normalized(accumulate(e_src, e_tgt, s), 4, 4)
        _, norm, _ = normalized(accumulate(e_src, e_tgt), 4, 4)
        away = (norm - 0.5).abs() > 1e-4
        assert torch.equal((norm_s > 0.5)[away], mask.bool()[away])
    _, mask_p2, _ = edit_mask(accumulate(e_src, e_tgt, 0.25), 4, 4)
    assert torch.equal(mask_p2, mask)                # a power of two scales every value exactly


def test_threshold_is_strictly_above_one_half():
    # 3 pixels: mean m = (a + b + c) / 3, M = 3m = a + b + c; pixel / M vs 0.5
    acc = torch.tensor([[[2.0, 1.0, 1.0]]]) * 4      # n*C = 4: map = [2, 1, 1], M = 4 -> [0.5, 0.25, 0.25]
    emap, mask, _ = edit_mask(acc, 1, 4)
    assert torch.equal(emap.flatten(), torch.tensor([2.0, 1.0, 1.0]))
    assert torch.equal(mask.flatten(), torch.tensor([0.0, 0.0, 0.0]))                       # exactly 0.5 is not > 0.5
    _, mask, _ = edit_mask(torch.tensor([[[2.5, 1.0, 0.5]]]) * 4, 1, 4)                       # M = 4: [0.625, 0.25, 0.125]
    assert torch.equal(mask.flatten(), torch.tensor([1.0, 0.0, 0.0]))
    _, mask, _ = edit_mask(torch.tensor([[[9.0, 0.0, 0.0]]]), 1, 1, ratio=0.5)               # M = 1.5: clamped to 1 -> 1 > 0.5
    assert torch.equal(mask.flatten(), torch.tensor([1.0, 0.0, 0.0]))


def test_upsampled_mask_pools_back_exactly():
    e_src, e_tgt = _preds(B=2, h=6, w=10, seed=2)
    for f in (8, 4):
        _, mask, img = edit_mask(accumulate(e_src, e_tgt), 4, 4, f=f)
        assert img.shape == (2, 1, 6 * f, 10 * f)
        assert torch.equal(F.avg_pool2d(img, f), mask)
        assert torch.equal(img[..., ::f, ::f], mask)


def test_edit_mask_symbols_are_exported():
    for s in ('cdx_edit_map', 'cdx_edit_map_from_eps', 'cdx_edit_mask'):
        assert s in _cabi.SIGNATURES and hasattr(_cabi.lib, s)
    from cycle_diffusion_b200.engine import Engine, UNet
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    assert hasattr(UNet, 'edit_map') and hasattr(Engine, 'edit_mask') and hasattr(Engine, 'edit_map_from_eps')
    p = inspect.signature(CycleDiffusionPipeline.generate_mask).parameters
    assert p['num_maps_per_mask'].default == 10 and p['mask_encode_strength'].default == 0.5
    assert p['mask_thresholding_ratio'].default == 3.0 and p['num_inference_steps'].default == 50
