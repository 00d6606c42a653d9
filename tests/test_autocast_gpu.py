"""precision="autocast" (mma mode 5) on the GPU: the one-term fused attention kernel, the networks and latent loops against the
reference run under CUDA autocast's cast policy (tests/golden/make_golden_autocast.py), and the scoped switch in the wrappers and
the pipeline.

Every network bound comes from the fixture's own e_ref: the relative error (max |delta| / max |y|) of the reference's autocast
output against its fp32 output.  Mode 5 keeps activations in fp32 and rounds only the tensor-core inputs, so it should be at least
as close to fp32 as the reference's autocast is."""
import pytest
import torch

from cycle_diffusion_b200 import specs
from tests.common import NARROW, VAE_SMALL, WIDE, golden, maxdiff

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def eng():
    from cycle_diffusion_b200.engine import Engine
    return Engine(0)


def rel(a, b):
    return maxdiff(a.cpu(), b.cpu()) / float(b.abs().max())


def _encode_noise(sched, n_rec, shape):
    noise = torch.zeros((n_rec + 1,) + tuple(shape))
    noise[0] = torch.randn(shape)
    for i in range(n_rec):
        if sched.refine_steps - 1 - i != 0:
            noise[1 + i] = torch.randn(shape)
    return noise


def _attn_ref(q, k, v, heads, scale):
    B, N, C = q.shape
    d = C // heads
    sp = lambda x: x.double().view(B, x.shape[1], heads, d).transpose(1, 2)
    p = torch.softmax(sp(q) @ sp(k).transpose(-1, -2) * scale, dim=-1)
    return (p @ sp(v)).transpose(1, 2).reshape(B, N, C)


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize('N,Nk,heads,d', [(1024, 1024, 8, 40), (256, 256, 8, 80), (1024, 77, 8, 40), (256, 77, 8, 80), (512, 77, 4, 64)])
def test_op_attention_one_term(eng, N, Nk, heads, d):
    g = torch.Generator(device=eng.device).manual_seed(N + Nk + d)
    B = 2
    q, k, v = (torch.randn(B, n, heads * d, device=eng.device, generator=g) for n in (N, Nk, Nk))
    scale = d ** -0.5
    ref = _attn_ref(q, k, v, heads, scale)
    outs = {}
    try:
        for m in (1, 4, 5):
            eng.set_mma_mode(m)
            outs[m] = eng.op_attention(q, k, v, heads, scale).cpu()
    finally:
        eng.set_mma_mode(1)
    e5, e1 = rel(outs[5], ref), rel(outs[1], ref)
    print(f'attention N{N} Nk{Nk} d{d}: mode 5 rel {e5:.2e}, mode 1 rel {e1:.2e}')
    assert e5 < 4e-3                                  # fp16 inputs, fp32 accumulation
    assert not torch.equal(outs[5], outs[1])          # the one-term kernel ran
    assert torch.equal(outs[4], outs[1])              # mode 4 keeps the three-term attention


# ------------------------------------------------------------------------------------------------ networks
@pytest.mark.parametrize('tag,cfg', [('wide', WIDE), ('narrow', NARROW)])
def test_unet_autocast_fixture(eng, tag, cfg):
    from cycle_diffusion_b200.engine import UNet
    g = golden('unet_sd_autocast')
    unet = UNet(eng, cfg, 'openai').load_state_dict(specs.synth_state_dict(specs.openai_unet_params(cfg), int(g[f'seed_{tag}'])))
    y32, yac = g[f'y32_{tag}'], g[f'yac_{tag}']
    e_ref = rel(yac, y32)
    with eng.precision('autocast'):
        y = unet(g[f'x_{tag}'], g[f't_{tag}'], g[f'ctx_{tag}']).cpu()
    full = unet(g[f'x_{tag}'], g[f't_{tag}'], g[f'ctx_{tag}']).cpu()
    print(f'unet[{tag}]: e_ref {e_ref:.2e}  mode 5 vs fp32 {rel(y, y32):.2e}  vs ref autocast {rel(y, yac):.2e}  full vs fp32 {rel(full, y32):.2e}')
    assert rel(y, y32) <= 2 * e_ref
    assert rel(y, yac) <= 3 * e_ref
    assert eng.mma_mode == 1 and rel(full, y32) < 1e-4


def test_vae_autocast_fixture(eng):
    from cycle_diffusion_b200.engine import VAE
    g = golden('vae_autocast')
    vae = VAE(eng, VAE_SMALL).load_state_dict(specs.synth_state_dict(specs.kl_vae_params(VAE_SMALL), int(g['seed'])))
    with eng.precision('autocast'):
        m = vae.encode_moments(g['img']).cpu()
        r = vae.decode(g['z']).cpu()
    for name, y, y32, yac in (('moments', m, g['moments32'], g['momentsac']), ('rec', r, g['rec32'], g['recac'])):
        e_ref = rel(yac, y32)
        print(f'vae {name}: e_ref {e_ref:.2e}  mode 5 vs fp32 {rel(y, y32):.2e}  vs ref autocast {rel(y, yac):.2e}')
        assert rel(y, y32) <= 2 * e_ref
        assert rel(y, yac) <= 3 * e_ref


# ------------------------------------------------------------------------------------------------ latent loops
def _cycle_setup(eng):
    from cycle_diffusion_b200.engine import UNet
    from cycle_diffusion_b200.schedule import DDIMSchedule
    g = golden('ddim_cycle_autocast')
    S, skip, wb, enc_scale, dec_scale, seed = [float(v) for v in g['cfg']]
    sched = DDIMSchedule(int(S), 0.1, int(skip))
    unet = UNet(eng, NARROW, 'openai').load_state_dict(specs.synth_state_dict(specs.openai_unet_params(NARROW), 11))
    torch.manual_seed(int(seed))
    noise = _encode_noise(sched, sched.refine_steps, g['x0'].shape)
    return g, unet, sched, noise, enc_scale, dec_scale


def test_cycle_lockstep_autocast(eng):
    g, unet, sched, noise, enc_scale, dec_scale = _cycle_setup(eng)
    e_ref = rel(g['tgtac'], g['tgt32'])
    with eng.precision('autocast'):
        out = unet.cycle_lockstep(g['x0'], g['c_src'], g['c_tgt'], g['uc'], enc_scale, dec_scale, sched, noise).cpu()
    print(f'cycle lock-step: e_ref {e_ref:.2e}  mode 5 vs fp32 {rel(out, g["tgt32"]):.2e}')
    assert rel(out, g['tgt32']) <= 2 * e_ref


def test_cycle_two_phase_ens_autocast(eng):
    g, unet, sched, noise, enc_scale, dec_scale = _cycle_setup(eng)
    e_ref = rel(g['tgtac'], g['tgt32'])
    B = g['x0'].shape[0]
    with eng.precision('autocast'):
        z = unet.latent_encode_ens(g['x0'], g['c_src'], g['uc'], [enc_scale] * B, sched, sched.refine_steps, noise)
        out = unet.latent_decode_ens(z, g['c_tgt'], g['uc'], [dec_scale] * B, sched).cpu()
    print(f'cycle two-phase: e_ref {e_ref:.2e}  mode 5 vs fp32 {rel(out, g["tgt32"]):.2e}')
    assert rel(out, g['tgt32']) <= 2 * e_ref


# ------------------------------------------------------------------------------------------------ wrappers, pipeline, scope
def _wrapper(eng, **kw):
    from cycle_diffusion_b200.wrappers import SDStochasticTextWrapper, SyntheticTextEncoder
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    vsd = specs.synth_state_dict(specs.kl_vae_params(VAE_SMALL), 21)
    sd = {'model.diffusion_model.' + k: v for k, v in usd.items()}
    sd.update({'first_stage_model.' + k: v for k, v in vsd.items()})
    args = dict(custom_steps=6, eta=0.1, white_box_steps=7, skip_steps=[2], encoder_unconditional_guidance_scales=[1.0],
                decoder_unconditional_guidance_scales=[3.0], n_trials=1)
    args.update(kw)
    return SDStochasticTextWrapper('synthetic', engine=eng, state_dict=sd, cond_stage=SyntheticTextEncoder(48), unet_config=NARROW,
                                   vae_config=VAE_SMALL, latent_size=16, resolution=128, **args)


IMAGE = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(0))
SRC, TGT = ['a photo of a cat', 'a tree'], ['a photo of a dog', 'a tree in winter']


def _cycle_bound():
    # Images, not latents: around the latent cycle the wrappers add the VAE encode, the posterior sample and the VAE decode.  The
    # posterior's std = exp(logvar / 2) turns the moments' fp16-level relative error into a relative error of std scaled by |logvar|
    # (up to ~10 with synthetic weights), and the decoder carries the latent's error through 1 / 0.18215 and ~30 layers.  Hence a
    # factor 16 over the latent cycle's e_ref; a scope that did not take effect gives a zero difference instead.
    g = golden('ddim_cycle_autocast')
    return 16 * rel(g['tgtac'], g['tgt32'])


def test_wrapper_cycle_autocast(eng):
    w = _wrapper(eng)
    assert w.single_member()
    res = {}
    for prec in ('full', 'autocast'):
        w.precision = prec
        torch.manual_seed(5)
        res[prec] = w.cycle(IMAGE, SRC, TGT).cpu()
    d = rel(res['autocast'], res['full'])
    print(f'wrapper cycle: autocast vs full {d:.2e} (bound {_cycle_bound():.2e})')
    assert not torch.equal(res['autocast'], res['full'])
    assert d <= _cycle_bound()
    assert eng.mma_mode == 1


def test_wrapper_ensemble_autocast(eng):
    """Batched encode() + forward() of a two-member ensemble (two encoder scales); the ranking runs outside the scope."""
    ranker = lambda img, orig, et, dt: (None, -((img - orig.to(img.device)) ** 2).mean(dim=(1, 2, 3)))
    w = _wrapper(eng, encoder_unconditional_guidance_scales=[1.0, 2.0])
    w.directional_clip = ranker
    res, gens = {}, {}
    for prec in ('full', 'autocast'):
        w.precision = prec
        torch.manual_seed(9)
        z = w.encode(IMAGE, SRC)
        assert len(z) == 2
        st = torch.get_rng_state()
        gens[prec] = [x.cpu() for x in w.generate(z, TGT)]
        torch.set_rng_state(st)
        res[prec] = w(z, IMAGE, SRC, TGT).cpu()
        assert eng.mma_mode == 1
    for a, b in zip(gens['autocast'], gens['full']):
        assert not torch.equal(a, b)
        assert rel(a, b) <= _cycle_bound()
    d = rel(res['autocast'], res['full'])
    print(f'wrapper ensemble: autocast vs full {d:.2e}, members {[round(rel(a, b), 6) for a, b in zip(gens["autocast"], gens["full"])]}')
    assert not torch.equal(res['autocast'], res['full'])
    assert d <= _cycle_bound()


def test_scope_restores_mode(eng):
    from cycle_diffusion_b200.engine import UNet
    g = golden('unet_sd_autocast')
    unet = UNet(eng, NARROW, 'openai').load_state_dict(specs.synth_state_dict(specs.openai_unet_params(NARROW), 11))
    call = lambda: unet(g['x_narrow'], g['t_narrow'], g['ctx_narrow']).cpu()
    before = call()
    w = _wrapper(eng)
    w.precision = 'autocast'
    torch.manual_seed(5)
    w.cycle(IMAGE, SRC, TGT)
    assert eng.mma_mode == 1
    assert torch.equal(call(), before)                # bit-identical fp32 call after an autocast call
    with pytest.raises(RuntimeError, match='inside'):
        with eng.precision('autocast'):
            assert eng.mma_mode == 5
            raise RuntimeError('inside the scope')
    assert eng.mma_mode == 1
    assert torch.equal(call(), before)
    eng.set_mma_mode(3)                               # a tool running in mode 3 keeps it
    try:
        with eng.precision('autocast'):
            assert eng.mma_mode == 5
        assert eng.mma_mode == 3
        with eng.precision('full'):
            assert eng.mma_mode == 3
    finally:
        eng.set_mma_mode(1)


def test_unknown_precision_rejected(eng):
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    w = _wrapper(eng)
    w.precision = 'autocats'
    with pytest.raises(ValueError):
        w.cycle(IMAGE, SRC, TGT)
    with pytest.raises(ValueError):
        w.encode(IMAGE, SRC)
    with pytest.raises(ValueError):
        with eng.precision('half'):
            pass
    with pytest.raises(ValueError):
        CycleDiffusionPipeline(w.generator, precision='fp16')
    assert eng.mma_mode == 1


def test_pipeline_precision(eng):
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    w = _wrapper(eng)
    kw = dict(image=IMAGE, strength=0.8, num_inference_steps=6, guidance_scale=3.0, eta=0.1)
    out = {}
    for prec in ('full', 'autocast'):
        p = CycleDiffusionPipeline(w.generator, precision=prec)
        out[prec] = p(TGT, SRC, generator=torch.Generator().manual_seed(3), **kw).images.cpu()
        assert eng.mma_mode == 1
    d = rel(out['autocast'], out['full'])
    print(f'pipeline: autocast vs full {d:.2e}')
    assert not torch.equal(out['autocast'], out['full'])
    assert d <= _cycle_bound()
    w.precision = 'autocast'
    p = CycleDiffusionPipeline.from_wrapper(w)
    assert p.precision == 'autocast'
    assert torch.equal(p(TGT, SRC, generator=torch.Generator().manual_seed(3), **kw).images.cpu(), out['autocast'])
