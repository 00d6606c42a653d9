"""The lock-step ensemble search (cdx_latent_cycle_fan + cdx_ensemble_select, _StochasticTextWrapperBase.cycle_ensemble) against the
engine's two-phase drivers, the two-phase wrapper path and the CPU oracle: per-chain parity, U-Net rows, model routing, the selection
rule, device memory, precision scope and the fallback."""
import pytest
import torch

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.ensemble import guidance_rows
from tests.common import NARROW, VAE_SMALL, maxdiff
from tests.test_clip_rank_gpu import TC, VC, _sd as _clip_sd

pytestmark = pytest.mark.gpu

KW = dict(custom_steps=6, eta=0.1, white_box_steps=7, skip_steps=[2, 3], encoder_unconditional_guidance_scales=[1.0, 3.0],
          decoder_unconditional_guidance_scales=[1.0, 0.0, 3.0], n_trials=2)
SRC, TGT = ['enc:0', 'enc:1'], ['dec:0', 'dec:1']


@pytest.fixture(scope='module')
def eng():
    from cycle_diffusion_b200.engine import Engine
    return Engine(0)


def _weights():
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    vsd = specs.synth_state_dict(specs.kl_vae_params(VAE_SMALL), 21)
    sd = {'model.diffusion_model.' + k: v for k, v in usd.items()}
    sd.update({'first_stage_model.' + k: v for k, v in vsd.items()})
    return usd, vsd, sd


def _dclip(eng):
    """The small synthetic CLIP of test_clip_rank_gpu.py; the stub tokenizer maps 'enc:i' / 'dec:i' to rows of the fixture ids."""
    from cycle_diffusion_b200.clip_rank import DirectionalCLIP
    from tests.common import golden
    g = golden('clip_rank')
    table = {'enc': g['ids_e'].long(), 'dec': g['ids_d'].long()}
    tok = lambda texts: torch.stack([table[t.split(':')[0]][int(t.split(':')[1])] for t in texts])
    return DirectionalCLIP(eng, _clip_sd(), tok, vision_cfg=VC, text_cfg=TC)


def _wrapper(cls, eng, ranker, **over):
    from cycle_diffusion_b200.wrappers import SyntheticTextEncoder
    kw = dict(KW, **over)
    return cls('synthetic', engine=eng, state_dict=_weights()[2], cond_stage=SyntheticTextEncoder(48), unet_config=NARROW,
               vae_config=VAE_SMALL, latent_size=16, resolution=128, ranker=ranker, **kw)


def _l1_ranker(calls=None, engine=None):
    def rank(img, orig, et, dt):
        if calls is not None:
            calls.append(engine.mma_mode)
        return None, -(img - orig.to(img.device)).flatten(1).abs().mean(1)
    return rank


def _fan_inputs(seed=0):
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(3, 4, 16, 16, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(3, 77, 48, generator=g) for _ in range(3))
    return x0, c_src, c_tgt, uc


def test_fan_driver_vs_two_phase(eng):
    """Three source chains at encoder scales 1, 3, 0, each driving decoder scales [1, 0, 3]: every target latent and every z equal
    latent_encode_ens + latent_decode_ens on the same noise (bounds of test_lockstep_driver_vs_reference_fixture_and_two_phase)."""
    from cycle_diffusion_b200.engine import UNet
    from cycle_diffusion_b200.schedule import DDIMSchedule
    unet = UNet(eng, NARROW, 'openai').load_state_dict(_weights()[0])
    x0, c_src, c_tgt, uc = _fan_inputs()
    src, dec = [1.0, 3.0, 0.0], [1.0, 0.0, 3.0]
    sched = DDIMSchedule(6, 0.1, 2)
    n = sched.refine_steps
    noise = torch.randn(n + 1, 3, 4, 16, 16, generator=torch.Generator().manual_seed(1))
    noise[n] = 0                                                                     # index 0 draws nothing (ddim.py:583-584)
    out, z = unet.cycle_fan(x0, c_src, c_tgt, uc, src, [dec] * 3, sched, noise, return_z=True)
    z2 = unet.latent_encode_ens(x0, c_src, uc, src, sched, n, noise)
    rep = lambda t: t.to(eng.device).repeat_interleave(3, dim=0)
    out2 = unet.latent_decode_ens(rep(z2), rep(c_tgt), rep(uc), dec * 3, sched)
    rz = maxdiff(z.cpu(), z2.cpu()) / float(z2.abs().max())
    dx = maxdiff(out.cpu(), out2.cpu())
    print(f'fan vs two-phase: rel|dz| {rz:.2e}  |dx| {dx:.2e}  bit-identical x {bool(torch.equal(out, out2))}')
    assert out.shape == (9, 4, 16, 16) and z.shape == (3, n + 1, 4, 16, 16)
    assert rz < 2e-5 and dx < 1e-4


def test_fan_runs_only_the_rows_its_scales_need(eng):
    """conv3x3 FLOPs of one loop == rows x steps x those of a batch-1 U-Net call (shape-derived, so exact): chains at scale 1 or 0
    ran one row."""
    from cycle_diffusion_b200.engine import UNet
    from cycle_diffusion_b200.schedule import DDIMSchedule
    unet = UNet(eng, NARROW, 'openai').load_state_dict(_weights()[0])
    x0, c_src, c_tgt, uc = _fan_inputs(2)
    src, dec = [1.0, 3.0, 0.0], [1.0, 0.0, 3.0]
    sched = DDIMSchedule(6, 0.1, 2)
    noise = torch.randn(sched.refine_steps + 1, 3, 4, 16, 16)
    conv = lambda r: sum(v['flops'] for k, v in r.items() if k.startswith('conv3x3'))
    eng.profile(True)
    unet.cycle_fan(x0, c_src, c_tgt, uc, src, [dec] * 3, sched, noise)
    loop = conv(eng.profile_read())
    eng.profile(True)
    unet(x0[:1], torch.tensor([500.0]), c_src[:1])
    one = conv(eng.profile_read())
    eng.profile(False)
    rows = sum(guidance_rows(s) for s in src) + 3 * sum(guidance_rows(s) for s in dec)
    print(f'fan rows {rows} (two-phase chains would run {2 * 3 * (1 + len(dec))}): conv3x3 {loop:.4g} FLOP = {loop / one:.3f} batch-1 calls')
    assert rows == 16 and one > 0
    assert loop == rows * sched.refine_steps * one


@pytest.mark.parametrize('kind', ['sd', 'ldm'])
def test_model_forward_vs_two_phase_and_oracle(eng, kind):
    """TextUnsupervisedTranslation.forward takes the lock-step path for a ranked ensemble; its scores, choice and image agree with
    encode() + rank() under the same seed and with the CPU oracle's candidate."""
    from cycle_diffusion_b200.models import TextUnsupervisedTranslation
    from cycle_diffusion_b200.wrappers import SyntheticTextEncoder
    from oracle import dpm_encoder, unet_openai, vae_kl
    usd, vsd, sd = _weights()
    dclip = _dclip(eng)
    gan_type = {'sd': 'SDStochasticText', 'ldm': 'LatentDiffStochasticText'}[kind]
    cond = SyntheticTextEncoder(48)
    m = TextUnsupervisedTranslation(dict(gan=dict(gan_type=gan_type, source_model_type='synthetic', **KW)), engine=eng, state_dict=sd,
                                    cond_stage=cond, unet_config=NARROW, vae_config=VAE_SMALL, latent_size=16, resolution=128,
                                    ranker=dclip).eval()
    w = m.gan_wrapper
    assert w.lockstep_ensemble() and not w.single_member()
    image = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(5))
    torch.manual_seed(77)
    (_, img), _, _ = m(torch.tensor([0, 1]), image, SRC, TGT)
    torch.manual_seed(77)
    img_c, idx, scores = w.cycle_ensemble(image, SRC, TGT)
    assert torch.equal(img, img_c)
    torch.manual_seed(77)
    z = w.encode(image, SRC)
    cands = [eng.shift_scale(i, 1.0, 0.5) for i in w.generate(z, TGT)]
    _, idx2, scores2 = dclip.rank(cands, image, SRC, TGT)
    ora = dpm_encoder.LatentCycle(lambda x, t, c: unet_openai.unet_forward(usd, NARROW, x, t, c),
                                  lambda im: vae_kl.encode_moments(vsd, VAE_SMALL, im), lambda zz: vae_kl.decode(vsd, VAE_SMALL, zz), cond,
                                  channels=4, latent_size=16, resolution=128, sample_posterior=(kind == 'sd'), **KW)
    torch.manual_seed(77)
    with torch.no_grad():
        imgs_ref = ora.forward_all(ora.encode(image, SRC), TGT)
    n_cand = len(imgs_ref)
    assert scores.shape == scores2.shape == (2, n_cand) == (2, 2 * 2 * 2 * 3) and idx.dtype == torch.int64
    ds = maxdiff(scores.cpu(), scores2.cpu())
    top2 = scores2.cpu().topk(2, dim=1).values
    gap = top2[:, 0] - top2[:, 1]
    di = max(maxdiff(img[b].cpu(), imgs_ref[int(idx[b])][b]) for b in range(2))
    print(f'{kind} ensemble: |d score| {ds:.2e}  index {idx.tolist()} vs two-phase {idx2.tolist()} (gap {gap.tolist()})  |d img| vs oracle {di:.2e}')
    assert ds < 1e-4
    for b in range(2):
        if gap[b] > 1e-3:
            assert int(idx[b]) == int(idx2[b])
    assert di < 1e-3


def test_select_ties_nans_and_arrival_order(eng):
    nan = float('nan')
    mat = torch.tensor([[0.5, 0.9, 0.9, 0.1, nan, 0.9, nan],
                        [0.2, 0.7, 0.1, 0.7, 0.7, -1.0, 0.3],
                        [-float('inf')] * 7,
                        [0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.6]])
    B, n = mat.shape
    imgs = torch.randn(B, n, 3, 8, 8, generator=torch.Generator().manual_seed(3))
    entries = torch.randperm(B * n, generator=torch.Generator().manual_seed(4))
    sel = eng.ensemble_select(B, n, 8, 8)
    for part in (entries[:9], entries[9:20], entries[20:]):
        b, c = part // n, part % n
        sel.add(mat[b, c], c, b, imgs[b, c])
    best = torch.argmax(mat, dim=1)
    assert torch.equal(sel.best_idx.cpu(), best)
    got = sel.scores.cpu()
    assert torch.equal(got.isnan(), mat.isnan()) and torch.equal(got.nan_to_num(), mat.nan_to_num())
    for b in range(B):
        assert torch.equal(sel.best_img[b].cpu(), imgs[b, best[b]])


def test_device_memory_does_not_grow_with_the_ensemble():
    """Peak of torch allocations + engine workspace at n_trials 1 and 4: the lock-step path grows by < 1 MiB; the two-phase path by
    at least the extra z it keeps."""
    from cycle_diffusion_b200.engine import Engine
    from cycle_diffusion_b200.wrappers import SDStochasticTextWrapper
    image = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(6))
    kw = dict(skip_steps=[2, 3], encoder_unconditional_guidance_scales=[1.0], decoder_unconditional_guidance_scales=[1.0, 3.0])
    z_per_member = {2: 2 * 5 * 4 * 16 * 16 * 4, 3: 2 * 4 * 4 * 16 * 16 * 4}       # bytes of one member's z [B, n_rec+1, 4,16,16]

    def peak(w, fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        torch.manual_seed(1)
        fn()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() + w.engine.workspace_bytes

    res = {}
    for path in ('lockstep', 'two_phase'):
        e = Engine(0)
        w = _wrapper(SDStochasticTextWrapper, e, _l1_ranker(), ensemble_rows=2 * (1 + 1 + 2), **kw)    # one member per chunk
        fn = (lambda: w.cycle_ensemble(image, SRC, TGT)) if path == 'lockstep' else (lambda: w(w.encode(image, SRC), image, SRC, TGT))
        for trials in (1, 4):
            w.n_trials = trials
            res[path, trials] = peak(w, fn)
        del w, e
    grow_l = res['lockstep', 4] - res['lockstep', 1]
    grow_t = res['two_phase', 4] - res['two_phase', 1]
    extra_z = 3 * sum(z_per_member.values())
    print(f'peak growth n_trials 1 -> 4: lock-step {grow_l / 2**20:.3f} MiB, two-phase {grow_t / 2**20:.3f} MiB (extra z {extra_z / 2**20:.3f} MiB)')
    assert grow_l < 2 ** 20
    assert grow_t >= extra_z


def test_precision_scope_loops_inside_ranker_outside(eng):
    from cycle_diffusion_b200.wrappers import SDStochasticTextWrapper
    calls, loops = [], []
    w = _wrapper(SDStochasticTextWrapper, eng, _l1_ranker(calls, eng))
    fan = w.generator.unet.cycle_fan
    w.generator.unet.cycle_fan = lambda *a, **k: (loops.append(eng.mma_mode), fan(*a, **k))[1]
    image = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(8))
    torch.manual_seed(3)
    full = w.cycle_ensemble(image, SRC, TGT)[0]
    w.precision = 'autocast'
    torch.manual_seed(3)
    auto = w.cycle_ensemble(image, SRC, TGT)[0]
    n_chunks = len(w.ensemble_plan(2)[0].chunks)
    print(f'precision: loops ran in modes {sorted(set(loops))}, ranker saw {sorted(set(calls))}; |full - autocast| {maxdiff(full.cpu(), auto.cpu()):.2e}')
    assert loops == [1] * n_chunks + [5] * n_chunks
    assert calls == [1] * (2 * n_chunks)
    assert maxdiff(full.cpu(), auto.cpu()) > 0 and eng.mma_mode == 1

    def boom(*a):
        raise RuntimeError('ranker failed')
    w.directional_clip = boom
    with pytest.raises(RuntimeError, match='ranker failed'):
        w.cycle_ensemble(image, SRC, TGT)
    assert eng.mma_mode == 1


def test_unrecovered_steps_fall_back_to_encode_forward(eng):
    """white_box_steps leaving steps unrecovered: forward is encode() + forward(), bit for bit.  No ranker: the same
    NotImplementedError as before, raised before any sampling."""
    from cycle_diffusion_b200.models import TextUnsupervisedTranslation
    from cycle_diffusion_b200.wrappers import SyntheticTextEncoder
    sd = _weights()[2]
    image = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(9))

    def model(ranker, **over):
        gan = dict(gan_type='SDStochasticText', source_model_type='synthetic', **dict(KW, **over))
        return TextUnsupervisedTranslation(dict(gan=gan), engine=eng, state_dict=sd, cond_stage=SyntheticTextEncoder(48), unet_config=NARROW,
                                           vae_config=VAE_SMALL, latent_size=16, resolution=128, ranker=ranker).eval()

    m = model(_l1_ranker(), white_box_steps=5)
    w = m.gan_wrapper
    assert not w.lockstep_ensemble()
    torch.manual_seed(4)
    (_, img), _, _ = m(torch.tensor([0, 1]), image, SRC, TGT)
    torch.manual_seed(4)
    ref = w(w.encode(image, SRC), image, SRC, TGT)
    assert torch.equal(img, ref)
    m = model(None)
    assert not m.gan_wrapper.lockstep_ensemble()
    torch.manual_seed(4)
    state = torch.get_rng_state()
    with pytest.raises(NotImplementedError):
        m(torch.tensor([0, 1]), image, SRC, TGT)
    assert torch.equal(torch.get_rng_state(), state)
