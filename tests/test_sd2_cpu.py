"""SD 2.x without a GPU: engine inventories vs specs, the OpenCLIP -> HF name mapping, the test restatements vs the fixtures, the
float64 v identities, the oracle cycle identity under v, and the wrapper factory."""
import numpy as np
import pytest
import torch

from cycle_diffusion_b200 import specs
from tests import sd2_oracle
from tests.common import golden, maxdiff

NARROW2 = dict(in_channels=4, out_channels=4, model_channels=64, attention_resolutions=(4, 2, 1), num_res_blocks=1,
               channel_mult=(1, 2, 2), num_head_channels=32, context_dim=40, use_linear_in_transformer=True)
OPENCLIP_SMALL = specs.openclip_h14_text_config(layers=2, total_layers=3, vocab_size=1000, width=64, heads=4, mlp_width=256)


@pytest.fixture(scope='module')
def lib():
    from cycle_diffusion_b200 import _build
    _build.build()


@pytest.mark.parametrize('cfg', [specs.sd2_unet_config(), NARROW2])
def test_unet_inventory_matches_specs(lib, cfg):
    from cycle_diffusion_b200.engine import UNet
    u = UNet(None, cfg)
    assert u.inventory() == [(n, tuple(s)) for n, s, _ in specs.openai_unet_params(cfg)]
    # the engine stores the Linear projections as the equivalent 1x1 convolutions
    eng_inv = dict(u._engine_inventory())
    C = cfg['model_channels']
    assert eng_inv['input_blocks.1.1.proj_in.weight'] == (C, C, 1, 1) and dict(u.inventory())['input_blocks.1.1.proj_in.weight'] == (C, C)


def test_unet_heads_need_whole_head_width(lib):
    from cycle_diffusion_b200.engine import UNet
    with pytest.raises(AssertionError, match='whole heads'):
        UNet(None, dict(NARROW2, num_head_channels=48))


def test_openclip_inventory_and_mapping(lib):
    from cycle_diffusion_b200.engine import TextEncoder
    full = specs.openclip_h14_text_config()
    inv = TextEncoder(None, full).inventory()
    small = dict(full, vocab_size=50, width=32, heads=2, mlp_width=64)     # the same names at a size that is cheap to draw
    oc = specs.synth_state_dict(specs.openclip_text_params(small), 3)
    hf = specs.openclip_to_hf(oc, full['layers'])
    assert sorted(n for n, _ in inv) == sorted(hf) and len(inv) == 4 + 16 * 23
    assert dict(inv)['text_model.encoder.layers.22.mlp.fc1.weight'] == (4096, 1024)
    assert not any('.layers.23.' in n for n, _ in inv)                   # "penultimate": block 23 never runs
    back = specs.hf_to_openclip(hf, full['layers'])
    assert set(back) == {k for k in oc if k not in ('text_projection', 'logit_scale') and '.resblocks.23.' not in k}
    assert all(torch.equal(back[k], oc[k]) for k in back)
    q, k, v = (hf[f'text_model.encoder.layers.5.self_attn.{n}.weight'] for n in ('q_proj', 'k_proj', 'v_proj'))
    assert torch.equal(torch.cat([q, k, v]), oc['transformer.resblocks.5.attn.in_proj_weight'])


def test_unet_oracle_matches_fixture():
    g = golden('unet_sd2_narrow')
    sd = specs.synth_state_dict(specs.openai_unet_params(NARROW2), int(g['seed']))
    with torch.no_grad():
        y = sd2_oracle.unet_forward(sd, NARROW2, g['x'], g['t'], g['ctx'])
    assert maxdiff(y, g['y']) / float(g['y'].abs().max()) < 1e-5


def test_openclip_oracle_matches_fixture():
    """The fixture's transformers output equals a direct restatement of encode_with_transformer on the OpenCLIP-named weights."""
    import torch.nn.functional as F
    g = golden('openclip_text')
    c = OPENCLIP_SMALL
    sd = specs.synth_state_dict(specs.openclip_text_params(c), int(g['seed']), gain=float(g['gain']))
    ids = g['ids'].long()
    W, H = c['width'], c['heads']
    x = sd['token_embedding.weight'][ids] + sd['positional_embedding']
    L = ids.shape[1]
    mask = torch.full((L, L), float('-inf')).triu(1)
    for l in range(c['layers']):
        p = f'transformer.resblocks.{l}.'
        h = F.layer_norm(x, (W,), sd[p + 'ln_1.weight'], sd[p + 'ln_1.bias'])
        q, k, v = F.linear(h, sd[p + 'attn.in_proj_weight'], sd[p + 'attn.in_proj_bias']).chunk(3, dim=-1)
        sp = lambda t: t.view(t.shape[0], L, H, W // H).transpose(1, 2)
        a = torch.softmax(sp(q) * (W // H) ** -0.5 @ sp(k).transpose(-1, -2) + mask, dim=-1) @ sp(v)
        x = x + F.linear(a.transpose(1, 2).reshape(-1, L, W), sd[p + 'attn.out_proj.weight'], sd[p + 'attn.out_proj.bias'])
        h = F.layer_norm(x, (W,), sd[p + 'ln_2.weight'], sd[p + 'ln_2.bias'])
        x = x + F.linear(F.gelu(F.linear(h, sd[p + 'mlp.c_fc.weight'], sd[p + 'mlp.c_fc.bias'])), sd[p + 'mlp.c_proj.weight'], sd[p + 'mlp.c_proj.bias'])
    y = F.layer_norm(x, (W,), sd['ln_final.weight'], sd['ln_final.bias'])
    assert maxdiff(y, g['out']) < 1e-4


def test_v_identities_float64():
    """x_t = sa pred_x0 + s1 e_t and v = sa e_t - s1 pred_x0: the conversion of the step kernels (e_t = sa v + s1 x_t,
    pred_x0 = sa x_t - s1 v) inverts the definition of v."""
    from cycle_diffusion_b200.schedule import ldm_alphas_cumprod_f64, v_tables
    ac = ldm_alphas_cumprod_f64()
    sa64, s164 = np.sqrt(ac), np.sqrt(1.0 - ac)
    sa, s1 = v_tables()
    assert sa.dtype == np.float32 and np.array_equal(sa, sa64.astype(np.float32)) and np.array_equal(s1, s164.astype(np.float32))
    ora_sa, ora_s1 = sd2_oracle.v_tables()
    assert np.array_equal(ora_sa.numpy(), sa) and np.array_equal(ora_s1.numpy(), s1)
    rng = np.random.default_rng(0)
    x0, eps = rng.standard_normal((2, 1000)), rng.standard_normal((2, 1000))
    for t in (1, 251, 501, 999):
        xt = sa64[t] * x0 + s164[t] * eps
        v = sa64[t] * eps - s164[t] * x0
        e_t, pred_x0 = sa64[t] * v + s164[t] * xt, sa64[t] * xt - s164[t] * v
        assert np.abs(e_t - eps).max() < 1e-12 and np.abs(pred_x0 - x0).max() < 1e-12
        assert np.abs(sa64[t] * pred_x0 + s164[t] * e_t - xt).max() < 1e-12
        assert np.abs(sa64[t] * e_t - s164[t] * pred_x0 - v).max() < 1e-12


def test_v_cycle_oracle_matches_fixture_and_reconstructs():
    g = golden('ddim_cycle_v')
    S, skip, eta, enc, dec = g['cfg'].tolist()
    S, skip = int(S), int(skip)
    sd = specs.synth_state_dict(specs.openai_unet_params(NARROW2), int(g['seed']))
    fn = lambda x, t, c: sd2_oracle.unet_forward(sd, NARROW2, x, t, c)
    torch.manual_seed(int(g['noise_seed']))
    with torch.no_grad():
        z = torch.stack(sd2_oracle.latent_encode(fn, g['x0'], g['c_src'], g['uc'], S, eta, skip, enc, 'v'), dim=1)
        same = sd2_oracle.latent_decode(fn, z[:, 0], z[:, 1:], g['c_src'], g['uc'], S, eta, skip, enc, 'v')
    assert maxdiff(z, g['z']) / float(g['z'].abs().max()) < 1e-5
    assert maxdiff(same, g['same']) < 1e-4
    assert maxdiff(same, g['x0']) < 1e-3 and maxdiff(g['same'], g['x0']) < 1e-3      # cycle identity (SURVEY 4)
    assert maxdiff(g['tgt'], g['x0']) > 1e-2                                           # another condition does change the result


def test_factory_resolves_sd2():
    from cycle_diffusion_b200 import wrappers
    seen = {}

    class Stub:
        def __init__(self, **kw):
            seen.update(kw)
    orig = wrappers.SD2StochasticTextWrapper
    wrappers.SD2StochasticTextWrapper = Stub
    try:
        w = wrappers.get_gan_wrapper(dict(gan_type='SD2StochasticText', source_model_type='v2-1_768-ema-pruned.ckpt', custom_steps=50,
                                          parameterization='v', target_model_type='x'))
    finally:
        wrappers.SD2StochasticTextWrapper = orig
    assert isinstance(w, Stub) and seen == dict(source_model_type='v2-1_768-ema-pruned.ckpt', custom_steps=50, parameterization='v')
    assert issubclass(orig, wrappers._StochasticTextWrapperBase) and orig.CONTEXT_DIM == 1024
    assert orig.COND_PREFIX == 'cond_stage_model.model.' and orig.COND_CLASS is wrappers.OpenClipTextCondStage
    assert orig.RESOLUTIONS == {'eps': 512, 'v': 768}
