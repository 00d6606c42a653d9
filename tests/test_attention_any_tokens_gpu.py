"""The fused attention kernel at any token count and at 160-channel heads: ragged query / key tiles (N not a multiple of 128, per-image
key counts off the 8-key TMA granule), d = 160 (SD v1 / LDM levels 3 and mid), and the U-Net sizes that put every attention level on
those shapes.  No N x N score matrix is materialised: each attention is one `batched_tc` launch, with no softmax or FFMA family."""
import pytest
import torch

from cycle_diffusion_b200 import specs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def engs():
    from cycle_diffusion_b200.engine import Engine
    out = {}
    for m in (1, 3, 4, 5):
        out[m] = Engine(0)
        out[m].set_mma_mode(m)
    return out


def _attn_ref(q, k, v, heads, scale):
    B, N, C = q.shape
    d = C // heads
    sp = lambda x: x.double().view(B, x.shape[1], heads, d).transpose(1, 2)
    p = torch.softmax(sp(q) @ sp(k).transpose(-1, -2) * scale, dim=-1)
    return (p @ sp(v)).transpose(1, 2).reshape(B, N, C)


def _run(eng, q, k, v, heads, scale):
    eng.profile(True)
    y = eng.op_attention(q, k, v, heads, scale)
    fam = eng.profile_read()
    eng.profile(False)
    return y, fam


def _check_modes(engs, B, N, Nk, heads, d):
    dev = engs[1].device
    g = torch.Generator(device=dev).manual_seed(N * 7 + Nk + d + B)
    C = heads * d
    q = torch.randn(B, N, C, device=dev, generator=g) * 1.5
    k, v = (torch.randn(B, Nk, C, device=dev, generator=g) for _ in range(2))
    scale = d ** -0.5
    ref = _attn_ref(q, k, v, heads, scale)
    ys = {}
    for m in (1, 3, 4, 5):
        if m == 3 and d > 80:
            continue                      # TF32 planes at d = 160 keep the unfused route
        y, fam = _run(engs[m], q, k, v, heads, scale)
        assert 'batched_tc' in fam and fam['batched_tc']['launches'] == 1, (m, fam)
        assert 'softmax' not in fam and 'batched_ffma' not in fam, (m, sorted(fam))
        ys[m] = y.double()
    err = {m: float((y - ref).abs().max()) for m, y in ys.items()}
    r5 = float((ys[5] - ref).abs().max() / ref.abs().max())
    print(f'attention B{B} N{N} Nk{Nk} h{heads} d{d}: max abs err {err}  mode 5 rel {r5:.2e}')
    assert err[1] < 2e-5
    if 3 in err:
        assert err[3] < 2e-5
    assert torch.equal(ys[4], ys[1])                 # mode 4 keeps the three-term attention
    assert r5 < 4e-3 and not torch.equal(ys[5], ys[1])


@pytest.mark.parametrize('d', [16, 40, 64, 80, 160])
@pytest.mark.parametrize('N', [16, 64, 81, 144, 200, 576, 1600, 5184])
@pytest.mark.parametrize('B', [1, 3])
def test_self_attention_any_tokens(engs, B, N, d):
    _check_modes(engs, B, N, N, 2, d)


@pytest.mark.parametrize('d', [16, 40, 64, 80, 160])
@pytest.mark.parametrize('N', [16, 81, 200, 576])
@pytest.mark.parametrize('B', [1, 3])
def test_cross_attention_any_tokens(engs, B, N, d):
    _check_modes(engs, B, N, 77, 2, d)


@pytest.mark.parametrize('sq,sk,sv', [(1e3, 1e-3, 1.0), (1e-4, 1e4, 3e4), (1.0, 1.0, 1e-10), (2e-3, 5e2, 1e6)])
def test_attention_h16_d160_ragged_is_scale_invariant(engs, sq, sk, sv):
    """As test_attention_h16_is_scale_invariant, at d = 160 and a ragged token count (the key-split kernel's merge and the row guard)."""
    e = engs[1]
    B, N, heads, d = 2, 200, 2, 160
    g = torch.Generator().manual_seed(77)
    C = heads * d
    q, k, v = (torch.randn(B, N, C, generator=g) for _ in range(3))
    q, k, v = q * 1.5 * sq, k * sk, v * sv
    ref = _attn_ref(q, k, v, heads, d ** -0.5)
    y, fam = _run(e, q.cuda(), k.cuda(), v.cuda(), heads, d ** -0.5)
    r = float((y.cpu().double() - ref).abs().max() / ref.abs().max())
    print(f'attention d160 N200 scales q{sq:g} k{sk:g} v{sv:g}: rel err {r:.2e}')
    assert fam['batched_tc']['launches'] == 1
    assert r < 2e-5


# ------------------------------------------------------------------------------------------------ networks
@pytest.fixture(scope='module')
def sd_unet():
    from cycle_diffusion_b200.engine import Engine, UNet
    cfg = specs.sd_unet_config(768)
    sd = specs.synth_state_dict(specs.openai_unet_params(cfg), 1234)
    return cfg, sd, (lambda eng: UNet(eng, cfg, 'openai').load_state_dict(sd)), Engine


def test_sd_v1_unet_576(sd_unet):
    """SD v1 at 576x576 (latent 72x72): 5184 / 1296 / 324 / 81 tokens, all fused, against the CPU oracle."""
    from oracle import unet_openai
    cfg, sd, make, Engine = sd_unet
    eng = Engine(0)
    net = make(eng)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 4, 72, 72, generator=g)
    ctx = torch.randn(2, 77, 768, generator=g)
    t = torch.tensor([981., 21.])
    eng.profile(True)
    y = net(x, t, ctx).cpu()
    fam = eng.profile_read()
    eng.profile(False)
    with torch.no_grad():
        ref = unet_openai.unet_forward(sd, cfg, x, t.long(), ctx)
    r = float((y.double() - ref.double()).abs().max() / ref.double().abs().max())
    print(f'SD v1 U-Net 72x72 B2: rel max err vs oracle {r:.3e}  families {sorted(fam)}')
    assert 'softmax' not in fam, sorted(fam)
    assert r < 2e-4


def test_sd_v1_unet_960_twelve_rows(sd_unet):
    """SD v1 at 960x960 (latent 120x120, 14400 tokens at level 0) with 12 rows on a fresh engine.  An unfused level-0 layer would
    allocate 12 rows x 8 heads x 14400^2 x 4 B = 79.6 GB of scores; the whole workspace (the U-Net's O(N C) activations) stays below
    the scores of a single head of that layer, 12 x 14400^2 x 4 B = 9.95 GB."""
    cfg, sd, make, Engine = sd_unet
    eng = Engine(0)
    net = make(eng)
    g = torch.Generator().manual_seed(9)
    R = 12
    x = torch.randn(R, 4, 120, 120, generator=g)
    ctx = torch.randn(R, 77, 768, generator=g)
    t = torch.linspace(981., 1., R)
    y = net(x, t, ctx).cpu()
    ws = eng.workspace_bytes
    print(f'SD v1 U-Net 120x120 x{R}: workspace {ws / 1e9:.2f} GB')
    assert ws < R * 14400 ** 2 * 4
    worst = 0.0
    for i in range(R):
        yi = net(x[i:i + 1], t[i:i + 1], ctx[i:i + 1]).cpu()
        worst = max(worst, float((y[i:i + 1].double() - yi.double()).abs().max() / yi.double().abs().max()))
    print(f'  max row-vs-1-row rel diff {worst:.2e}')
    assert worst < 2e-4
