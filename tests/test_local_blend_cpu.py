"""Prompt-to-Prompt's LocalBlend on the CPU: the oracle's mask against a literal transcription of P2P's get_mask, the weight identity
the engine's probe relies on, the oracle's no-op settings, word_token_weights, the pipeline's rejections and the C interface."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as nnf

from cycle_diffusion_b200.attn_control import LocalBlend, resolve_local_blend, word_token_weights
from cycle_diffusion_b200.wrappers import ClipTextCondStage, SyntheticTextEncoder
from tests.local_blend_oracle import blend_cycle, grid_mask, upsample4


def p2p_get_mask(x_shape, maps, alpha, use_pool, th):
    """prompt-to-prompt's LocalBlend.get_mask, transcribed: maps [prompts, layers*heads, 1, gh, gw, L], alpha [prompts, 1, 1, 1, 1, L]."""
    k = 1
    maps = (maps * alpha).sum(-1).mean(1)
    if use_pool:
        maps = nnf.max_pool2d(maps, (k * 2 + 1, k * 2 + 1), (1, 1), padding=(k, k))
    mask = nnf.interpolate(maps, size=x_shape)
    mask = mask / mask.max(2, keepdims=True)[0].max(3, keepdims=True)[0]
    mask = mask.gt(th[1 - int(use_pool)])
    mask = mask[:1] + mask
    return mask


def p2p_local_blend(x_shape, maps, alpha, sub, th):
    mask = p2p_get_mask(x_shape, maps, alpha, True, th)
    if sub is not None:
        mask = mask * ~p2p_get_mask(x_shape, maps, sub, False, th)
    return mask.float()


@pytest.mark.parametrize('gh,gw', [(16, 16), (16, 24)])
@pytest.mark.parametrize('case', ['random', 'ties', 'zero', 'constant'])
@pytest.mark.parametrize('subtract', [False, True])
def test_mask_is_p2p_get_mask(gh, gw, case, subtract):
    """The oracle's grid mask (one image: source and target prompt) equals P2P's get_mask on the image, float64 maps over 5 layers x
    2 heads: random, with ties (maps on a coarse lattice), a zero map (empty, no NaN) and a constant map (full above any th < 1)."""
    g = torch.Generator().manual_seed(gh * gw + len(case))
    L, lh = 12, 10
    maps = torch.rand(2, lh, 1, gh, gw, L, generator=g, dtype=torch.float64)
    if case == 'ties':
        maps = (maps * 4).floor() / 4
    alpha = torch.zeros(2, 1, 1, 1, 1, L, dtype=torch.float64)
    alpha[0, ..., 3] = 1.0
    alpha[1, ..., 4:6] = 1.0
    sub = None
    if subtract:
        sub = torch.zeros_like(alpha)
        sub[:, ..., 7] = 1.0
    if case == 'zero':
        maps[..., 3] = 0.0
        maps[1, ..., 4:6] = 0.0
    if case == 'constant':
        maps[..., 3] = 0.5
    th = (0.3, 0.4)
    want = p2p_local_blend((4 * gh, 4 * gw), maps, alpha, sub, th)[1, 0]
    W = (maps * alpha).sum(-1).sum(1)[:, 0]                          # [2, gh, gw]: the sum, not the mean (the scale cancels)
    S = (maps * sub).sum(-1).sum(1)[:, 0] if subtract else None
    got = upsample4(grid_mask(W[:1], W[1:], th[0], *((S[:1], S[1:], th[1]) if subtract else ())))[0, 0].double()
    assert torch.equal(got, want)
    if case == 'zero' and not subtract:
        assert not bool(got.any())
    if case == 'constant':
        assert bool(got.all()) or subtract


@pytest.mark.parametrize('kind', ['replace', 'reweight', 'refine'])
def test_weight_identity(kind):
    """The edited target map contracted with alpha equals the source row's map with weights A alpha (plus, for refine, the own map
    with w * alpha), to 1e-12 in float64: the engine probes that instead of forming the edited map."""
    g = torch.Generator().manual_seed(5)
    H, N, L = 4, 64, 12
    P_src = torch.rand(H, N, L, generator=g, dtype=torch.float64).softmax(-1)
    P_own = torch.rand(H, N, L, generator=g, dtype=torch.float64).softmax(-1)
    A = torch.eye(L, dtype=torch.float64)[torch.randperm(L, generator=g)]
    if kind != 'replace':
        A = A * torch.rand(L, generator=g, dtype=torch.float64) * 3
    w = torch.rand(L, generator=g, dtype=torch.float64) if kind == 'refine' else None
    alpha = torch.zeros(L, dtype=torch.float64)
    alpha[[2, 5]] = 1.0
    edited = torch.einsum('hpw,wn->hpn', P_src, A) + (P_own * w if w is not None else 0)
    explicit = torch.einsum('hpn,n->p', edited, alpha)
    identity = torch.einsum('hpn,n->p', P_src, A @ alpha) + (torch.einsum('hpn,n->p', P_own, w * alpha) if w is not None else 0)
    assert float((explicit - identity).abs().max()) < 1e-12


@pytest.fixture(scope='module')
def tiny():
    from cycle_diffusion_b200 import specs
    from tests.common import NARROW
    usd = specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)
    g = torch.Generator().manual_seed(3)
    B, L = 1, 8
    x0 = torch.randn(B, 4, 8, 8, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(B, L, 48, generator=g) for _ in range(3))
    a_src, a_tgt = torch.zeros(B, L), torch.zeros(B, L)
    a_src[:, 2], a_tgt[:, 2:4] = 1.0, 1.0
    return usd, NARROW, x0, c_src, c_tgt, uc, a_src, a_tgt


def test_oracle_no_ops(tiny):
    """start_step = n: the loop is the unblended P2P loop (p2p_oracle) bit for bit.  th_blend = 0 without subtract: every blended
    step's mask is 1 everywhere (the probabilities are strictly positive), and the result is again the unblended loop's."""
    from tests.p2p_oracle import p2p_cycle
    usd, cfg, x0, c_src, c_tgt, uc, a_src, a_tgt = tiny
    with torch.no_grad():
        torch.manual_seed(1)
        ref, _ = p2p_cycle(usd, cfg, x0, c_src, c_tgt, uc, 4, 0.1, 1, 1.0, 3.0, 2, 1, 64)
        torch.manual_seed(1)
        late, _ = blend_cycle(usd, cfg, x0, c_src, c_tgt, uc, 4, 0.1, 1, 1.0, 3.0, a_src, a_tgt, 3, 0.3, cross_steps=2, self_steps=1,
                              self_max_tokens=64)
        rec = []
        torch.manual_seed(1)
        full, _ = blend_cycle(usd, cfg, x0, c_src, c_tgt, uc, 4, 0.1, 1, 1.0, 3.0, a_src, a_tgt, 0, 0.0, cross_steps=2, self_steps=1,
                              self_max_tokens=64, record=rec)
    assert torch.equal(late, ref) and torch.equal(full, ref)
    assert all(bool((r['mask'] == 1).all()) for r in rec) and len(rec) == 3
    assert all(bool((r['R'] > 0).all()) for r in rec)


def test_word_token_weights():
    """Multi-token words, repeated words (every occurrence), an absent word, and positions past L (dropped)."""
    ids = [49406, 320, 1929, 2368, 537, 320, 1929, 2368, 49407]
    w = word_token_weights(ids, [1929, 2368], 12)
    assert w.tolist() == [0, 0, 1, 1, 0, 0, 1, 1, 0, 0, 0, 0]
    assert word_token_weights(ids, [537], 12).nonzero().flatten().tolist() == [4]
    assert word_token_weights(ids, [1929, 2368], 7).tolist() == [0, 0, 1, 1, 0, 0, 1]
    with pytest.raises(ValueError):
        word_token_weights(ids, [999], 12)
    with pytest.raises(ValueError):
        word_token_weights(ids, [537], 4)                            # only past L
    syn = SyntheticTextEncoder(8, n_tokens=10)
    got = syn.word_token_weights(['a cat on a mat', 'a red cat'], [('cat', 'mat'), ('red cat',)])
    assert got.shape == (2, 10) and got[0].nonzero().flatten().tolist() == [2, 5] and got[1].nonzero().flatten().tolist() == [2, 3]
    assert syn.word_token_weights(['a cat', 'the cat'], 'cat')[:, 2].tolist() == [1.0, 1.0]


class _ToyTokenizer:
    """Word -> one or two ids (a 'multi-token' word), start 49406, end 49407, zero padding to 16."""
    VOCAB = {'a': [320], 'cat': [2368], 'dog': [1929], 'hotdog': [1929, 3], 'on': [525], 'grass': [4]}

    def __call__(self, texts):
        rows = []
        for t in texts:
            ids = [49406] + [i for word in t.split() for i in self.VOCAB[word]] + [49407]
            rows.append(ids + [0] * (16 - len(ids)))
        return torch.tensor(rows)


def test_clip_stage_weights():
    stage = object.__new__(ClipTextCondStage)
    stage.tokenizer = _ToyTokenizer()
    got = stage.word_token_weights(['a hotdog on grass', 'a cat'], [('hotdog',), ('cat',)])
    assert got.shape == (2, 16) and got[0].nonzero().flatten().tolist() == [2, 3] and got[1].nonzero().flatten().tolist() == [2]
    with pytest.raises(ValueError):
        stage.word_token_weights(['a cat'], 'dog')


def test_local_blend_validation():
    a = torch.zeros(8)
    a[2] = 1.0
    LocalBlend(a, a)
    for bad in (dict(alpha_src=torch.zeros(8)), dict(alpha_src=-a), dict(alpha_src=a * float('nan')), dict(sub_src=a),
                dict(threshold=(1.0, 0.3)), dict(threshold=(0.3,)), dict(start_blend=1.5), dict(alpha_src=[1.0])):
        with pytest.raises(ValueError):
            LocalBlend(**{'alpha_src': a, 'alpha_tgt': a, **bad})
    syn = SyntheticTextEncoder(8, n_tokens=10)
    lb = resolve_local_blend({'words': ('cat', 'dog'), 'subtract_words': ('mat', 'mat'), 'threshold': (0.2, 0.5)}, syn,
                             ['a cat on a mat'], ['a dog on a mat'])
    assert lb.threshold == (0.2, 0.5) and lb.start_blend == 0.2 and lb.sub_tgt[0, 5] == 1
    with pytest.raises(ValueError):
        resolve_local_blend({'word': ('cat', 'dog')}, syn, ['a cat'], ['a dog'])
    with pytest.raises(ValueError):
        resolve_local_blend({'words': ('cow', 'dog')}, syn, ['a cat'], ['a dog'])


def test_pipeline_rejections():
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline
    parse = CycleDiffusionPipeline._local_blend
    spec = {'words': ('cat', 'dog')}
    ok = {'edit_type': 'replace', 'cross_replace_steps': 0.5, 'self_replace_steps': 0.5, 'local_blend': spec}
    assert parse(ok, 1.0, 7.5, False, None) is spec and parse({'local_blend': spec}, 1.0, 7.5, False, None) is spec
    assert parse({'scale': 1.0}, 1.0, 7.5, False, None) is None
    assert CycleDiffusionPipeline._attn_control(ok, 1.0, False).cross_steps == 0.5
    for args in ((ok, 1.0, 7.5, True, None), (ok, 1.0, 7.5, False, 'glasses'), (ok, 0.0, 7.5, False, None), (ok, 1.0, 0.0, False, None),
                 ({'local_blend': spec, 'token_map': None}, 1.0, 7.5, False, None)):
        with pytest.raises(ValueError):
            parse(*args)
    for kind in ('mutual_self', 'pnp'):
        with pytest.raises(ValueError):
            CycleDiffusionPipeline._attn_control({'edit_type': kind, 'local_blend': spec}, 1.0, False)


def test_c_interface():
    from cycle_diffusion_b200 import _cabi
    for name in ('cdx_cycle_lockstep_blend', 'cdx_local_blend_mask', 'cdx_op_attention_net_weighted'):
        assert hasattr(_cabi.lib, name)
    f = _cabi.LocalBlendC
    assert [x[0] for x in f._fields_] == ['alpha_src', 'alpha_tgt', 'sub_src', 'sub_tgt', 'start_step', 'th_blend', 'th_sub']
    assert f.start_step.offset == 32 and f.th_sub.offset == 40 and C.sizeof(f) == 48
