"""LEDITS++'s implicit masks without a GPU: the oracle's smoothing, map and lambda = 0 loop against independent statements, the
SemanticGuidance fields, the conditioning models' token counts, the pipeline's rejections and the new C symbols."""
import math

import pytest
import torch
import torch.nn.functional as F

from cycle_diffusion_b200 import specs
from cycle_diffusion_b200.semantic import SemanticGuidance
from tests.common import NARROW
from tests.ledits_oracle import channel_sum, head_span_probs, ledits_cycle, record_maps, smooth, smoothing_weights
from tests.sega_oracle import sega_cycle


def diffusers_kernel():
    """GaussianSmoothing(channels=1, kernel_size=3, sigma=0.5, dim=2)'s weights, by its own formula in fp32."""
    kernel = torch.ones(1)
    grids = torch.meshgrid(*[torch.arange(3, dtype=torch.float32)] * 2, indexing='ij')
    for mgrid in grids:
        mean = 1.0
        kernel = kernel * 1 / (0.5 * math.sqrt(2 * math.pi)) * torch.exp(-(((mgrid - mean) / (2 * 0.5)) ** 2))
    return kernel / torch.sum(kernel)


def test_weights_match_diffusers_formula():
    W = smoothing_weights()
    ref = diffusers_kernel()
    assert torch.allclose(W, ref, rtol=4 * 2.0 ** -24, atol=0)
    assert torch.equal(W, W.T) and torch.equal(W, W.flip(0)) and torch.equal(W, W.flip(1))
    # the literals the kernel carries (kernels_elem.cu, LEDITS_W_*)
    assert [float(W[0, 0]).hex(), float(W[0, 1]).hex(), float(W[1, 1]).hex()] == ['0x1.6ffa700000000p-5', '0x1.f422640000000p-4',
                                                                                    '0x1.53e0640000000p-2']


@pytest.mark.parametrize('gh,gw', [(2, 2), (4, 6), (8, 8), (5, 3), (30, 30)])
def test_smoothing_against_conv2d(gh, gw):
    """The oracle's single-op smoothing against F.conv2d on the reflect-padded map with diffusers' weights, within a few ulp."""
    A = torch.rand(3, gh, gw, generator=torch.Generator().manual_seed(gh * 31 + gw)) * 5
    ref = F.conv2d(F.pad(A.unsqueeze(1), (1, 1, 1, 1), mode='reflect'), diffusers_kernel().reshape(1, 1, 3, 3)).squeeze(1)
    got = smooth(A)
    assert got.shape == A.shape
    assert float(((got - ref).abs() / ref.abs()).max()) < 8 * 2.0 ** -24


def test_channel_sum_order():
    psi = torch.randn(2, 4, 5, 6, generator=torch.Generator().manual_seed(1))
    want = ((psi[:, 0].abs() + psi[:, 1].abs()) + psi[:, 2].abs()) + psi[:, 3].abs()
    assert torch.equal(channel_sum(psi), want)


def test_map_against_direct_softmax():
    """head_span_probs against a float64 softmax of the same q and k, per head, summed over the span."""
    g = torch.Generator().manual_seed(5)
    b, n, heads, d, L = 3, 16, 4, 8, 11
    q, k = torch.randn(b, n, heads * d, generator=g), torch.randn(b, L, heads * d, generator=g)
    span = [1, 5, L - 2]
    got = head_span_probs(q, k, heads, span)
    for r in range(b):
        want = torch.zeros(n, dtype=torch.float64)
        for hh in range(heads):
            s = q[r, :, hh * d:(hh + 1) * d].double() @ k[r, :, hh * d:(hh + 1) * d].double().T * d ** -0.5
            want += torch.softmax(s, dim=-1)[:, 1:1 + span[r]].sum(dim=-1)
        assert float((got[r].double() - want).abs().max()) < 1e-5


@pytest.fixture(scope='module')
def usd():
    return specs.synth_state_dict(specs.openai_unet_params(NARROW), 11)


def test_records_the_quarter_resolution_layers(usd):
    """NARROW at a 16x16 latent: input blocks 7, 8 and output blocks 3, 4, 5 are the 4x4 cross-attentions."""
    from oracle import unet_openai
    g = torch.Generator().manual_seed(2)
    x, c = torch.randn(2, 4, 16, 16, generator=g), torch.randn(2, 77, 48, generator=g)
    maps = {}
    with record_maps(16, [3, 75], maps):
        unet_openai.unet_forward(usd, NARROW, x, torch.tensor([10, 10]), c)
    assert maps['layers'] == 5 and maps['A'].shape == (2, 16)
    assert float(maps['A'].max()) <= 2 * 5 + 1e-4       # two heads, five layers, probabilities


@pytest.mark.parametrize('intersect', [False, True])
def test_lambda_zero_is_sega(usd, intersect):
    """At lambda = 0 every mask is all ones, so the oracle is sega_cycle at lambda = 0, bit for bit."""
    from oracle import unet_openai
    from cycle_diffusion_b200.schedule import DDIMSchedule  # noqa: F401  (the schedule tables come from oracle.schedules)
    g = torch.Generator().manual_seed(3)
    B, L = 1, 77
    x0 = torch.randn(B, 4, 16, 16, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(B, L, 48, generator=g) for _ in range(3))
    c_edit = torch.randn(B, 2, L, 48, generator=g)
    args = (x0, c_src, c_tgt, uc, c_edit, 4, 0.1, 1, 1.0, 3.0, [2.0, -1.5], [0.0, 0.0], [3, 2], 1, 0.3, 0.4)
    fn = lambda x, t, c: unet_openai.unet_forward(usd, NARROW, x, t, c)
    with torch.no_grad():
        torch.manual_seed(4)
        y_s, _ = sega_cycle(fn, *args)
        torch.manual_seed(4)
        y_l, _ = ledits_cycle(usd, NARROW, *args, n_tokens=[3, 1], intersect=intersect)
    assert torch.equal(y_s, y_l)


def test_semantic_guidance_fields():
    s = SemanticGuidance.for_concepts(2, use_cross_attn_mask=True, edit_token_counts=[3, 5])
    assert s.mask_mode == 1 and s.edit_token_counts == (3, 5)
    assert SemanticGuidance.for_concepts(2, use_intersect_mask=True, edit_token_counts=4).mask_mode == 2
    assert SemanticGuidance.for_concepts(2).mask_mode == 0
    am = s.attn_mask_struct(77)
    assert am.intersect == 0 and list(am.n_tokens) == [3, 5, 0, 0, 0, 0, 0, 0]
    for kw in (dict(use_cross_attn_mask=True), dict(use_intersect_mask=True), dict(use_cross_attn_mask=1, edit_token_counts=3),
               dict(use_cross_attn_mask=True, edit_token_counts=[3]), dict(use_cross_attn_mask=True, edit_token_counts=0),
               dict(use_cross_attn_mask=True, edit_token_counts=[2, True]), dict(use_cross_attn_mask=True, edit_token_counts=2.0)):
        with pytest.raises(ValueError):
            SemanticGuidance.for_concepts(2, **kw)
    for bad in (0, 76):
        with pytest.raises(ValueError):
            SemanticGuidance.for_concepts(1, use_cross_attn_mask=True, edit_token_counts=bad).attn_mask_struct(77)
    SemanticGuidance.for_concepts(1, use_cross_attn_mask=True, edit_token_counts=75).attn_mask_struct(77)


class _Tok:
    def __init__(self, rows):
        self.rows = rows

    def __call__(self, texts):
        return torch.tensor([self.rows[t] for t in texts])


def test_token_counts():
    from cycle_diffusion_b200.wrappers import BertTextCondStage, ClipTextCondStage, OpenClipTextCondStage, SyntheticTextEncoder
    clip = object.__new__(ClipTextCondStage)
    clip.tokenizer = _Tok({'glasses': [49406, 7, 49407, 49407, 49407], 'a red hat': [49406, 1, 2, 3, 49407], 'long': [49406, 1, 2, 3, 4]})
    assert clip.token_counts(['glasses', 'a red hat', 'long']) == [1, 3, 4]
    oc = object.__new__(OpenClipTextCondStage)
    oc.tokenizer = _Tok({'a hat': [49406, 1, 2, 49407, 0, 0]})
    assert oc.token_counts(['a hat']) == [2]
    bert = object.__new__(BertTextCondStage)
    bert.tokenizer = _Tok({'a hat': [101, 1, 2, 102, 0, 0], 'x': [101, 9, 102, 0, 0, 0]})
    assert bert.token_counts(['a hat', 'x']) == [2, 1]
    assert SyntheticTextEncoder(8).token_counts(['glasses', 'a red  hat', '']) == [1, 3, 0]


def test_c_symbols():
    import ctypes as C
    from cycle_diffusion_b200 import _cabi
    assert hasattr(_cabi.lib, 'cdx_cycle_lockstep_semantic_attn') and hasattr(_cabi.lib, 'cdx_cycle_lockstep_semantic')
    assert issubclass(_cabi.LatentChainsMaskDesc, _cabi.LatentChainsDesc)
    assert [f[0] for f in _cabi.LatentChainsMaskDesc._fields_] == ['sg_map', 'sg_mask', 'sg_gh', 'sg_gw', 'w']
    # the C struct's offsets (include/cdx.h): the pointer starts the trailing fields on the 8-byte boundary where the base ends
    assert _cabi.LatentChainsMaskDesc.sg_map.offset == C.sizeof(_cabi.LatentChainsDesc)
    assert _cabi.LatentChainsMaskDesc.w.offset == _cabi.LatentChainsMaskDesc.sg_map.offset + 8 + 12
    names = [f[0] for f in _cabi.AttentionNetDesc._fields_]
    assert names[-4:] == ['probe_rows', 'probe_spans', 'n_probe', 'probe_map']
    assert [f[0] for f in _cabi.SemanticAttnMaskC._fields_] == ['intersect', 'n_tokens']


def test_pipeline_rejections():
    """A mask flag without editing_prompt, and a conditioning callable without token_counts and no edit_token_counts."""
    from cycle_diffusion_b200.pipeline import CycleDiffusionPipeline

    class G:
        cond_stage = staticmethod(lambda texts: torch.zeros(len(texts), 77, 8))
        get_learned_conditioning = cond_stage

    pipe = object.__new__(CycleDiffusionPipeline)
    pipe.g = G()
    with pytest.raises(ValueError, match='token_counts'):
        pipe._token_counts(['glasses'], None)
    assert pipe._token_counts(['glasses'], [3]) == [3]
    with pytest.raises(ValueError, match='editing_prompt'):
        CycleDiffusionPipeline.__call__(pipe, 'a dog', 'a cat', None, use_cross_attn_mask=True)
