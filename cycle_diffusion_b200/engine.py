"""Python handles over the libcdx C ABI: Engine (per device), UNet / VAE networks, per-step kernels, loop drivers.

PyTorch is used only as plumbing: device memory (``torch.empty(..., device='cuda')``), streams and
``torch.distributed``.  Every compute call goes through ctypes into hand-written sm_90a kernels; there is no
torch.nn / CPU fallback anywhere on this path.
"""
import contextlib
import ctypes as C
import math

import torch

from . import _cabi
from ._cabi import lib, check, UnetConfig, VaeConfig, TextConfig, DdimCoef, PixelCoef
from .attn_control import LocalBlend, MutualSelfControl, PnPControl
from .schedule import EditFriendlySchedule
from .semantic import SemanticGuidance


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _f32c(t, device):
    assert t.dtype == torch.float32, f'expected float32, got {t.dtype}'
    if t.device != device:
        t = t.to(device)
    return t.contiguous()


def check_mask(mask, shape, device, what='mask'):
    """A masked-editing mask from the caller: float32 of exactly ``shape`` ([B,1,h,w]), finite, every value in [0, 1] (1 = may
    change).  Raises ValueError otherwise; returns it contiguous on ``device``."""
    if not torch.is_tensor(mask) or mask.dtype != torch.float32:
        raise ValueError(f'{what}: expected a float32 tensor, got {getattr(mask, "dtype", type(mask))}')
    if tuple(mask.shape) != tuple(shape):
        raise ValueError(f'{what}: shape {tuple(mask.shape)}, expected {tuple(shape)}')
    if not bool(torch.isfinite(mask).all()) or bool((mask < 0).any()) or bool((mask > 1).any()):
        raise ValueError(f'{what}: values must be finite and within [0, 1]')
    return _f32c(mask, device)


class Engine:
    """One per CUDA device / rank.  Not thread-safe; all work is enqueued on the current torch stream."""

    def __init__(self, device=0):
        if not torch.cuda.is_available():
            raise RuntimeError('cycle_diffusion_b200 needs a CUDA device: the engine has no CPU fallback')
        self.device = torch.device('cuda', device if isinstance(device, int) else torch.device(device).index or 0)
        torch.cuda.set_device(self.device)
        h = C.c_void_p()
        check(lib.cdx_engine_create(self.device.index, C.byref(h)))
        self.h = h
        self.mma_mode = 1                # what cdx_engine_create selects

    def close(self):
        if getattr(self, 'h', None):
            lib.cdx_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    @property
    def launches(self):
        return int(lib.cdx_engine_launch_count(self.h))

    @property
    def workspace_bytes(self):
        return int(lib.cdx_engine_workspace_bytes(self.h))

    def set_mma_mode(self, mode):
        check(lib.cdx_engine_set_mma_mode(self.h, int(mode)))
        self.mma_mode = int(mode)

    def set_persist(self, enable, max_ctas=0):
        """Persistent tensor-core GEMM for unsplit dense fp16-split work: on by default (CDX_PERSIST=0 at creation: off).
        max_ctas > 0 caps its grid, so each CTA walks more work items (tests); outputs are bit-identical in every setting."""
        check(lib.cdx_engine_set_persist(self.h, int(bool(enable)), int(max_ctas)))

    # the reference wrappers' `precision` values (SDW:117, txt2img.py --precision {full,autocast}) and the mma mode each selects;
    # None: the engine keeps its current mode
    PRECISIONS = {'full': None, 'autocast': 5}

    @contextlib.contextmanager
    def precision(self, precision):
        """``with engine.precision('autocast'):`` runs the enclosed calls in mma mode 5 (single-term fp16 weight GEMMs, convs and
        fused attention, fp32 activations and accumulation) and restores the previous mode on exit, also on an exception.
        ``'full'`` leaves the current mode as it is.  Any other value raises ValueError."""
        if precision not in self.PRECISIONS:
            raise ValueError(f'precision must be one of {sorted(self.PRECISIONS)}, got {precision!r}')
        mode, prev = self.PRECISIONS[precision], self.mma_mode
        if mode is None:
            yield self
            return
        self.set_mma_mode(mode)
        try:
            yield self
        finally:
            self.set_mma_mode(prev)

    PROF_TAGS = ['conv3x3_ffma', 'dense_ffma', 'batched_ffma', 'conv3x3_tc', 'dense_tc', 'batched_tc', 'groupnorm', 'layernorm',
                 'softmax', 'other']

    def profile(self, enable):
        check(lib.cdx_engine_profile(self.h, int(enable)))

    def profile_read(self):
        """{tag: dict(ms, flops, bytes, launches)} of everything recorded since profile(True)."""
        out = {}
        for i, name in enumerate(self.PROF_TAGS):
            ms, fl, by, n = C.c_double(), C.c_double(), C.c_double(), C.c_uint64()
            check(lib.cdx_engine_profile_read(self.h, i, C.byref(ms), C.byref(fl), C.byref(by), C.byref(n)))
            if n.value:
                out[name] = dict(ms=ms.value, flops=fl.value, bytes=by.value, launches=int(n.value))
        return out

    def empty(self, *shape):
        return torch.empty(*shape, dtype=torch.float32, device=self.device)

    # ------------------------------------------------------------------ per-step kernels
    def affine(self, x, a, b):
        x = _f32c(x, self.device)
        out = torch.empty_like(x)
        check(lib.cdx_affine(self.h, _ptr(x), a, b, _ptr(out), x.numel(), self.stream))
        return out

    def shift_scale(self, x, b, a):
        x = _f32c(x, self.device)
        out = torch.empty_like(x)
        check(lib.cdx_shift_scale(self.h, _ptr(x), b, a, _ptr(out), x.numel(), self.stream))
        return out

    def mask_pool(self, mask, f):
        """Image-resolution mask [B,1,H,W] in [0,1] -> latent-resolution [B,1,H/f,W/f], the mean of each f x f block (f: the first
        stage's factor); equals torch.nn.functional.avg_pool2d(mask, f) to within 1 ulp."""
        if mask.dim() != 4 or mask.shape[1] != 1 or mask.shape[2] % f or mask.shape[3] % f:
            raise ValueError(f'mask: expected [B,1,H,W] with H, W multiples of {f}, got {tuple(mask.shape)}')
        mask = check_mask(mask, mask.shape, self.device)
        B, _, H, W = mask.shape
        out = self.empty(B, 1, H // f, W // f)
        check(lib.cdx_mask_pool(self.h, _ptr(mask), _ptr(out), B, H, W, int(f), self.stream))
        return out

    def op_local_blend_mask(self, maps, n_terms, n_vec, run, h, w, th_blend, th_sub, user_mask=None):
        """LocalBlend's mask stage alone (cdx_local_blend_mask): maps [B*n_vec*n_terms, (h/4)(w/4)] of one step are added into the
        running sums run [B*n_vec, (h/4)(w/4)] (updated in place) -> the latent mask [B,1,h,w] (times user_mask [B,1,h,w] when given)."""
        B = run.shape[0] // n_vec
        for name, t in (('maps', maps), ('run', run), ('user_mask', user_mask)):
            assert t is None or (torch.is_tensor(t) and t.dtype == torch.float32 and t.device == self.device and t.is_contiguous()), \
                f'op_local_blend_mask: {name} must be a contiguous float32 tensor on {self.device}'
        out = self.empty(B, 1, h, w)
        check(lib.cdx_local_blend_mask(self.h, _ptr(maps), int(n_terms), int(n_vec), _ptr(run), _ptr(user_mask), float(th_blend), float(th_sub),
                                       _ptr(out), B, h, w, self.stream))
        return out

    def mask_composite(self, dec, image, mask):
        """Paste-back: dec [B,C,H,W] (first-stage output in [-1,1]), image [B,C,H,W] in [0,1], mask [B,1,H,W] ->
        m * clamp((dec + 1) * 0.5, 0, 1) + (1 - m) * image; exactly the image where m == 0, the clamped decode where m == 1."""
        dec, image = _f32c(dec, self.device), _f32c(image, self.device)
        B, Cc, H, W = dec.shape
        if tuple(image.shape) != tuple(dec.shape):
            raise ValueError(f'image shape {tuple(image.shape)} != decode shape {tuple(dec.shape)}')
        mask = check_mask(mask, (B, 1, H, W), self.device)
        out = torch.empty_like(dec)
        check(lib.cdx_mask_composite(self.h, _ptr(dec), _ptr(image), _ptr(mask), _ptr(out), B, Cc, H, W, self.stream))
        return out

    def edit_map_from_eps(self, e_src, e_tgt, vscale=1.0, maps_per_launch=None):
        """DiffEdit accumulation on given predictions (cdx_edit_map_from_eps): e_src, e_tgt [B,n,C,h,w] -> acc [B,h,w], acc[b] the
        sum over maps k ascending of sum_c |vscale * (e_tgt[b,k] - e_src[b,k])|, fp32.  Bit-identical for any maps_per_launch
        (default: all n maps in one launch)."""
        e_src, e_tgt = _f32c(e_src, self.device), _f32c(e_tgt, self.device)
        assert e_src.dim() == 5 and e_src.shape == e_tgt.shape, f'{tuple(e_src.shape)} vs {tuple(e_tgt.shape)}'
        B, n, Cc, h, w = e_src.shape
        acc = self.empty(B, h, w)
        check(lib.cdx_edit_map_from_eps(self.h, _ptr(e_src), _ptr(e_tgt), float(vscale), n, int(maps_per_launch or n), _ptr(acc), B, Cc,
                                        h, w, self.stream))
        return acc

    def edit_mask(self, acc, n_maps, ratio=3.0, f=None, channels=4):
        """DiffEdit mask from the accumulator of UNet.edit_map (cdx_edit_mask): acc [B,h,w] over n_maps maps of a `channels`-channel
        latent -> (map [B,1,h,w] = acc / (n_maps * channels), mask [B,1,h,w] in {0, 1}, mask_img [B,1,f*h,f*w] or None when f is
        None).  Per image, mask = min(map, M) / M > 0.5 with M = ratio * mean(map); an all-zero map gives an all-zero mask.
        mask_img is the mask nearest-upsampled by f (the first stage's factor), ready for the pipeline's ``mask_image``."""
        if not ratio > 0:
            raise ValueError(f'mask_thresholding_ratio must be > 0, got {ratio}')
        acc = _f32c(acc, self.device)
        B, h, w = acc.shape
        emap, mask = self.empty(B, 1, h, w), self.empty(B, 1, h, w)
        img = self.empty(B, 1, f * h, f * w) if f else None
        check(lib.cdx_edit_mask(self.h, _ptr(acc), int(n_maps), float(ratio), _ptr(emap), _ptr(mask), _ptr(img), int(f or 1), B,
                                int(channels), h, w, self.stream))
        return emap, mask, img

    def q_sample(self, x0, noise, sqrt_a, sqrt_1ma):
        x0, noise = _f32c(x0, self.device), _f32c(noise, self.device)
        out = torch.empty_like(x0)
        check(lib.cdx_q_sample(self.h, _ptr(x0), _ptr(noise), sqrt_a, sqrt_1ma, _ptr(out), x0.numel(), self.stream))
        return out

    def vae_posterior(self, moments, noise, scale_factor):
        moments = _f32c(moments, self.device)
        B, C2, h, w = moments.shape
        out = self.empty(B, C2 // 2, h, w)
        if noise is not None:
            noise = _f32c(noise, self.device)
            assert noise.shape == out.shape
        check(lib.cdx_vae_posterior(self.h, _ptr(moments), _ptr(noise), scale_factor, _ptr(out), B, C2 // 2, h * w, self.stream))
        return out

    def ddim_posterior_sample(self, x0, xt, noise, coef):
        x0, xt, noise = (_f32c(t, self.device) for t in (x0, xt, noise))
        out = torch.empty_like(x0)
        check(lib.cdx_ddim_posterior_sample(self.h, _ptr(x0), _ptr(xt), _ptr(noise), C.byref(coef), _ptr(out), x0.numel(), self.stream))
        return out

    def ddim_compute_eps(self, xt, xt_next, e_c, e_uc, scale, coef):
        xt, xt_next, e_c = (_f32c(t, self.device) for t in (xt, xt_next, e_c))
        e_uc = _f32c(e_uc, self.device) if e_uc is not None else None
        out = torch.empty_like(xt)
        check(lib.cdx_ddim_compute_eps(self.h, _ptr(xt), _ptr(xt_next), _ptr(e_c), _ptr(e_uc), scale, C.byref(coef), _ptr(out),
                                       xt.numel(), self.stream))
        return out

    def ddim_step_with_eps(self, x, e_c, e_uc, scale, eps, coef):
        x, e_c, eps = (_f32c(t, self.device) for t in (x, e_c, eps))
        e_uc = _f32c(e_uc, self.device) if e_uc is not None else None
        out = torch.empty_like(x)
        check(lib.cdx_ddim_step_with_eps(self.h, _ptr(x), _ptr(e_c), _ptr(e_uc), scale, _ptr(eps), C.byref(coef), _ptr(out),
                                         x.numel(), self.stream))
        return out

    def pixel_posterior_sample(self, x0, xt, noise, coef):
        x0, xt, noise = (_f32c(t, self.device) for t in (x0, xt, noise))
        out = torch.empty_like(x0)
        check(lib.cdx_pixel_posterior_sample(self.h, _ptr(x0), _ptr(xt), _ptr(noise), C.byref(coef), _ptr(out), x0.numel(), self.stream))
        return out

    def pixel_compute_eps(self, xt, xt_next, et, coef):
        xt, xt_next, et = (_f32c(t, self.device) for t in (xt, xt_next, et))
        B = xt.shape[0]
        out = torch.empty_like(xt)
        check(lib.cdx_pixel_compute_eps(self.h, _ptr(xt), _ptr(xt_next), _ptr(et), C.byref(coef), _ptr(out), B, xt[0].numel(),
                                        et[0].numel(), self.stream))
        return out

    def pixel_step_with_eps(self, xt, et, eps, coef):
        xt, et = _f32c(xt, self.device), _f32c(et, self.device)
        eps = _f32c(eps, self.device) if eps is not None else None
        B = xt.shape[0]
        out = torch.empty_like(xt)
        check(lib.cdx_pixel_step_with_eps(self.h, _ptr(xt), _ptr(et), _ptr(eps), C.byref(coef), _ptr(out), B, xt[0].numel(),
                                          et[0].numel(), self.stream))
        return out

    # ------------------------------------------------------------------ unit-test hooks (NHWC)
    def op_conv3x3(self, x_nhwc, w_oihw, bias, stride=1, pad_lo=1, upsample=1):
        x, w = _f32c(x_nhwc, self.device), _f32c(w_oihw, self.device)
        bias = _f32c(bias, self.device) if bias is not None else None
        B, H, W, Cin = x.shape
        Cout = w.shape[0]
        Hl, Wl = H * upsample, W * upsample
        Ho, Wo = (Hl, Wl) if stride == 1 else (Hl // 2, Wl // 2)
        y = self.empty(B, Ho, Wo, Cout)
        check(lib.cdx_op_conv3x3(self.h, _ptr(x), _ptr(w), _ptr(bias), _ptr(y), B, H, W, Cin, Cout, stride, pad_lo, upsample, self.stream))
        return y

    def op_linear(self, x, w, bias):
        x, w = _f32c(x, self.device), _f32c(w, self.device)
        bias = _f32c(bias, self.device) if bias is not None else None
        M, K = x.shape
        N = w.shape[0]
        y = self.empty(M, N)
        check(lib.cdx_op_linear(self.h, _ptr(x), _ptr(w), _ptr(bias), _ptr(y), M, K, N, self.stream))
        return y

    # ---- Directional-CLIP ranking / evaluation metrics (SURVEY 8f-3)
    def clip_preprocess(self, img, size=224):
        """clean_clip.py:14-17 on a float batch in [0,1]: bicubic resize to size x size + CLIP normalisation."""
        x = _f32c(img, self.device)
        B, Cc, R, R2 = x.shape
        assert Cc == 3 and R == R2, 'square RGB batches (the reference feeds R x R sampler outputs)'
        out = self.empty(B, 3, size, size)
        check(lib.cdx_clip_preprocess(self.h, _ptr(x), B, R, size, _ptr(out), self.stream))
        return out

    def dclip_scores(self, img_f, orig_f, enc_f, dec_f):
        fs = [_f32c(t, self.device) for t in (img_f, orig_f, enc_f, dec_f)]
        B, D = fs[0].shape
        clip, dclip = self.empty(B), self.empty(B)
        check(lib.cdx_dclip_scores(self.h, *[_ptr(t) for t in fs], B, D, _ptr(clip), _ptr(dclip), self.stream))
        return clip, dclip

    def image_metrics(self, a, b):
        """-> [B, 3] = (psnr, ssim, l2) per image pair (evaluation/translate_text.py:76-89)."""
        a, b = _f32c(a, self.device), _f32c(b, self.device)
        B, Cc, H, W = a.shape
        assert Cc == 3 and a.shape == b.shape
        out = self.empty(B, 3)
        check(lib.cdx_image_metrics(self.h, _ptr(a), _ptr(b), B, H, W, _ptr(out), self.stream))
        return out

    def ensemble_select(self, B, n_candidates, H, W):
        """Running per-sample best of an ensemble whose candidates arrive in chunks (cdx_ensemble_select): returns an
        EnsembleSelection holding best_img [B,3,H,W], best_idx [B] (int64), best_score [B] and the score matrix
        scores [B, n_candidates] on this engine's device."""
        return EnsembleSelection(self, B, n_candidates, H, W)

    def op_groupnorm(self, x_nhwc, gamma, beta, eps, silu):
        x, gamma, beta = (_f32c(t, self.device) for t in (x_nhwc, gamma, beta))
        B, H, W, Cc = x.shape
        y = torch.empty_like(x)
        check(lib.cdx_op_groupnorm(self.h, _ptr(x), _ptr(gamma), _ptr(beta), eps, int(silu), _ptr(y), B, H * W, Cc, self.stream))
        return y

    def op_layernorm(self, x, gamma, beta):
        x, gamma, beta = (_f32c(t, self.device) for t in (x, gamma, beta))
        M, Cc = x.shape
        y = torch.empty_like(x)
        check(lib.cdx_op_layernorm(self.h, _ptr(x), _ptr(gamma), _ptr(beta), _ptr(y), M, Cc, self.stream))
        return y

    def _gn_operands(self, x1, x2, gamma, beta, scale, shift):
        x1, gamma, beta = (_f32c(t, self.device) for t in (x1, gamma, beta))
        B, H, W, C1 = x1.shape
        x2 = _f32c(x2, self.device) if x2 is not None else None
        C2 = x2.shape[3] if x2 is not None else 0
        assert (scale is None) == (shift is None)
        ld_ss = 0
        if scale is not None:
            for t in (scale, shift):
                assert t.dtype == torch.float32 and t.device == self.device and tuple(t.shape) == (B, C1 + C2) and t.stride(1) == 1
            assert scale.stride(0) == shift.stride(0), 'scale and shift share one row stride'
            ld_ss = scale.stride(0)
        return x1, x2, gamma, beta, B, H, W, C1, C2, ld_ss

    def op_groupnorm_ex(self, x1, x2, gamma, beta, eps, silu, scale=None, shift=None):
        """GroupNorm(32) of the channel concat [x1 | x2] (NHWC [B,H,W,C1], [B,H,W,C2] or None) as the network executors run it,
        optional gn(x) * (1 + scale) + shift and SiLU.  scale / shift: [B, C] device views with unit column stride and one common
        row stride (e.g. the two halves of a [B, 2C] embedding projection).  Returns (y, amax, ab): y [B,H,W,C], amax [1] the
        tracked range slot of y, ab [B, C, 2] the (a, o) table the norm applies, y = silu?(x * a + o)."""
        x1, x2, gamma, beta, B, H, W, C1, C2, ld_ss = self._gn_operands(x1, x2, gamma, beta, scale, shift)
        y = self.empty(B, H, W, C1 + C2)
        amax = torch.zeros(1, dtype=torch.float32, device=self.device)
        ab = self.empty(B, C1 + C2, 2)
        check(lib.cdx_op_groupnorm_ex(self.h, _ptr(x1), C1, _ptr(x2), C2, _ptr(gamma), _ptr(beta), eps, int(silu), _ptr(scale), _ptr(shift),
                                      ld_ss, _ptr(y), _ptr(amax), _ptr(ab), B, H * W, self.stream))
        return y, amax, ab

    def op_groupnorm_rows(self, x1, x2, gamma, beta, eps, silu, src_rows, scale=None, shift=None):
        """op_groupnorm_ex's norm twice from one set of statistics (cdx_op_groupnorm_rows): plain, and with the row table src_rows
        ([B] ints), image b of the second being image src_rows[b]'s norm.  Returns (y, amax, y_rows, amax_rows), amax / amax_rows [1]
        the tracked range slots."""
        x1, x2, gamma, beta, B, H, W, C1, C2, ld_ss = self._gn_operands(x1, x2, gamma, beta, scale, shift)
        rows = [int(r) for r in src_rows]
        assert len(rows) == B, f'src_rows: {len(rows)} entries for {B} images'
        y, y_rows = self.empty(B, H, W, C1 + C2), self.empty(B, H, W, C1 + C2)
        amax, amax_rows = (torch.zeros(1, dtype=torch.float32, device=self.device) for _ in range(2))
        check(lib.cdx_op_groupnorm_rows(self.h, _ptr(x1), C1, _ptr(x2), C2, _ptr(gamma), _ptr(beta), eps, int(silu), _ptr(scale), _ptr(shift),
                                        ld_ss, (C.c_int * B)(*rows), _ptr(y), _ptr(amax), _ptr(y_rows), _ptr(amax_rows), B, H * W, self.stream))
        return y, amax, y_rows, amax_rows

    def op_layernorm_ex(self, x, gamma, beta):
        """LayerNorm over the last dim of x [M, C] (eps 1e-5) -> (y, amax [1] the tracked range slot of y)."""
        x, gamma, beta = (_f32c(t, self.device) for t in (x, gamma, beta))
        M, Cc = x.shape
        y = torch.empty_like(x)
        amax = torch.zeros(1, dtype=torch.float32, device=self.device)
        check(lib.cdx_op_layernorm_ex(self.h, _ptr(x), _ptr(gamma), _ptr(beta), _ptr(y), _ptr(amax), M, Cc, self.stream))
        return y, amax

    def op_softmax_rows(self, x, causal_nq=0):
        """Row softmax of x [rows, L] in place (x is returned); causal_nq > 0: row r sees columns j <= r % causal_nq only."""
        assert x.dtype == torch.float32 and x.device == self.device and x.is_contiguous()
        rows, L = x.shape
        check(lib.cdx_op_softmax_rows(self.h, _ptr(x), rows, L, L, int(causal_nq), self.stream))
        return x

    PRODUCE_PATHS = ('ffma', 'fused', 'tc_standalone', 'splitk')

    def op_produce_norm(self, x, w, bias, gamma, beta, eps, conv=False):
        """A producer GEMM with its GroupNorm side outputs wired as the executors wire them, then the GroupNorm that trusts them.
        Linear: x [B, HW, Cin], w [Cout, Cin]; conv: NHWC x [B, H, W, Cin], w OIHW [Cout, Cin, 3, 3] (stride 1, pad 1).
        Returns (y [B*HW, Cout], amax [1], stats [B, Cout, 2] float64, yn [B*HW, Cout], path), path one of PRODUCE_PATHS."""
        x, w, gamma, beta = (_f32c(t, self.device) for t in (x, w, gamma, beta))
        bias = _f32c(bias, self.device) if bias is not None else None
        if conv:
            B, H, W, Cin = x.shape
        else:
            B, HW, Cin = x.shape
            H, W = HW, 1
        Cout = w.shape[0]
        y = self.empty(B * H * W, Cout)
        yn = self.empty(B * H * W, Cout)
        amax = torch.zeros(1, dtype=torch.float32, device=self.device)
        stats = torch.empty(B, Cout, 2, dtype=torch.float64, device=self.device)
        path = C.c_int(-1)
        check(lib.cdx_op_produce_norm(self.h, _ptr(x), _ptr(w), _ptr(bias), int(bool(conv)), B, H, W, Cin, Cout, _ptr(gamma), _ptr(beta),
                                      eps, _ptr(y), _ptr(amax), _ptr(stats), _ptr(yn), C.byref(path), self.stream))
        return y, amax, stats, yn, self.PRODUCE_PATHS[path.value]

    GEMM_POINTERS = ('A', 'A2', 'w', 'bias', 'rowvec', 'residual', 'C', 'C_lo', 'Ct_hi', 'Ct_lo', 'a_amax', 'a2_amax', 'c_amax', 'c_stats')
    GEMM_KINDS = ('ss', 'ts', 'h16', 'h16_fast')

    def op_gemm(self, **fields):
        """One contraction through the production GEMM with any of its epilogue terms (cdx_op_gemm in include/cdx.h, whose
        cdx_gemm_desc fields are the keyword arguments).  Every buffer is a float32 tensor (c_stats: float64) on this engine's
        device, passed as it is -- a view at an offset or a column slice keeps its address, so the strides (lda, ldc, ...) are the
        caller's.  Outputs land in the caller's C / C_lo / Ct_hi / Ct_lo / c_amax / c_stats.  Defaults: alpha 1, stride 1, pad 1, up 1,
        one image per row block.  Returns the plan the call ran: dict(kind: 'ffma' or one of GEMM_KINDS, width: tile width
        (FFMA: tile side), splits: split-K factor, amax_fused, stats_fused: side outputs made by the tensor-core epilogue)."""
        d = _cabi.GemmDesc(alpha=1.0, stride=1, pad=1, batch=1, heads=1, rows_per_batch=1, up=1)
        for name, v in fields.items():
            if name in self.GEMM_POINTERS:
                if v is not None:
                    want = torch.float64 if name == 'c_stats' else torch.float32
                    assert torch.is_tensor(v) and v.dtype == want and v.device == self.device, f'op_gemm: {name} must be a {want} tensor on {self.device}'
                setattr(d, name, v.data_ptr() if v is not None else None)
            else:
                assert hasattr(d, name), f'op_gemm: no field {name}'
                setattr(d, name, v)
        plan = C.c_int(0)
        check(lib.cdx_op_gemm(self.h, C.byref(d), C.byref(plan), self.stream))
        return self.gemm_plan(plan.value)

    @classmethod
    def gemm_plan(cls, p):
        """decode the plan word cdx_op_gemm reports"""
        return dict(kind=cls.GEMM_KINDS[(p >> 4) & 3] if p & 8 else 'ffma', width=(p >> 8) & 255, splits=(p >> 16) & 255,
                    amax_fused=bool(p & 1), stats_fused=bool(p & 2))

    def op_latent_chains(self, stage, chains, chw, n_src, K, rows, c=None, cnext=None, **fields):
        """One launch of the latent loops' production step kernels (cdx_op_latent_chains): stage 0 latent_chains_init, 1
        latent_chains_step.  chains: [(row, row2, scale)] for the n_src source chains then the n_src*K target chains; rows: the row
        count of xin / eout; c, cnext: DdimCoef; the other cdx_latent_chains_desc fields are keyword arguments, buffers as contiguous
        float32 tensors on this engine's device (a view at an offset keeps its address).  Each buffer must hold every element the
        launch may touch; outputs land in the caller's tensors.
        Semantic guidance: sg_rows [(row) * n_src*K*m] (host ints, the concept rows of target chain t at t*m + k) sets sg_m = m;
        stage 2 is its threshold stage (writes sg_thr), stage 1 then runs the step with the concept terms; sg_scale and sg_lambda are
        lists of m floats, sg_active / sg_apply / sg_mu / sg_beta / sg_beta1 scalars, sg_thr and sg_nu tensors.  LEDITS++'s masks:
        sg_mask 1 or 2 with sg_map [n_src*K*m, sg_gh*sg_gw] (a tensor), sg_gh, sg_gw and the latent width w; sg_thr then holds 2
        thresholds per concept row.  Edit-friendly inversion: solver 1 or 2, next 3 with the draw scalars qa / q1, and under solver 2
        dc (a DpmCoef) with the history buffers d_src [n_src*chw] and d_tgt [n_src*K*chw] (tensors)."""
        sg_rows = fields.pop('sg_rows', None)
        m = len(sg_rows) // max(n_src * K, 1) if sg_rows else 0
        hw = fields.get('hw', 0)
        need = dict(x0=n_src * chw, noise0=n_src * chw, xt=n_src * chw, xn=n_src * chw, noise_next=n_src * chw, xn2=n_src * chw,
                    eout=rows * chw, xin=rows * chw, yt=n_src * K * chw, y_out=n_src * K * chw,
                    z_out=(n_src - 1) * fields.get('z_stride', 0) + chw, eps_in=(n_src - 1) * fields.get('eps_stride', 0) + chw,
                    mask=n_src * hw, sg_thr=n_src * K * m * ((chw // hw if hw else 0) if not fields.get('sg_mask') else 2),
                    sg_nu=n_src * K * chw, sg_map=n_src * K * m * fields.get('sg_gh', 0) * fields.get('sg_gw', 0), d_src=n_src * chw,
                    d_tgt=n_src * K * chw)
        assert len(chains) == n_src * (1 + K), f'op_latent_chains: {len(chains)} chains for n_src={n_src}, K={K}'
        table = (_cabi.LatentChain * len(chains))(*[_cabi.LatentChain(int(r), int(r2), float(s)) for r, r2, s in chains])
        d = _cabi.LatentChainsSamplerDesc(chw=chw, n_src=n_src, K=K, rows=rows, chains=table)
        if sg_rows:
            assert len(sg_rows) == n_src * K * m, f'op_latent_chains: {len(sg_rows)} concept rows for {n_src * K} target chains'
            sg_table = (C.c_int * len(sg_rows))(*[int(r) for r in sg_rows])
            d.sg_m, d.sg_rows = m, sg_table
        for name in ('sg_scale', 'sg_lambda'):
            if name in fields:
                vals = [float(v) for v in fields.pop(name)]
                setattr(d, name, (C.c_float * 8)(*(vals + [0.0] * (8 - len(vals)))))
        if c is not None:
            d.c = c
        if cnext is not None:
            d.cnext = cnext
        for name, v in fields.items():
            if name in need:
                if v is None:
                    continue
                assert torch.is_tensor(v) and v.dtype == torch.float32 and v.device == self.device and v.is_contiguous(), \
                    f'op_latent_chains: {name} must be a contiguous float32 tensor on {self.device}'
                assert v.numel() >= need[name], f'op_latent_chains: {name} holds {v.numel()} elements, the launch may touch {need[name]}'
                setattr(d, name, v.data_ptr())
            else:
                assert hasattr(d, name), f'op_latent_chains: no field {name}'
                setattr(d, name, v)
        check(lib.cdx_op_latent_chains(self.h, C.byref(d), int(stage), self.stream))

    def op_pixel_lockstep(self, x0, xs, ys, et_src, et_tgt, noise, coef):
        """One step of the two-model pixel loop (cdx_op_pixel_lockstep): xs, ys [B,C,R,R] (source and target x_t, contiguous
        float32 on the device) are advanced in place; et_src / et_tgt [B,Cnet,R,R] U-Net outputs whose first C channels are used."""
        x0, noise, et_src, et_tgt = (_f32c(t, self.device) for t in (x0, noise, et_src, et_tgt))
        for t in (xs, ys):
            assert t.dtype == torch.float32 and t.device == self.device and t.is_contiguous() and t.shape == x0.shape
        B = x0.shape[0]
        assert noise.shape == x0.shape and et_src.shape[0] == et_tgt.shape[0] == B
        chw, ns, nt = x0[0].numel(), et_src[0].numel(), et_tgt[0].numel()
        check(lib.cdx_op_pixel_lockstep(self.h, _ptr(x0), _ptr(xs), _ptr(ys), _ptr(et_src), _ptr(et_tgt), _ptr(noise), C.byref(coef), B, chw,
                                        ns, nt, self.stream))

    def op_attention(self, q, k, v, heads, scale, qk_rows=None, accumulate_rows=None, out=None, kv_rows=None):
        """softmax(q k^T * scale) v per head.  qk_rows: optional [B] ints, image b attends with image qk_rows[b]'s q and k and its
        own v (cdx_op_attention_rows; fused kernel only).  kv_rows: optional [B] ints, image b attends with its own q over image
        kv_rows[b]'s k and v (cdx_op_attention_kv_rows; fused kernel only; not with qk_rows).  accumulate_rows: optional list of
        images r, out[r] += the attention of image r, the other images of `out` (a [B, Nq, C] float32 tensor on the device, updated
        in place and returned) untouched (cdx_op_attention_accum; fused kernel only)."""
        q, k, v = (_f32c(t, self.device) for t in (q, k, v))
        B, Nq, Cc = q.shape
        Nk = k.shape[1]
        assert qk_rows is None or kv_rows is None, 'qk_rows and kv_rows are exclusive: one row table per launch'
        if accumulate_rows is not None:
            assert qk_rows is None and kv_rows is None, 'row tables and accumulate_rows are separate launches'
            assert out is not None and out.shape == q.shape and out.dtype == torch.float32 and out.is_contiguous() and out.device == q.device, \
                'accumulate_rows: out must be a contiguous float32 tensor shaped like q on the engine device'
            rows = [int(r) for r in accumulate_rows]
            check(lib.cdx_op_attention_accum(self.h, _ptr(q), _ptr(k), _ptr(v), _ptr(out), B, Nq, Nk, heads, Cc // heads, scale,
                                             (C.c_int * max(len(rows), 1))(*rows), len(rows), self.stream))
            return out
        assert out is None, 'out is the accumulation target of accumulate_rows'
        out = torch.empty_like(q)
        table = qk_rows if qk_rows is not None else kv_rows
        if table is None:
            check(lib.cdx_op_attention(self.h, _ptr(q), _ptr(k), _ptr(v), _ptr(out), B, Nq, Nk, heads, Cc // heads, scale, self.stream))
        else:
            rows = [int(r) for r in table]
            assert len(rows) == B, f'{"qk" if qk_rows is not None else "kv"}_rows: {len(rows)} entries for {B} images'
            fn = lib.cdx_op_attention_rows if qk_rows is not None else lib.cdx_op_attention_kv_rows
            check(fn(self.h, _ptr(q), _ptr(k), _ptr(v), _ptr(out), B, Nq, Nk, heads, Cc // heads, scale, (C.c_int * B)(*rows), self.stream))
        return out

    ATTN_ROUTES = ('generic', 'unfused_tc', 'fused_h16', 'fused_tf32', 'fused_one')

    def op_attention_net(self, kind, out, B, N, heads, d, scale, qkv=None, q=None, kv=None, k=None, v=None, L=0, ctx_lp=0, causal=False,
                         qk_rows=None, kv_rows=None, acc_rows=None, slot=0.0, q_slot=0.0, probe_rows=None, probe_spans=None, probe_map=None,
                         probe_weights=None):
        """One attention with its operands prepared as the network executors prepare them (cdx_op_attention_net in include/cdx.h,
        whose descriptor fields are the arguments).  kind: 'self' (qkv [B*N, 3C], one range slot), 'cross' (q [B*N, C], kv
        [B*ctx_lp, 2C] the padded context's K | V) or 'generic' (q, k, v; optional causal mask).  Every buffer is a float32 tensor on
        this engine's device passed as it is; out [B*N, C] (a view inside a larger buffer is fine) is written, or added to for the
        images of acc_rows.  slot / q_slot > 0 replace the measured range slots.  Returns the plan: dict(route, qrows, rag, ksplit,
        ring, Nks, Nvs).  probe_rows / probe_spans (host int lists) with probe_map [n_probe, N] (kind 'cross'): LEDITS++'s probe on
        the operands the route multiplied, map[i] <- sum over heads of the softmax over tokens 1..probe_spans[i] of image probe_rows[i].
        probe_weights (host float tensor [n_probe, L], instead of probe_spans): LocalBlend's weighted probe (cdx_op_attention_net_weighted),
        map[i] <- sum over heads of sum over j of probe_weights[i, j] * softmax_j of image probe_rows[i]."""
        kinds = ('self', 'cross', 'generic')
        assert kind in kinds, kind
        for name, t in (('out', out), ('qkv', qkv), ('q', q), ('kv', kv), ('k', k), ('v', v), ('probe_map', probe_map)):
            assert t is None or (torch.is_tensor(t) and t.dtype == torch.float32 and t.device == self.device), \
                f'op_attention_net: {name} must be a float32 tensor on {self.device}'
        rows = lambda r: None if r is None else (C.c_int * max(len(r), 1))(*[int(x) for x in r])
        ptr = lambda t: t.data_ptr() if t is not None else None
        desc = _cabi.AttentionNetDesc(kind=kinds.index(kind), causal=int(bool(causal)), qkv=ptr(qkv), q=ptr(q), kv=ptr(kv), k=ptr(k), v=ptr(v),
                                      B=B, N=N, L=L, ctx_lp=ctx_lp, heads=heads, d=d, scale=scale, qk_rows=rows(qk_rows), kv_rows=rows(kv_rows),
                                      acc_rows=rows(acc_rows), n_acc=len(acc_rows) if acc_rows is not None else 0, slot=slot, q_slot=q_slot,
                                      out=ptr(out))
        wts = None
        if probe_rows is not None:
            assert (probe_spans is None) != (probe_weights is None) and probe_map is not None
            assert probe_spans is None or len(probe_spans) == len(probe_rows)
            assert probe_map.is_contiguous() and probe_map.numel() >= len(probe_rows) * N, 'op_attention_net: probe_map [n_probe, N]'
            desc.probe_rows, desc.probe_spans, desc.n_probe = rows(probe_rows), rows(probe_spans), len(probe_rows)
            desc.probe_map = ptr(probe_map)
            if probe_weights is not None:
                w = torch.as_tensor(probe_weights, dtype=torch.float32).cpu().contiguous()
                assert tuple(w.shape) == (len(probe_rows), L), f'op_attention_net: probe_weights [{len(probe_rows)}, {L}]'
                wts = (C.c_float * w.numel()).from_buffer_copy(w.numpy().tobytes())
        plan = (C.c_int * 7)()
        if wts is not None:
            check(lib.cdx_op_attention_net_weighted(self.h, C.byref(desc), wts, plan, self.stream))
        else:
            check(lib.cdx_op_attention_net(self.h, C.byref(desc), plan, self.stream))
        return dict(zip(('route', 'qrows', 'rag', 'ksplit', 'ring', 'Nks', 'Nvs'), [self.ATTN_ROUTES[plan[0]]] + list(plan[1:])))

    def op_nchw_to_nhwc(self, x):
        x = _f32c(x, self.device)
        B, Cc, H, W = x.shape
        y = self.empty(B, H, W, Cc)
        check(lib.cdx_op_nchw_to_nhwc(self.h, _ptr(x), _ptr(y), B, Cc, H * W, self.stream))
        return y

    def op_nhwc_to_nchw(self, x):
        x = _f32c(x, self.device)
        B, H, W, Cc = x.shape
        y = self.empty(B, Cc, H, W)
        check(lib.cdx_op_nhwc_to_nchw(self.h, _ptr(x), _ptr(y), B, Cc, H * W, self.stream))
        return y


class EnsembleSelection:
    """State of Engine.ensemble_select.  ``add(scores, cand_idx, sample_idx, images)`` folds in one chunk: scores [n], cand_idx [n]
    (column of the score matrix, the reference's candidate order), sample_idx [n], images [n,3,H,W].  After every candidate has
    arrived, best_idx equals torch.argmax(scores, dim=1) and best_img[b] is candidate best_idx[b]'s image of sample b, whatever the
    arrival order.  Columns not yet supplied hold NaN."""

    def __init__(self, engine, B, n_candidates, H, W):
        self.engine, self.B, self.n_candidates, self.H, self.W = engine, B, n_candidates, H, W
        dev = engine.device
        self.best_img = engine.empty(B, 3, H, W)
        self.best_idx = torch.full((B,), -1, dtype=torch.int64, device=dev)
        self.best_score = engine.empty(B)
        self.scores = torch.full((B, n_candidates), float('nan'), dtype=torch.float32, device=dev)

    def add(self, scores, cand_idx, sample_idx, images):
        e = self.engine
        scores, images = _f32c(scores, e.device), _f32c(images, e.device)
        cand = torch.as_tensor(cand_idx).to(device=e.device, dtype=torch.int64).contiguous()
        samp = torch.as_tensor(sample_idx).to(device=e.device, dtype=torch.int32).contiguous()
        n = scores.numel()
        assert cand.shape == samp.shape == (n,) and images.shape == (n, 3, self.H, self.W), \
            f'chunk shapes {tuple(scores.shape)} {tuple(cand.shape)} {tuple(samp.shape)} {tuple(images.shape)}'
        check(lib.cdx_ensemble_select(e.h, n, _ptr(scores), _ptr(cand), _ptr(samp), _ptr(images), _ptr(self.best_score), _ptr(self.best_idx),
                                      _ptr(self.best_img), _ptr(self.scores), self.B, self.n_candidates, self.H, self.W, e.stream))


def _int_arr8(vals):
    a = (C.c_int * 8)()
    for i, v in enumerate(vals):
        a[i] = int(v)
    return a


class Net:
    """A network living in the engine: parameter inventory + packed weight blob."""

    def __init__(self, engine, handle):
        self.engine = engine
        self.h = handle
        self.finalized = False

    def close(self):
        if getattr(self, 'h', None):
            lib.cdx_net_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def inventory(self):
        """[(name, shape)] in the reference checkpoint's key names."""
        return self._engine_inventory()

    def _engine_inventory(self):
        """[(name, shape)] as the engine stores the parameters (cdx_net_param_shape)."""
        out = []
        dims = (C.c_int64 * 4)()
        for i in range(lib.cdx_net_num_params(self.h)):
            name = lib.cdx_net_param_name(self.h, i).decode()
            rank = lib.cdx_net_param_shape(self.h, i, dims)
            out.append((name, tuple(int(dims[k]) for k in range(rank))))
        return out

    def load_state_dict(self, sd, prefix='', strict=True):
        """Load a reference-style state_dict (keys optionally under ``prefix``, e.g. 'model.diffusion_model.')."""
        inv = self.inventory()
        names = {n for n, _ in inv}
        if strict:
            extra = [k[len(prefix):] for k in sd if k.startswith(prefix) and k[len(prefix):] not in names]
            assert not extra, f'unexpected keys in state_dict: {extra[:5]}...'
        for (name, shape), (_, eshape) in zip(inv, self._engine_inventory()):
            key = prefix + name
            assert key in sd, f'missing key in state_dict: {key}'
            t = sd[key]
            assert tuple(t.shape) == shape, f'{key}: shape {tuple(t.shape)} != {shape}'
            t = t.detach().to(torch.float32).reshape(eshape).contiguous()        # a checkpoint's own layout viewed as the engine's
            dims = (C.c_int64 * 4)(*(list(eshape) + [1] * (4 - len(eshape))))
            check(lib.cdx_net_load_param(self.h, name.encode(), _ptr(t), 1 if t.is_cuda else 0, dims, len(eshape)))
        self.finalize()
        return self

    def finalize(self):
        check(lib.cdx_net_finalize(self.h))
        self.finalized = True

    def weight_blob(self):
        """(device pointer, bytes) of the packed weights -- the buffer rank 0 broadcasts over NCCL."""
        p, n = C.c_void_p(), C.c_size_t()
        check(lib.cdx_net_weight_blob(self.h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def blob_tensor(self):
        """A torch view of the packed weight blob (no copy), for torch.distributed.broadcast."""
        p, n = self.weight_blob()

        class _Blob:
            __cuda_array_interface__ = {'shape': (n // 4,), 'typestr': '<f4', 'data': (p, False), 'version': 2}
        return torch.as_tensor(_Blob(), device=self.engine.device)

    def adopt_blob(self):
        check(lib.cdx_net_adopt_blob(self.h))
        self.finalized = True


class UNet(Net):
    """SD/LDM (kind='openai') or improved-DDPM (kind='iddpm') U-Net; eps-prediction unless set_prediction('v') (SD 2.x "-v")."""

    def __init__(self, engine, cfg, kind='openai'):
        self.cfg = dict(cfg)
        self.kind = kind
        self.prediction = 'eps'
        c = UnetConfig()
        c.kind = {'openai': _cabi.CDX_UNET_OPENAI, 'iddpm': _cabi.CDX_UNET_IDDPM, 'ddpm': _cabi.CDX_UNET_DDPM}[kind]
        c.in_channels, c.out_channels = cfg['in_channels'], cfg['out_channels']
        c.model_channels, c.num_res_blocks = cfg['model_channels'], cfg['num_res_blocks']
        c.n_mult = len(cfg['channel_mult'])
        c.channel_mult = _int_arr8(cfg['channel_mult'])
        c.n_attn = len(cfg['attention_resolutions'])
        c.attention_ds = _int_arr8(cfg['attention_resolutions'])
        c.num_heads = cfg.get('num_heads', 0)
        c.num_head_channels = cfg.get('num_head_channels', 0)
        c.context_dim = cfg.get('context_dim', 0)
        h = C.c_void_p()
        check(lib.cdx_unet_create(engine.h if engine is not None else None, C.byref(c), C.byref(h)))
        super().__init__(engine, h)
        if engine is not None:
            # sinusoid frequencies with the reference expression (util.py:161-163 / nn.py:112-114), evaluated by torch on
            # the host so that they are bit-identical to what the reference / oracle computes on this machine
            half = cfg['model_channels'] // 2
            if kind == 'ddpm':          # get_timestep_embedding, ddpm/diffusion.py:15-18: log(10000) / (half - 1)
                freqs = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000) / (half - 1)))
            else:
                freqs = torch.exp(-math.log(10000) * torch.arange(start=0, end=half, dtype=torch.float32) / half)
            arr = (C.c_float * half)(*freqs.tolist())
            check(lib.cdx_unet_set_time_freqs(self.h, arr, half))

    def inventory(self):
        """As Net.inventory, except that an SD 2.x config (``use_linear_in_transformer``) lists the spatial transformers'
        proj_in / proj_out weights as the checkpoint stores them, [C, C] Linear weights; the engine holds them as the equivalent
        [C, C, 1, 1] 1x1 convolutions and load_state_dict views one as the other."""
        inv = self._engine_inventory()
        if self.kind == 'openai' and self.cfg.get('use_linear_in_transformer') and self.cfg.get('context_dim'):
            inv = [(n, s[:2] if n.endswith(('.proj_in.weight', '.proj_out.weight')) and len(s) == 4 else s) for n, s in inv]
        return inv

    def set_prediction(self, prediction, alphas_cumprod_f64=None):
        """What the U-Net predicts: 'eps' (default) or 'v' (SD 2.x parameterization: "v").  Under 'v' the latent loop drivers
        convert the guidance-combined output at timestep t as e_t = sqrt(abar_t) v + sqrt(1 - abar_t) x_t and
        pred_x0 = sqrt(abar_t) x_t - sqrt(1 - abar_t) v inside their fused step kernels.  alphas_cumprod_f64: the float64
        abar table (register_schedule's, before the fp32 cast); default the LDM linear schedule."""
        from .schedule import v_tables
        if prediction not in ('eps', 'v'):
            raise ValueError(f"prediction must be 'eps' or 'v', got {prediction!r}")
        if prediction == 'eps':
            check(lib.cdx_unet_set_prediction(self.h, _cabi.CDX_PRED_EPS, None, None, 0))
        else:
            sa, s1 = v_tables(alphas_cumprod_f64)
            T = len(sa)
            check(lib.cdx_unet_set_prediction(self.h, _cabi.CDX_PRED_V, (C.c_float * T)(*sa.tolist()), (C.c_float * T)(*s1.tolist()), T))
        self.prediction = prediction
        return self

    def forward(self, x, timesteps, context=None):
        e = self.engine
        x = _f32c(x, e.device)
        B, _, H, W = x.shape
        t = timesteps.to(device=e.device, dtype=torch.float32).contiguous()
        assert t.shape == (B,)
        L = 0
        if context is not None:
            context = _f32c(context, e.device)
            assert context.shape[0] == B and context.shape[2] == self.cfg['context_dim']
            L = context.shape[1]
        out = e.empty(B, self.cfg['out_channels'], H, W)
        check(lib.cdx_unet_forward(self.h, _ptr(x), _ptr(t), _ptr(context), L, _ptr(out), B, H, W, e.stream))
        return out

    __call__ = forward

    # ---- loop drivers (whole chains enqueued inside libcdx)
    def latent_encode(self, x0, c, uc, scale, sched, n_rec, noise):
        """-> z [B, n_rec+1, C, h, w]; noise [n_rec+1, B, C, h, w] in the reference's draw order."""
        e = self.engine
        x0, noise = _f32c(x0, e.device), _f32c(noise, e.device)
        c = _f32c(c, e.device) if c is not None else None            # None: unconditional model (no context)
        uc = _f32c(uc, e.device) if uc is not None else None
        B, Cc, h, w = x0.shape
        assert noise.shape == (n_rec + 1, B, Cc, h, w), f'noise shape {tuple(noise.shape)}'
        z = e.empty(B, n_rec + 1, Cc, h, w)
        check(lib.cdx_latent_encode(self.h, _ptr(x0), _ptr(c), _ptr(uc), c.shape[1] if c is not None else 0, float(scale), sched.coef_array(), sched.t_array(),
                                    sched.refine_steps, n_rec, _ptr(noise), sched.sqrt_a_T, sched.sqrt_1ma_T, _ptr(z), B, Cc, h, w,
                                    e.stream))
        return z

    def latent_decode(self, z, c, uc, scale, sched, extra_noise=None):
        """z [B, n_eps+1, C, h, w] -> x0 [B, C, h, w]."""
        e = self.engine
        z = _f32c(z, e.device)
        c = _f32c(c, e.device) if c is not None else None
        uc = _f32c(uc, e.device) if uc is not None else None
        extra_noise = _f32c(extra_noise, e.device) if extra_noise is not None else None
        B, n1, Cc, h, w = z.shape
        out = e.empty(B, Cc, h, w)
        check(lib.cdx_latent_decode(self.h, _ptr(z), n1 - 1, _ptr(c), _ptr(uc), c.shape[1] if c is not None else 0, float(scale), sched.coef_array(),
                                    sched.t_array(), sched.refine_steps, _ptr(extra_noise), _ptr(out), B, Cc, h, w, e.stream))
        return out

    def latent_refine(self, x0, c, uc, scale, S, refine_steps, noise, alphas_cumprod=None):
        """DDIMSampler.refine / _refine (ddim.py:114-168, 339-393) as the latentdiff wrappers call it (eta = 1): re-noise x0 to the
        level of step `refine_steps - 1` of the S-step eta-1 schedule and run the last `refine_steps` stochastic DDIM steps with
        fresh noise.  noise [refine_steps + 1, B, C, h, w]: the x_t draw (ddim.py:349), then one per step (p_sample_ddim)."""
        from .schedule import DDIMSchedule
        assert 0 < refine_steps < S                                   # ddim.py:364
        sched = DDIMSchedule(S, 1.0, S - refine_steps, alphas_cumprod)
        noise = _f32c(noise, self.engine.device)
        assert noise.shape[0] == refine_steps + 1
        xt = self.engine.q_sample(x0, noise[0], sched.sqrt_a_T, sched.sqrt_1ma_T)
        return self.latent_decode(xt.unsqueeze(1).contiguous(), c, uc, scale, sched, extra_noise=noise[1:].contiguous())

    # ---- ensemble members batched along B (per-sample guidance scales; cdx_latent_loop_ens)
    def latent_encode_ens(self, x0, c, uc, scales, sched, n_rec, noise):
        """latent_encode with one guidance scale per sample: scales [B] -> z [B, n_rec+1, C, h, w]."""
        e = self.engine
        x0, c, uc, noise = (_f32c(t, e.device) for t in (x0, c, uc, noise))
        sc = _f32c(torch.as_tensor(scales, dtype=torch.float32), e.device)
        B, Cc, h, w = x0.shape
        assert noise.shape == (n_rec + 1, B, Cc, h, w) and sc.shape == (B,)
        z = e.empty(B, n_rec + 1, Cc, h, w)
        check(lib.cdx_latent_loop_ens(self.h, 1, _ptr(x0), _ptr(c), None, _ptr(uc), c.shape[1], _ptr(sc), None, sched.coef_array(), sched.t_array(),
                                      sched.refine_steps, n_rec, _ptr(noise), sched.sqrt_a_T, sched.sqrt_1ma_T, None, 0, None, _ptr(z), None,
                                      B, Cc, h, w, e.stream))
        return z

    def latent_decode_ens(self, z, c, uc, scales, sched, extra_noise=None):
        """latent_decode with one guidance scale per sample: z [B, n_eps+1, C, h, w], scales [B] -> x0 [B, C, h, w]."""
        e = self.engine
        z, c, uc = (_f32c(t, e.device) for t in (z, c, uc))
        sc = _f32c(torch.as_tensor(scales, dtype=torch.float32), e.device)
        extra_noise = _f32c(extra_noise, e.device) if extra_noise is not None else None
        B, n1, Cc, h, w = z.shape
        assert sc.shape == (B,)
        out = e.empty(B, Cc, h, w)
        check(lib.cdx_latent_loop_ens(self.h, 2, None, None, _ptr(c), _ptr(uc), c.shape[1], None, _ptr(sc), sched.coef_array(), sched.t_array(),
                                      sched.refine_steps, 0, None, 0.0, 0.0, _ptr(z), n1 - 1, _ptr(extra_noise), None, _ptr(out),
                                      B, Cc, h, w, e.stream))
        return out

    def cycle_lockstep(self, x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise, return_z=False, mask=None, attn_control=None,
                       semantic=None, c_edit=None, local_blend=None):
        """Both chains in one loop (one U-Net call + one fused elementwise kernel per step, no z buffer unless asked for):
        x0 [B,C,h,w] -> translated latent [B,C,h,w] (and z [B, n+1, C,h,w] when return_z).  noise as for latent_encode with
        n_rec == sched.refine_steps.  mask [B,1,h,w] in [0,1] (1 = may change): masked editing (cdx_cycle_lockstep_masked), the
        target chain is blended with the source chain's x_{t-1} after every step; ones give the unmasked result, zeros give x0.
        attn_control: an attn_control.AttentionControl, Prompt-to-Prompt's "replace" edit on the target chain's cond row
        (cdx_cycle_lockstep_ctl), or its "refine" edit when the control has an own_weight (cdx_cycle_lockstep_refine); or an
        attn_control.MutualSelfControl, MasaCtrl's mutual self-attention on the target chain's rows (cdx_cycle_lockstep_mutual); or
        an attn_control.PnPControl, Plug-and-Play's feature and self-attention injection on the target chain's rows
        (cdx_cycle_lockstep_pnp).  Each composes with mask.
        semantic: a semantic.SemanticGuidance of m concepts, with c_edit [B, m, L, D] (or [m, L, D], every sample's): SEGA's
        concept terms on the target chain (cdx_cycle_lockstep_semantic), or with use_cross_attn_mask / use_intersect_mask LEDITS++'s
        implicit masks (cdx_cycle_lockstep_semantic_attn); it needs uc, composes with mask, and an attn_control with it raises
        ValueError.
        sched: a schedule.DDIMSchedule runs the DPM-Encoder chain above; a schedule.EditFriendlySchedule runs LEDITS++'s edit-friendly
        inversion instead (independent draws of the source's x, stepped by the eta = 1 DDIM step or the SDE-DPM-Solver++ step), with
        every control above, through cdx_cycle_lockstep_sampler.
        local_blend: an attn_control.LocalBlend, Prompt-to-Prompt's LocalBlend (cdx_cycle_lockstep_blend): from step
        int(start_blend * n) on the target chain is kept to where the blend words' cross-attention points, under either schedule.  It
        composes with mask and with an AttentionControl (replace, reweight, refine) or none; with semantic, MutualSelfControl or
        PnPControl it raises ValueError."""
        e = self.engine
        x0, c_src, c_tgt, noise = (_f32c(t, e.device) for t in (x0, c_src, c_tgt, noise))
        uc = _f32c(uc, e.device) if uc is not None else None
        B, Cc, h, w = x0.shape
        n = sched.refine_steps
        assert noise.shape == (n + 1, B, Cc, h, w), f'noise shape {tuple(noise.shape)}'
        assert c_src.shape == c_tgt.shape
        mask = check_mask(mask, (B, 1, h, w), e.device) if mask is not None else None
        if local_blend is not None:
            return self._cycle_blend(x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise, return_z, mask, attn_control, semantic,
                                     local_blend)
        if isinstance(sched, EditFriendlySchedule):
            return self._cycle_sampler(x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise, return_z, mask, attn_control, semantic,
                                       c_edit)
        if semantic is not None:
            c_edit = self._semantic_contexts(semantic, c_edit, attn_control, B, c_src.shape[1:])
            sg = semantic.c_struct(n)
            out = e.empty(B, Cc, h, w)
            z = e.empty(B, n + 1, Cc, h, w) if return_z else None
            args = (self.h, _ptr(x0), _ptr(c_src), _ptr(c_tgt), _ptr(uc), c_src.shape[1], float(src_scale), float(tgt_scale),
                    sched.coef_array(), sched.t_array(), n, _ptr(noise), sched.sqrt_a_T, sched.sqrt_1ma_T, _ptr(out), _ptr(z), B, Cc, h, w,
                    e.stream, _ptr(mask), _ptr(c_edit), C.byref(sg))
            if semantic.mask_mode:       # LEDITS++'s implicit masks
                am = semantic.attn_mask_struct(c_src.shape[1])
                check(lib.cdx_cycle_lockstep_semantic_attn(*args, C.byref(am)))
            else:
                check(lib.cdx_cycle_lockstep_semantic(*args))
            return (out, z) if return_z else out
        mutual, pnp = isinstance(attn_control, MutualSelfControl), isinstance(attn_control, PnPControl)
        ctl, _token_map, own = attn_control.c_struct(n, B, c_src.shape[1], e.device) if attn_control is not None and not (mutual or pnp) \
            else (None, None, None)
        out = e.empty(B, Cc, h, w)
        z = e.empty(B, n + 1, Cc, h, w) if return_z else None
        args = (self.h, _ptr(x0), _ptr(c_src), _ptr(c_tgt), _ptr(uc), c_src.shape[1], float(src_scale), float(tgt_scale), sched.coef_array(),
                sched.t_array(), n, _ptr(noise), sched.sqrt_a_T, sched.sqrt_1ma_T, _ptr(out), _ptr(z), B, Cc, h, w, e.stream, _ptr(mask))
        if mutual:
            check(lib.cdx_cycle_lockstep_mutual(*args, attn_control.start_step, attn_control.start_layer))
            return (out, z) if return_z else out
        if pnp:
            blocks = attn_control.feature_blocks
            check(lib.cdx_cycle_lockstep_pnp(*args, *attn_control.steps(n), attn_control.attention_start_layer,
                                             (C.c_int * max(len(blocks), 1))(*blocks), len(blocks)))
            return (out, z) if return_z else out
        args += (C.byref(ctl) if ctl is not None else None,)
        if own is None:
            check(lib.cdx_cycle_lockstep_ctl(*args))
        else:
            check(lib.cdx_cycle_lockstep_refine(*args, _ptr(own)))
        return (out, z) if return_z else out

    def _semantic_contexts(self, semantic, c_edit, attn_control, B, ctx_shape):
        if attn_control is not None:
            raise ValueError('semantic guidance does not combine with attention control in one loop')
        if not isinstance(semantic, SemanticGuidance):
            raise ValueError(f'semantic: expected a semantic.SemanticGuidance, got {type(semantic)}')
        if c_edit is None:
            raise ValueError('semantic guidance needs the concept contexts c_edit [B, m, L, D]')
        c_edit = _f32c(c_edit, self.engine.device)
        if c_edit.dim() == 3:
            c_edit = c_edit.unsqueeze(0).expand(B, -1, -1, -1).contiguous()
        if tuple(c_edit.shape) != (B, semantic.m) + tuple(ctx_shape):
            raise ValueError(f'c_edit: shape {tuple(c_edit.shape)}, expected {(B, semantic.m) + tuple(ctx_shape)}')
        return c_edit

    def _cycle_sampler(self, x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise, return_z, mask, attn_control, semantic, c_edit):
        """cycle_lockstep under an EditFriendlySchedule: every control through the one entry point cdx_cycle_lockstep_sampler"""
        e = self.engine
        B, Cc, h, w = x0.shape
        n, L = sched.refine_steps, c_src.shape[1]
        sp, _keep = sched.sampler_struct()
        ctl = own = mutual = pnp = sg = am = None
        if semantic is not None:
            c_edit = self._semantic_contexts(semantic, c_edit, attn_control, B, c_src.shape[1:])
            sg = semantic.c_struct(n)
            am = semantic.attn_mask_struct(L) if semantic.mask_mode else None
        else:
            c_edit = None
        blocks = None
        if isinstance(attn_control, MutualSelfControl):
            mutual = _cabi.MutualControlC(attn_control.start_step, attn_control.start_layer)
        elif isinstance(attn_control, PnPControl):
            blocks = (C.c_int * max(len(attn_control.feature_blocks), 1))(*attn_control.feature_blocks)
            fs, ats = attn_control.steps(n)
            pnp = _cabi.PnpControlC(fs, ats, attn_control.attention_start_layer, C.cast(blocks, C.POINTER(C.c_int)),
                                    len(attn_control.feature_blocks))
        elif attn_control is not None:
            ctl, _token_map, own = attn_control.c_struct(n, B, L, e.device)
        out = e.empty(B, Cc, h, w)
        z = e.empty(B, n + 1, Cc, h, w) if return_z else None
        ref = lambda s: C.byref(s) if s is not None else None
        check(lib.cdx_cycle_lockstep_sampler(self.h, _ptr(x0), _ptr(c_src), _ptr(c_tgt), _ptr(uc), L, float(src_scale), float(tgt_scale),
                                             sched.coef_array(), sched.t_array(), n, _ptr(noise), sched.sqrt_a_T, sched.sqrt_1ma_T, _ptr(out),
                                             _ptr(z), B, Cc, h, w, e.stream, C.byref(sp), _ptr(mask), ref(ctl), _ptr(own), ref(mutual),
                                             ref(pnp), _ptr(c_edit), ref(sg), ref(am)))
        return (out, z) if return_z else out

    def _cycle_blend(self, x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise, return_z, mask, attn_control, semantic, local_blend):
        """cycle_lockstep under a LocalBlend: cdx_cycle_lockstep_blend, with the sampler of an EditFriendlySchedule or none"""
        if not isinstance(local_blend, LocalBlend):
            raise ValueError(f'local_blend: expected an attn_control.LocalBlend, got {type(local_blend)}')
        if semantic is not None or isinstance(attn_control, (MutualSelfControl, PnPControl)):
            raise ValueError('LocalBlend runs with Prompt-to-Prompt edits (replace, reweight, refine) or none, not with semantic guidance, '
                             'MasaCtrl or Plug-and-Play')
        e = self.engine
        B, Cc, h, w = x0.shape
        n, L = sched.refine_steps, c_src.shape[1]
        if h % 4 or w % 4:
            raise ValueError(f'LocalBlend: the latent sides must be multiples of 4, got {h}x{w}')
        sp, _keep = sched.sampler_struct() if isinstance(sched, EditFriendlySchedule) else (None, None)
        ctl = own = None
        if attn_control is not None:
            ctl, _token_map, own = attn_control.c_struct(n, B, L, e.device)
        lb, _vecs = local_blend.c_struct(n, B, L, e.device)
        out = e.empty(B, Cc, h, w)
        z = e.empty(B, n + 1, Cc, h, w) if return_z else None
        ref = lambda s: C.byref(s) if s is not None else None
        check(lib.cdx_cycle_lockstep_blend(self.h, _ptr(x0), _ptr(c_src), _ptr(c_tgt), _ptr(uc), L, float(src_scale), float(tgt_scale),
                                           sched.coef_array(), sched.t_array(), n, _ptr(noise), sched.sqrt_a_T, sched.sqrt_1ma_T, _ptr(out),
                                           _ptr(z), B, Cc, h, w, e.stream, ref(sp), _ptr(mask), ref(ctl), _ptr(own), None, None, None, None,
                                           None, C.byref(lb)))
        return (out, z) if return_z else out

    def cycle_fan(self, x0, c_src, c_tgt, uc, src_scales, tgt_scales, sched, noise, return_z=False, mask=None):
        """The ensemble search's lock-step loop (cdx_latent_cycle_fan): source chain j (x0[j], c_src[j] at src_scales[j]) drives K
        target chains (c_tgt[j] at tgt_scales[j][k]) with the noise it recovers; one U-Net call per step over only the rows the
        scales need.  x0 [n_src,C,h,w]; c_src, c_tgt, uc [n_src,L,D]; src_scales [n_src] and tgt_scales [n_src][K] host numbers;
        noise [n+1, n_src,C,h,w] as for latent_encode with n_rec == sched.refine_steps -> latents [n_src*K,C,h,w] (row j*K + k)
        and, when return_z, z [n_src, n+1, C,h,w].  mask [n_src,1,h,w]: source chain j's targets are masked by mask[j] as in
        cycle_lockstep."""
        e = self.engine
        x0, c_src, c_tgt, uc, noise = (_f32c(t, e.device) for t in (x0, c_src, c_tgt, uc, noise))
        n_src, Cc, h, w = x0.shape
        src = [float(s) for s in src_scales]
        tgt = [[float(s) for s in row] for row in tgt_scales]
        K = len(tgt[0]) if tgt else 0
        assert len(src) == len(tgt) == n_src and all(len(r) == K for r in tgt), 'src_scales [n_src], tgt_scales [n_src][K]'
        n = sched.refine_steps
        assert noise.shape == (n + 1, n_src, Cc, h, w), f'noise shape {tuple(noise.shape)}'
        assert c_src.shape == c_tgt.shape == uc.shape and c_src.shape[0] == n_src
        mask = check_mask(mask, (n_src, 1, h, w), e.device) if mask is not None else None
        out = e.empty(n_src * K, Cc, h, w)
        z = e.empty(n_src, n + 1, Cc, h, w) if return_z else None
        check(lib.cdx_latent_cycle_fan_masked(self.h, n_src, K, _ptr(x0), _ptr(c_src), _ptr(c_tgt), _ptr(uc), c_src.shape[1],
                                              (C.c_float * n_src)(*src), (C.c_float * (n_src * K))(*[s for r in tgt for s in r]),
                                              sched.coef_array(), sched.t_array(), n, _ptr(noise), sched.sqrt_a_T, sched.sqrt_1ma_T,
                                              _ptr(out), _ptr(z), Cc, h, w, e.stream, _ptr(mask)))
        return (out, z) if return_z else out

    def edit_map(self, x0, c_src, c_tgt, sched, noise, rows_per_call=None):
        """DiffEdit's mask statistics (cdx_edit_map): x0 [B,C,h,w], c_src / c_tgt [B,L,D], noise [B,n,C,h,w] -> acc [B,h,w], the sum
        over the n maps of sum_c |e_tgt - e_src| of x_t = q_sample(x0[b], noise[b,k]) at sched's first timestep (v nets: in eps
        units).  Engine.edit_mask turns it into the mask.  rows_per_call: U-Net rows per call, two per (map, image) pair; default
        min(48, max(12, 3B)) -- the lock-step cycle's own 3B rows from batch 4 up, at least 12, at most the 48 rows whose GroupNorm
        statistics fit the engine's pool at SD width.  The result does not depend on it."""
        e = self.engine
        x0, c_src, c_tgt, noise = (_f32c(t, e.device) for t in (x0, c_src, c_tgt, noise))
        B, Cc, h, w = x0.shape
        assert noise.dim() == 5 and noise.shape[0] == B and noise.shape[2:] == x0.shape[1:], f'noise shape {tuple(noise.shape)}'
        assert c_src.shape == c_tgt.shape and c_src.shape[0] == B
        rows = int(rows_per_call) if rows_per_call is not None else min(48, max(12, 3 * B))
        acc = e.empty(B, h, w)
        check(lib.cdx_edit_map(self.h, _ptr(x0), _ptr(c_src), _ptr(c_tgt), c_src.shape[1], sched.t_loop[0], sched.sqrt_a_T,
                               sched.sqrt_1ma_T, _ptr(noise), noise.shape[1], rows, _ptr(acc), B, Cc, h, w, e.stream))
        return acc

    def pixel_encode(self, x0, sched, noise):
        e = self.engine
        x0, noise = _f32c(x0, e.device), _f32c(noise, e.device)
        B, Cc, R, _ = x0.shape
        n_rec = sched.es_steps - 1
        assert noise.shape == (n_rec + 1, B, Cc, R, R)
        z = e.empty(B, n_rec + 1, Cc, R, R)
        t = (C.c_float * max(n_rec, 1))(*sched.t_loop[:n_rec])
        check(lib.cdx_pixel_encode(self.h, _ptr(x0), sched.coef_array(sched.coef[:n_rec]) if n_rec else None, t, n_rec, _ptr(noise),
                                   sched.sqrt_a_T, sched.sqrt_1ma_T, _ptr(z), B, Cc, R, e.stream))
        return z

    def pixel_cycle_lockstep(self, target, x0, sched, state, noise, i0, i1):
        """Steps [i0, i1) of the two-model pixel loop (cdx_pixel_cycle_lockstep): this net runs the source chain's DPM-Encoder,
        ``target`` (a UNet) the target chain's decode, both on ``sched``.  state [2, B, C, R, R] (source x_t, target x_t) is
        advanced in place; noise [i1 - i0, B, C, R, R], preceded by the x_T draw when i0 == 0 (which initialises state)."""
        e = self.engine
        x0, noise = _f32c(x0, e.device), _f32c(noise, e.device)
        B, Cc, R, _ = x0.shape
        n_rec = sched.es_steps - 1
        assert 0 <= i0 <= i1 <= n_rec, f'steps [{i0}, {i1}) of {n_rec}'
        assert state.shape == (2, B, Cc, R, R) and state.dtype == torch.float32 and state.is_contiguous() and state.device == e.device
        assert noise.shape == (i1 - i0 + (i0 == 0), B, Cc, R, R), f'noise shape {tuple(noise.shape)}'
        coef = sched.coef_array(sched.coef[:n_rec]) if n_rec else None
        t = (C.c_float * max(n_rec, 1))(*sched.t_loop[:n_rec])
        check(lib.cdx_pixel_cycle_lockstep(self.h, target.h, _ptr(x0), coef, t, i0, i1, _ptr(noise), sched.sqrt_a_T, sched.sqrt_1ma_T,
                                           _ptr(state), B, Cc, R, e.stream))

    def latent_cycle_pair(self, target, x0, sched, n_rec, noise, extra_noise=None):
        """latent_encode under this net followed by latent_decode under ``target`` (a UNet), both context-free at scale 1, in one
        lock-step loop (cdx_latent_cycle_pair): x0 [B,C,h,w] -> decoded latent [B,C,h,w].  noise as for latent_encode; extra_noise
        [refine_steps - n_rec, B,C,h,w] for the steps the target chain runs alone."""
        e = self.engine
        x0, noise = _f32c(x0, e.device), _f32c(noise, e.device)
        extra_noise = _f32c(extra_noise, e.device) if extra_noise is not None else None
        B, Cc, h, w = x0.shape
        assert noise.shape == (n_rec + 1, B, Cc, h, w), f'noise shape {tuple(noise.shape)}'
        out = e.empty(B, Cc, h, w)
        check(lib.cdx_latent_cycle_pair(self.h, target.h, _ptr(x0), sched.coef_array(), sched.t_array(), sched.refine_steps, n_rec, _ptr(noise),
                                        sched.sqrt_a_T, sched.sqrt_1ma_T, _ptr(extra_noise), _ptr(out), B, Cc, h, w, e.stream))
        return out

    def pixel_decode(self, z, sched, coefs=None, t_loop=None, last_noise=None):
        e = self.engine
        z = _f32c(z, e.device)
        last_noise = _f32c(last_noise, e.device) if last_noise is not None else None
        B, n1, Cc, R, _ = z.shape
        coefs = sched.coef if coefs is None else coefs
        t_loop = sched.t_loop if t_loop is None else t_loop
        out = e.empty(B, Cc, R, R)
        t = (C.c_float * len(t_loop))(*t_loop)
        check(lib.cdx_pixel_decode(self.h, _ptr(z), n1 - 1, sched.coef_array(coefs), t, len(coefs), _ptr(last_noise), _ptr(out), B, Cc,
                                   R, e.stream))
        return out


class VAE(Net):
    """KL-f8 autoencoder (AutoencoderKL)."""

    def __init__(self, engine, cfg):
        self.cfg = dict(cfg)
        c = VaeConfig()
        c.ch, c.n_mult = cfg['ch'], len(cfg['ch_mult'])
        c.ch_mult = _int_arr8(cfg['ch_mult'])
        c.num_res_blocks = cfg['num_res_blocks']
        c.in_channels, c.out_ch = cfg['in_channels'], cfg['out_ch']
        c.z_channels, c.embed_dim = cfg['z_channels'], cfg['embed_dim']
        c.vq, c.n_embed = int(bool(cfg.get('vq', False))), cfg.get('n_embed', 0)
        h = C.c_void_p()
        check(lib.cdx_vae_create(engine.h if engine is not None else None, C.byref(c), C.byref(h)))
        super().__init__(engine, h)
        self.down = 2 ** (len(cfg['ch_mult']) - 1)

    def encode_moments(self, img):
        """img [B,3,H,W] in [-1,1], H and W multiples of ``self.down`` -> moments [B, 2*embed_dim, H/down, W/down]."""
        e = self.engine
        img = _f32c(img, e.device)
        B, _, H, W = img.shape
        out = e.empty(B, (1 if self.cfg.get('vq') else 2) * self.cfg['embed_dim'], H // self.down, W // self.down)      # vq: h itself
        check(lib.cdx_vae_encode_hw(self.h, _ptr(img), _ptr(out), B, H, W, e.stream))
        return out

    def decode(self, z):
        """z [B,embed_dim,h,w] -> img [B, out_ch, h*down, w*down]."""
        e = self.engine
        z = _f32c(z, e.device)
        B, _, h, w = z.shape
        out = e.empty(B, self.cfg['out_ch'], h * self.down, w * self.down)
        check(lib.cdx_vae_decode_hw(self.h, _ptr(z), _ptr(out), B, h, w, e.stream))
        return out


class TextEncoder(Net):
    """Text conditioning towers: CLIP (HF CLIPTextModel layout -> last_hidden_state; FrozenCLIPEmbedder,
    ldm/modules/encoders/modules.py:140-158) or, with ``cfg['kind'] == 'xtransformer'``, the LDM BERTEmbedder's in-tree
    encoder (modules.py:79-98, x_transformer.py).  Tokenisation stays on the host (vocabulary files are not part of the engine)."""

    def __init__(self, engine, cfg):
        self.cfg = dict(cfg)
        c = TextConfig()
        c.vocab_size, c.width, c.layers = cfg['vocab_size'], cfg['width'], cfg['layers']
        c.heads, c.max_len, c.mlp_width = cfg['heads'], cfg['max_len'], cfg['mlp_width']
        c.kind = {'clip': 1, 'xtransformer': 2, 'clip_vision': 3, 'openclip': 4}[cfg.get('kind', 'clip')]
        c.dim_head = cfg.get('dim_head', cfg['width'] // cfg['heads'])
        c.proj_dim, c.patch, c.image_size = cfg.get('proj_dim', 0), cfg.get('patch', 0), cfg.get('image_size', 0)
        h = C.c_void_p()
        check(lib.cdx_text_create(engine.h if engine is not None else None, C.byref(c), C.byref(h)))
        super().__init__(engine, h)

    def load_state_dict(self, sd, prefix='', strict=True):
        # older transformers versions register `embeddings.position_ids` as a persistent buffer: not a parameter
        # (and x_transformer's TransformerWrapper carries an unused `to_logits` head)
        sd = {k: v for k, v in sd.items() if not k.endswith('embeddings.position_ids') and '.to_logits.' not in k}
        return super().load_state_dict(sd, prefix, strict)

    def forward(self, input_ids):
        """input_ids [B, L] integer tensor -> [B, L, width] fp32 on the engine's device."""
        e = self.engine
        ids = input_ids.to(device=e.device, dtype=torch.int32).contiguous()
        B, L = ids.shape
        assert L <= self.cfg['max_len'], f'{L} tokens > {self.cfg["max_len"]} positions'
        out = torch.empty(B, L, self.cfg['width'], device=e.device, dtype=torch.float32)
        check(lib.cdx_text_encode(self.h, _ptr(ids), B, L, _ptr(out), e.stream))
        return out

    __call__ = forward

    def features(self, input_ids):
        """CLIP.encode_text: ids [B, L] -> [B, proj_dim] (final-LN state at the EOT token @ text_projection); needs cfg['proj_dim']."""
        e = self.engine
        ids = input_ids.to(device=e.device, dtype=torch.int32).contiguous()
        B, L = ids.shape
        out = torch.empty(B, self.cfg['proj_dim'], device=e.device, dtype=torch.float32)
        check(lib.cdx_text_features(self.h, _ptr(ids), B, L, _ptr(out), e.stream))
        return out


class ClipVision(TextEncoder):
    """CLIP ViT image tower (cfg: width, layers, heads, mlp_width, patch, image_size, proj_dim): CLIP.encode_image."""

    def __init__(self, engine, cfg):
        cfg = dict(cfg, kind='clip_vision', vocab_size=cfg.get('vocab_size', 0), max_len=cfg.get('max_len', 0))
        super().__init__(engine, cfg)

    def forward(self, pixels):
        """pixels [B,3,S,S] (already preprocessed) -> image features [B, proj_dim]."""
        e = self.engine
        x = _f32c(pixels, e.device)
        B, _, S, S2 = x.shape
        assert S == S2 == self.cfg['image_size'], f'{tuple(x.shape)} vs image_size {self.cfg["image_size"]}'
        out = torch.empty(B, self.cfg['proj_dim'], device=e.device, dtype=torch.float32)
        check(lib.cdx_clip_image_features(self.h, _ptr(x), B, _ptr(out), e.stream))
        return out

    __call__ = forward
