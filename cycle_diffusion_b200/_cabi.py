"""ctypes binding of include/cdx.h (libcdx.so).  Thin by design: no arithmetic happens in Python.

There is NO CPU fallback: if the shared library is missing the import of this module raises, and
``Engine()`` raises when no CUDA device is usable (cdx_engine_create returns CDX_E_CUDA).
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'libcdx.so')

CDX_UNET_OPENAI = 1
CDX_UNET_IDDPM = 2
CDX_UNET_DDPM = 3
CDX_TEXT_OPENCLIP = 4
CDX_PRED_EPS = 0
CDX_PRED_V = 1


class UnetConfig(C.Structure):
    _fields_ = [('kind', C.c_int), ('in_channels', C.c_int), ('out_channels', C.c_int), ('model_channels', C.c_int),
                ('num_res_blocks', C.c_int), ('n_mult', C.c_int), ('channel_mult', C.c_int * 8), ('n_attn', C.c_int),
                ('attention_ds', C.c_int * 8), ('num_heads', C.c_int), ('num_head_channels', C.c_int),
                ('context_dim', C.c_int)]


class VaeConfig(C.Structure):
    _fields_ = [('ch', C.c_int), ('n_mult', C.c_int), ('ch_mult', C.c_int * 8), ('num_res_blocks', C.c_int),
                ('in_channels', C.c_int), ('out_ch', C.c_int), ('z_channels', C.c_int), ('embed_dim', C.c_int), ('vq', C.c_int), ('n_embed', C.c_int)]


class TextConfig(C.Structure):
    _fields_ = [('vocab_size', C.c_int), ('width', C.c_int), ('layers', C.c_int), ('heads', C.c_int), ('max_len', C.c_int),
                ('mlp_width', C.c_int), ('kind', C.c_int), ('dim_head', C.c_int), ('proj_dim', C.c_int), ('patch', C.c_int), ('image_size', C.c_int)]


class DdimCoef(C.Structure):
    _fields_ = [('sqrt_at', C.c_float), ('sqrt_1m_at', C.c_float), ('sqrt_1m_at_tab', C.c_float),
                ('sqrt_aprev', C.c_float), ('dir_coef', C.c_float), ('sigma', C.c_float)]


class PixelCoef(C.Structure):
    _fields_ = [('ddpm', C.c_int), ('sqrt_at', C.c_float), ('sqrt_1m_at', C.c_float), ('sqrt_at_next', C.c_float),
                ('c1', C.c_float), ('c2', C.c_float), ('w0', C.c_float), ('wt', C.c_float), ('post_std', C.c_float),
                ('weight', C.c_float), ('inv_sqrt_1m_bt', C.c_float), ('std_model', C.c_float), ('mask', C.c_float)]


_P = C.c_void_p          # device / opaque pointers


class AttnControl(C.Structure):
    _fields_ = [('cross_steps', C.c_int), ('self_steps', C.c_int), ('self_max_tokens', C.c_int), ('token_map', C.c_void_p)]


class GemmDesc(C.Structure):
    _fields_ = [('mode', C.c_int), ('M', C.c_int), ('N', C.c_int), ('K', C.c_int),
                ('A', _P), ('lda', C.c_int), ('C1', C.c_int), ('A2', _P), ('lda2', C.c_int), ('C2', C.c_int),
                ('Hin', C.c_int), ('Win', C.c_int), ('Hout', C.c_int), ('Wout', C.c_int), ('stride', C.c_int), ('pad', C.c_int),
                ('w', _P), ('ldb', C.c_int), ('b_kn', C.c_int), ('bias', _P),
                ('rowvec', _P), ('ld_rowvec', C.c_int), ('rows_per_batch', C.c_int), ('residual', _P), ('ldr', C.c_int),
                ('alpha', C.c_float), ('geglu', C.c_int), ('out_nchw', C.c_int), ('rows_per_img', C.c_int),
                ('C', _P), ('ldc', C.c_int), ('C_lo', _P), ('Ct_hi', _P), ('Ct_lo', _P), ('t_col0', C.c_int), ('ldt', C.c_int64),
                ('a_amax', _P), ('a2_amax', _P), ('c_amax', _P), ('c_stats', _P), ('w_range', C.c_float),
                ('batch', C.c_int), ('heads', C.c_int),
                ('sA_b', C.c_int64), ('sA_h', C.c_int64), ('sB_b', C.c_int64), ('sB_h', C.c_int64), ('sC_b', C.c_int64), ('sC_h', C.c_int64),
                ('up', C.c_int)]


class AttentionNetDesc(C.Structure):
    _fields_ = [('kind', C.c_int), ('causal', C.c_int), ('qkv', C.c_void_p), ('q', C.c_void_p), ('kv', C.c_void_p), ('k', C.c_void_p),
                ('v', C.c_void_p), ('B', C.c_int), ('N', C.c_int), ('L', C.c_int), ('ctx_lp', C.c_int), ('heads', C.c_int), ('d', C.c_int),
                ('scale', C.c_float), ('qk_rows', C.POINTER(C.c_int)), ('kv_rows', C.POINTER(C.c_int)), ('acc_rows', C.POINTER(C.c_int)),
                ('n_acc', C.c_int), ('slot', C.c_float), ('q_slot', C.c_float), ('out', C.c_void_p),
                ('probe_rows', C.POINTER(C.c_int)), ('probe_spans', C.POINTER(C.c_int)), ('n_probe', C.c_int), ('probe_map', C.c_void_p)]


class LatentChain(C.Structure):
    _fields_ = [('row', C.c_int), ('row2', C.c_int), ('scale', C.c_float)]


class LatentChainsDesc(C.Structure):
    _fields_ = [('chw', C.c_int), ('n_src', C.c_int), ('K', C.c_int), ('rows', C.c_int), ('chains', C.POINTER(LatentChain)), ('src', C.c_int),
                ('x0', _P), ('eout', _P), ('c', DdimCoef), ('noise0', _P), ('sa', C.c_float), ('s1', C.c_float), ('xt', _P), ('xn', _P),
                ('next', C.c_int), ('noise_next', _P), ('cnext', DdimCoef), ('xn2', _P), ('z_out', _P), ('z_stride', C.c_int64),
                ('eps_in', _P), ('eps_stride', C.c_int64), ('yt', _P), ('y_out', _P), ('xin', _P), ('pred', C.c_int), ('vsa', C.c_float),
                ('vs1', C.c_float), ('mask', _P), ('hw', C.c_int),
                ('sg_m', C.c_int), ('sg_rows', C.POINTER(C.c_int)), ('sg_thr', _P), ('sg_nu', _P), ('sg_scale', C.c_float * 8),
                ('sg_lambda', C.c_float * 8), ('sg_active', C.c_uint), ('sg_apply', C.c_int), ('sg_mu', C.c_float), ('sg_beta', C.c_float),
                ('sg_beta1', C.c_float)]


class LatentChainsMaskDesc(LatentChainsDesc):
    """The whole cdx_latent_chains_desc: LatentChainsDesc plus LEDITS++'s trailing mask fields (the C struct always has them, so every
    call passes this one)."""
    _fields_ = [('sg_map', _P), ('sg_mask', C.c_int), ('sg_gh', C.c_int), ('sg_gw', C.c_int), ('w', C.c_int)]


class DpmCoef(C.Structure):
    _fields_ = [('a', C.c_float), ('b', C.c_float), ('c', C.c_float), ('n', C.c_float), ('order', C.c_int)]


class LatentChainsSamplerDesc(LatentChainsMaskDesc):
    """The whole cdx_latent_chains_desc: LatentChainsMaskDesc plus the edit-friendly inversion's trailing fields."""
    _fields_ = [('solver', C.c_int), ('dc', DpmCoef), ('d_src', _P), ('d_tgt', _P), ('qa', C.c_float), ('q1', C.c_float)]


CDX_SAMPLER_DDIM_POSTERIOR = 0
CDX_SAMPLER_DDIM_DRAWS = 1
CDX_SAMPLER_DPMSOLVER_DRAWS = 2


class SamplerC(C.Structure):
    _fields_ = [('kind', C.c_int), ('dpm', C.POINTER(DpmCoef)), ('qa', C.POINTER(C.c_float)), ('q1', C.POINTER(C.c_float))]


class MutualControlC(C.Structure):
    _fields_ = [('start_step', C.c_int), ('start_layer', C.c_int)]


class PnpControlC(C.Structure):
    _fields_ = [('feature_steps', C.c_int), ('attention_steps', C.c_int), ('attention_start_layer', C.c_int),
                ('feature_blocks', C.POINTER(C.c_int)), ('n_feature_blocks', C.c_int)]


CDX_SEMANTIC_MAX = 8


class SemanticGuidanceC(C.Structure):
    _fields_ = [('m', C.c_int), ('scale', C.c_float * CDX_SEMANTIC_MAX), ('threshold', C.c_float * CDX_SEMANTIC_MAX),
                ('cooldown', C.c_int * CDX_SEMANTIC_MAX), ('warmup', C.c_int), ('momentum_scale', C.c_float), ('beta', C.c_float),
                ('beta1', C.c_float)]


class SemanticAttnMaskC(C.Structure):
    _fields_ = [('intersect', C.c_int), ('n_tokens', C.c_int * CDX_SEMANTIC_MAX)]


class LocalBlendC(C.Structure):
    _fields_ = [('alpha_src', C.c_void_p), ('alpha_tgt', C.c_void_p), ('sub_src', C.c_void_p), ('sub_tgt', C.c_void_p), ('start_step', C.c_int),
                ('th_blend', C.c_float), ('th_sub', C.c_float)]


_F = C.c_float
_I = C.c_int
_S = C.c_size_t

# name -> (restype, argtypes); every symbol include/cdx.h declares (tests/test_cabi.py checks the list against the header)
SIGNATURES = {
    'cdx_abi_version': (_I, []),
    'cdx_last_error': (C.c_char_p, []),
    'cdx_engine_create': (_I, [_I, C.POINTER(_P)]),
    'cdx_engine_destroy': (None, [_P]),
    'cdx_engine_workspace_bytes': (_S, [_P]),
    'cdx_engine_launch_count': (C.c_uint64, [_P]),
    'cdx_engine_set_mma_mode': (_I, [_P, _I]),
    'cdx_engine_set_persist': (_I, [_P, _I, _I]),
    'cdx_engine_profile': (_I, [_P, _I]),
    'cdx_engine_profile_read': (_I, [_P, _I, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_uint64)]),
    'cdx_unet_create': (_I, [_P, C.POINTER(UnetConfig), C.POINTER(_P)]),
    'cdx_vae_create': (_I, [_P, C.POINTER(VaeConfig), C.POINTER(_P)]),
    'cdx_text_create': (_I, [_P, C.POINTER(TextConfig), C.POINTER(_P)]),
    'cdx_net_destroy': (None, [_P]),
    'cdx_net_num_params': (_I, [_P]),
    'cdx_net_param_name': (C.c_char_p, [_P, _I]),
    'cdx_net_param_shape': (_I, [_P, _I, C.POINTER(C.c_int64)]),
    'cdx_net_load_param': (_I, [_P, C.c_char_p, _P, _I, C.POINTER(C.c_int64), _I]),
    'cdx_net_finalize': (_I, [_P]),
    'cdx_net_weight_blob': (_I, [_P, C.POINTER(_P), C.POINTER(_S)]),
    'cdx_net_adopt_blob': (_I, [_P]),
    'cdx_unet_set_time_freqs': (_I, [_P, C.POINTER(_F), _I]),
    'cdx_unet_set_prediction': (_I, [_P, _I, C.POINTER(_F), C.POINTER(_F), _I]),
    'cdx_unet_forward': (_I, [_P, _P, _P, _P, _I, _P, _I, _I, _I, _P]),
    'cdx_vae_encode': (_I, [_P, _P, _P, _I, _I, _P]),
    'cdx_text_encode': (_I, [_P, _P, _I, _I, _P, _P]),
    'cdx_vae_decode': (_I, [_P, _P, _P, _I, _I, _P]),
    'cdx_vae_encode_hw': (_I, [_P, _P, _P, _I, _I, _I, _P]),
    'cdx_vae_decode_hw': (_I, [_P, _P, _P, _I, _I, _I, _P]),
    'cdx_affine': (_I, [_P, _P, _F, _F, _P, _S, _P]),
    'cdx_shift_scale': (_I, [_P, _P, _F, _F, _P, _S, _P]),
    'cdx_q_sample': (_I, [_P, _P, _P, _F, _F, _P, _S, _P]),
    'cdx_vae_posterior': (_I, [_P, _P, _P, _F, _P, _I, _I, _I, _P]),
    'cdx_ddim_posterior_sample': (_I, [_P, _P, _P, _P, C.POINTER(DdimCoef), _P, _S, _P]),
    'cdx_ddim_compute_eps': (_I, [_P, _P, _P, _P, _P, _F, C.POINTER(DdimCoef), _P, _S, _P]),
    'cdx_ddim_step_with_eps': (_I, [_P, _P, _P, _P, _F, _P, C.POINTER(DdimCoef), _P, _S, _P]),
    'cdx_pixel_posterior_sample': (_I, [_P, _P, _P, _P, C.POINTER(PixelCoef), _P, _S, _P]),
    'cdx_pixel_compute_eps': (_I, [_P, _P, _P, _P, C.POINTER(PixelCoef), _P, _I, _I, _I, _P]),
    'cdx_pixel_step_with_eps': (_I, [_P, _P, _P, _P, C.POINTER(PixelCoef), _P, _I, _I, _I, _P]),
    'cdx_latent_encode': (_I, [_P, _P, _P, _P, _I, _F, C.POINTER(DdimCoef), C.POINTER(_F), _I, _I, _P, _F, _F, _P, _I, _I,
                               _I, _I, _P]),
    'cdx_latent_decode': (_I, [_P, _P, _I, _P, _P, _I, _F, C.POINTER(DdimCoef), C.POINTER(_F), _I, _P, _P, _I, _I, _I, _I,
                               _P]),
    'cdx_cycle_lockstep': (_I, [_P, _P, _P, _P, _P, _I, _F, _F, C.POINTER(DdimCoef), C.POINTER(_F), _I, _P, _F, _F, _P, _P, _I, _I, _I, _I,
                                _P]),
    'cdx_cycle_lockstep_masked': (_I, [_P, _P, _P, _P, _P, _I, _F, _F, C.POINTER(DdimCoef), C.POINTER(_F), _I, _P, _F, _F, _P, _P, _I, _I, _I,
                                       _I, _P, _P]),
    'cdx_cycle_lockstep_ctl': (_I, [_P, _P, _P, _P, _P, _I, _F, _F, C.POINTER(DdimCoef), C.POINTER(_F), _I, _P, _F, _F, _P, _P, _I, _I, _I,
                                    _I, _P, _P, C.POINTER(AttnControl)]),
    'cdx_cycle_lockstep_refine': (_I, [_P, _P, _P, _P, _P, _I, _F, _F, C.POINTER(DdimCoef), C.POINTER(_F), _I, _P, _F, _F, _P, _P, _I, _I,
                                       _I, _I, _P, _P, C.POINTER(AttnControl), _P]),
    'cdx_cycle_lockstep_mutual': (_I, [_P, _P, _P, _P, _P, _I, _F, _F, C.POINTER(DdimCoef), C.POINTER(_F), _I, _P, _F, _F, _P, _P, _I, _I,
                                       _I, _I, _P, _P, _I, _I]),
    'cdx_cycle_lockstep_pnp': (_I, [_P, _P, _P, _P, _P, _I, _F, _F, C.POINTER(DdimCoef), C.POINTER(_F), _I, _P, _F, _F, _P, _P, _I, _I,
                                    _I, _I, _P, _P, _I, _I, _I, C.POINTER(_I), _I]),
    'cdx_cycle_lockstep_semantic': (_I, [_P, _P, _P, _P, _P, _I, _F, _F, C.POINTER(DdimCoef), C.POINTER(_F), _I, _P, _F, _F, _P, _P, _I, _I,
                                         _I, _I, _P, _P, _P, C.POINTER(SemanticGuidanceC)]),
    'cdx_cycle_lockstep_semantic_attn': (_I, [_P, _P, _P, _P, _P, _I, _F, _F, C.POINTER(DdimCoef), C.POINTER(_F), _I, _P, _F, _F, _P, _P, _I,
                                              _I, _I, _I, _P, _P, _P, C.POINTER(SemanticGuidanceC), C.POINTER(SemanticAttnMaskC)]),
    'cdx_cycle_lockstep_sampler': (_I, [_P, _P, _P, _P, _P, _I, _F, _F, C.POINTER(DdimCoef), C.POINTER(_F), _I, _P, _F, _F, _P, _P, _I, _I,
                                        _I, _I, _P, C.POINTER(SamplerC), _P, C.POINTER(AttnControl), _P, C.POINTER(MutualControlC),
                                        C.POINTER(PnpControlC), _P, C.POINTER(SemanticGuidanceC), C.POINTER(SemanticAttnMaskC)]),
    'cdx_cycle_lockstep_blend': (_I, [_P, _P, _P, _P, _P, _I, _F, _F, C.POINTER(DdimCoef), C.POINTER(_F), _I, _P, _F, _F, _P, _P, _I, _I,
                                      _I, _I, _P, C.POINTER(SamplerC), _P, C.POINTER(AttnControl), _P, C.POINTER(MutualControlC),
                                      C.POINTER(PnpControlC), _P, C.POINTER(SemanticGuidanceC), C.POINTER(SemanticAttnMaskC),
                                      C.POINTER(LocalBlendC)]),
    'cdx_local_blend_mask': (_I, [_P, _P, _I, _I, _P, _P, _F, _F, _P, _I, _I, _I, _P]),
    'cdx_mask_pool': (_I, [_P, _P, _P, _I, _I, _I, _I, _P]),
    'cdx_mask_composite': (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    'cdx_edit_map': (_I, [_P, _P, _P, _P, _I, _F, _F, _F, _P, _I, _I, _P, _I, _I, _I, _I, _P]),
    'cdx_edit_map_from_eps': (_I, [_P, _P, _P, _F, _I, _I, _P, _I, _I, _I, _I, _P]),
    'cdx_edit_mask': (_I, [_P, _P, _I, _F, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    'cdx_latent_loop_ens': (_I, [_P, _I, _P, _P, _P, _P, _I, _P, _P, C.POINTER(DdimCoef), C.POINTER(_F), _I, _I, _P, _F, _F, _P, _I, _P, _P, _P,
                                 _I, _I, _I, _I, _P]),
    'cdx_clip_preprocess': (_I, [_P, _P, _I, _I, _I, _P, _P]),
    'cdx_clip_image_features': (_I, [_P, _P, _I, _P, _P]),
    'cdx_text_features': (_I, [_P, _P, _I, _I, _P, _P]),
    'cdx_dclip_scores': (_I, [_P, _P, _P, _P, _P, _I, _I, _P, _P, _P]),
    'cdx_image_metrics': (_I, [_P, _P, _P, _I, _I, _I, _P, _P]),
    'cdx_pixel_encode': (_I, [_P, _P, C.POINTER(PixelCoef), C.POINTER(_F), _I, _P, _F, _F, _P, _I, _I, _I, _P]),
    'cdx_pixel_decode': (_I, [_P, _P, _I, C.POINTER(PixelCoef), C.POINTER(_F), _I, _P, _P, _I, _I, _I, _P]),
    'cdx_pixel_cycle_lockstep': (_I, [_P, _P, _P, C.POINTER(PixelCoef), C.POINTER(_F), _I, _I, _P, _F, _F, _P, _I, _I, _I, _P]),
    'cdx_latent_cycle_pair': (_I, [_P, _P, _P, C.POINTER(DdimCoef), C.POINTER(_F), _I, _I, _P, _F, _F, _P, _P, _I, _I, _I, _I, _P]),
    'cdx_latent_cycle_fan': (_I, [_P, _I, _I, _P, _P, _P, _P, _I, C.POINTER(_F), C.POINTER(_F), C.POINTER(DdimCoef), C.POINTER(_F), _I, _P,
                                  _F, _F, _P, _P, _I, _I, _I, _P]),
    'cdx_latent_cycle_fan_masked': (_I, [_P, _I, _I, _P, _P, _P, _P, _I, C.POINTER(_F), C.POINTER(_F), C.POINTER(DdimCoef), C.POINTER(_F), _I,
                                         _P, _F, _F, _P, _P, _I, _I, _I, _P, _P]),
    'cdx_ensemble_select': (_I, [_P, _I, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    'cdx_op_conv3x3': (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    'cdx_op_linear': (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _P]),
    'cdx_op_groupnorm': (_I, [_P, _P, _P, _P, _F, _I, _P, _I, _I, _I, _P]),
    'cdx_op_layernorm': (_I, [_P, _P, _P, _P, _P, _I, _I, _P]),
    'cdx_op_attention': (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _F, _P]),
    'cdx_op_attention_rows': (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _F, C.POINTER(_I), _P]),
    'cdx_op_attention_kv_rows': (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _F, C.POINTER(_I), _P]),
    'cdx_op_attention_accum': (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _F, C.POINTER(_I), _I, _P]),
    'cdx_op_nchw_to_nhwc': (_I, [_P, _P, _P, _I, _I, _I, _P]),
    'cdx_op_nhwc_to_nchw': (_I, [_P, _P, _P, _I, _I, _I, _P]),
    'cdx_op_groupnorm_ex': (_I, [_P, _P, _I, _P, _I, _P, _P, _F, _I, _P, _P, _I, _P, _P, _P, _I, _I, _P]),
    'cdx_op_groupnorm_rows': (_I, [_P, _P, _I, _P, _I, _P, _P, _F, _I, _P, _P, _I, C.POINTER(_I), _P, _P, _P, _P, _I, _I, _P]),
    'cdx_op_layernorm_ex': (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _P]),
    'cdx_op_softmax_rows': (_I, [_P, _P, C.c_int64, _I, _I, _I, _P]),
    'cdx_op_produce_norm': (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _F, _P, _P, _P, _P, C.POINTER(_I), _P]),
    'cdx_op_gemm': (_I, [_P, C.POINTER(GemmDesc), C.POINTER(_I), _P]),
    'cdx_op_attention_net': (_I, [_P, C.POINTER(AttentionNetDesc), C.POINTER(_I), _P]),
    'cdx_op_attention_net_weighted': (_I, [_P, C.POINTER(AttentionNetDesc), C.POINTER(_F), C.POINTER(_I), _P]),
    'cdx_op_latent_chains': (_I, [_P, C.POINTER(LatentChainsDesc), _I, _P]),
    'cdx_op_pixel_lockstep': (_I, [_P, _P, _P, _P, _P, _P, _P, C.POINTER(PixelCoef), _I, _I, _I, _I, _P]),
}


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f'{LIB_PATH} is missing: build it with `python -c "import __graft_entry__ as g; g.build()"` '
            f'(nvcc, sm_90a).  The engine has no CPU fallback.')
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)      # AttributeError here = header / library mismatch
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


class CdxError(RuntimeError):
    pass


def check(rc):
    """Translate a CDX_E_* status into the exception type the reference's own checks raise."""
    if rc == 0:
        return
    msg = (lib.cdx_last_error() or b'').decode('utf-8', 'replace')
    if rc == -1:
        raise AssertionError(msg)     # the reference uses assert for preconditions (SDW:178, DDIM:268, DW:472)
    raise CdxError(f'libcdx error {rc}: {msg}')
