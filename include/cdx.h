/*
 * cdx.h -- C ABI of libcdx.so, the H100-native CycleDiffusion sampling engine.
 *
 * This is the drop-in boundary for the one hot path of ChenWu98/cycle-diffusion: the DPM-Encoder
 * inversion + decode-with-recovered-noise loops including the U-Net / VAE forwards.  Every entry
 * point cites the reference interface it replaces (paths relative to the reference repo root;
 * SDW = model/gan_wrapper/stable_diffusion_stochastic_text_wrapper.py,
 * DW  = model/gan_wrapper/ddpm_ddim_wrapper.py,
 * DDIM = model/lib/stable_diffusion/ldm/models/diffusion/ddim.py,
 * OAI = model/lib/stable_diffusion/ldm/modules/diffusionmodules/openaimodel.py,
 * AEM = model/lib/stable_diffusion/ldm/modules/diffusionmodules/model.py,
 * IU  = model/lib/ddpm_ddim/models/improved_ddpm/unet.py).
 *
 * Conventions
 *   - plain pointers and sizes only; no torch types.  All tensors are fp32.
 *   - "dev" pointers are CUDA device pointers owned by the caller (e.g. torch.Tensor.data_ptr()),
 *     never retained past the call.  Image / latent tensors at the boundary are NCHW contiguous,
 *     exactly the reference's layout; the engine converts to its internal NHWC layout itself.
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream).  No call synchronises
 *     the device; every call only enqueues work on `stream` (weight loading excepted).
 *   - every function returns 0 on success, a negative CDX_E_* code otherwise; cdx_last_error()
 *     returns a human-readable message for the calling thread's last failure.
 *   - an engine is bound to one device and is NOT thread-safe; use one engine per device/rank.
 */
#ifndef CDX_H_
#define CDX_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CDX_ABI_VERSION 2

#define CDX_OK 0
#define CDX_E_INVALID (-1)   /* bad argument / precondition (the reference's assert) */
#define CDX_E_CUDA (-2)      /* CUDA runtime error */
#define CDX_E_STATE (-3)     /* call order (e.g. forward before finalize) */
#define CDX_E_NOMEM (-4)

typedef struct cdx_engine cdx_engine;
typedef struct cdx_net cdx_net;

/* ---------------------------------------------------------------- engine ------------------- */
int cdx_abi_version(void);
const char* cdx_last_error(void);
/* Creates the per-device context (workspace arena, SM count).  Fails with CDX_E_CUDA when no CUDA
 * device is usable: there is no CPU fallback. */
int cdx_engine_create(int device, cdx_engine** out);
void cdx_engine_destroy(cdx_engine* e);
/* bytes currently reserved by the activation arena (for reporting) */
size_t cdx_engine_workspace_bytes(const cdx_engine* e);
/* number of kernels this engine has launched since creation (bench.py's gpu_launches) */
uint64_t cdx_engine_launch_count(const cdx_engine* e);
/* Per-kernel-family timing with CUDA events on the launching stream (off by default; bench.py turns it on for a
 * separate, untimed pass).  Tags: 0 conv3x3 FFMA, 1 dense FFMA, 2 batched (attention) FFMA, 3 conv3x3 tensor-core,
 * 4 dense tensor-core, 5 batched tensor-core, 6 GroupNorm, 7 LayerNorm, 8 softmax, 9 other.  profile_read synchronises the
 * device, sums the records of `tag` (ms, algorithmic flops / bytes, launches) and keeps them until profile(e, 1/0)
 * is called again. */
#define CDX_PROF_NTAGS 10
int cdx_engine_profile(cdx_engine* e, int enable);
int cdx_engine_profile_read(cdx_engine* e, int tag, double* ms, double* flops, double* bytes, uint64_t* launches);
/* select the dense-contraction path:
 *   0 = SIMT fp32 FFMA tiles (exact fp32)
 *   1 = tensor cores (wgmma), fp32-faithful split products (default): weight GEMMs / convs as 3 x wgmma .f16 over an fp16 hi/lo split of
 *       power-of-two-scaled operands, attention and activation x activation contractions as 3 x wgmma .tf32
 *   2 = as 1 but attention unfused (A/B comparisons)
 *   3 = as 1 with every contraction as 3 x wgmma .tf32 (the round-1 scheme)
 *   4 = FAST PATH, not fp32-faithful: weight GEMMs / convs with the hi*hi term only (plain fp16 inputs, fp32 accumulate);
 *       reported separately by bench.py together with its measured |delta pixel|
 *   5 = "autocast" (the reference wrappers' precision="autocast", txt2img.py --precision autocast): as 4, and the fused self- /
 *       cross-attention of the SD U-Net also single-term (S = Q_hi K_hi^T, O = P_hi V_hi over fp16 hi planes, P = fp16(p * 2^10)).
 *       Activations stay fp32 in memory and every accumulation is fp32; GroupNorm / LayerNorm / softmax, the sampler kernels and
 *       the paths that use 3xTF32 or FFMA in mode 1 (d = 160 attention, the VAE mid-block, M < 64, the text towers) are
 *       unchanged.  Not bit-compatible with torch.autocast, which rounds every op's output to fp16; at least as accurate. */
int cdx_engine_set_mma_mode(cdx_engine* e, int mode);
/* Persistent tensor-core GEMM for unsplit dense fp16-split work (default on; CDX_PERSIST=0 in the environment when the engine is
 * created turns it off).  enable 0: one CTA per work item.  max_ctas > 0 caps the persistent grid (a CTA then walks more work
 * items; for tests), 0: one CTA per SM.  Outputs are bit-identical in every setting. */
int cdx_engine_set_persist(cdx_engine* e, int enable, int max_ctas);

/* ---------------------------------------------------------------- networks ----------------- */
#define CDX_UNET_OPENAI 1 /* SD v1 / LDM text2img U-Net: OAI:413-742 + attention.py:152-261 */
#define CDX_UNET_IDDPM 2  /* improved-DDPM pixel U-Net: IU:401-668 */
#define CDX_UNET_DDPM 3   /* Ho et al. DDPM pixel U-Net (CelebA-HQ / LSUN checkpoints, DW:360-369): models/ddpm/diffusion.py:192-337 --
                             ResnetBlock + single-head AttnBlock (GroupNorm eps 1e-6, swish), [sin | cos] timestep embedding, conv
                             down / up sampling (asymmetric pad), num_res_blocks + 1 decoder blocks per level (SURVEY 8f-4) */

typedef struct cdx_unet_config {
  int kind;                /* CDX_UNET_* */
  int in_channels, out_channels, model_channels, num_res_blocks;
  int n_mult;
  int channel_mult[8];
  int n_attn;
  int attention_ds[8];     /* downsample factors at which attention runs (OAI:541 / IU:506) */
  int num_heads;           /* OPENAI: heads (d_head = ch / heads, legacy=False, OAI:542-549) */
  int num_head_channels;   /* IDDPM: channels per head (IU:287-293) */
  int context_dim;         /* OPENAI: cross-attention context width (768 SD, 1280 LDM); 0 = the unconditional LDM U-Net
                              (use_spatial_transformer=False, OAI:560-577): attention layers are AttentionBlock + QKVAttentionLegacy
                              (OAI:278-351) with num_head_channels (or num_heads) and the forward takes no context */
} cdx_unet_config;

typedef struct cdx_vae_config { /* AutoencoderKL ddconfig, v1-inference.yaml:51-65 */
  int ch;
  int n_mult;
  int ch_mult[8];
  int num_res_blocks;
  int in_channels, out_ch, z_channels, embed_dim;
  /* vq != 0: VQModelInterface first stage of the unconditional LDMs (ldm/models/autoencoder.py:14-21, 258-282; SURVEY 8f-4): encoder
     -> quant_conv gives h [B, embed_dim, h, w] (no moments, no quantisation on the way in); decode = nearest code of the n_embed x
     embed_dim codebook `quantize.embedding.weight` (taming VectorQuantizer2.forward: argmin of |z|^2 + |e|^2 - 2 z.e, straight-through
     value z + (z_q - z)) -> post_quant_conv -> decoder */
  int vq, n_embed;
} cdx_vae_config;

typedef struct cdx_text_config { /* CLIP ViT-L/14 text tower as FrozenCLIPEmbedder uses it (SURVEY 8f-1): HF CLIPTextModel
                                    "openai/clip-vit-large-patch14": 12 layers, width 768, 12 heads, 77 positions, quick-GELU */
  int vocab_size, width, layers, heads, max_len, mlp_width;
  int kind;     /* CDX_TEXT_CLIP (0 also accepted) or CDX_TEXT_XTRANSFORMER: the LDM BERTEmbedder's in-tree encoder
                   (encoders/modules.py:79-98 -> x_transformer.py TransformerWrapper(Encoder(dim, depth))): pre-LN blocks of
                   bias-free q/k/v (heads x dim_head), full attention, exact-GELU feed-forward; 30522 BERT word pieces */
  int dim_head; /* XTRANSFORMER: per-head width (x_transformer DEFAULT_DIM_HEAD = 64; heads * dim_head may differ from width) */
  /* DirectionalCLIP towers (SURVEY 8f-3; model/energy/clean_clip.py:7-41 runs OpenAI CLIP ViT-B/32 encode_image / encode_text):
     proj_dim > 0 adds the projection head (text: `text_projection.weight` [proj, width], applied to the EOT token's final-LN
     state; vision: `visual_projection.weight`).  kind CDX_CLIP_VISION: the ViT image tower, `patch` x `patch` patches of an
     `image_size`^2 input (HF CLIPVisionModel names under `vision_model.`; vocab_size / max_len unused) */
  int proj_dim, patch, image_size;
} cdx_text_config;
#define CDX_TEXT_CLIP 1
#define CDX_TEXT_XTRANSFORMER 2
#define CDX_CLIP_VISION 3
/* OpenCLIP ViT-H/14 text tower of SD 2.x (FrozenOpenCLIPEmbedder, layer="penultimate"): the parameter names and order of
   CDX_TEXT_CLIP, exact-erf GELU in the MLP instead of quick-GELU.  `layers` is the number of blocks that run (23 of 24 for the
   penultimate output); the final LayerNorm follows the last of them. */
#define CDX_TEXT_OPENCLIP 4

/* Build the host-side execution plan and parameter inventory (no GPU work). */
int cdx_unet_create(cdx_engine* e, const cdx_unet_config* cfg, cdx_net** out);
int cdx_vae_create(cdx_engine* e, const cdx_vae_config* cfg, cdx_net** out);
/* Text tower; parameter names are HF CLIPTextModel's (text_model.embeddings.token_embedding.weight, ...), i.e. the SD
 * checkpoint's cond_stage_model.transformer.* keys with that prefix stripped. */
int cdx_text_create(cdx_engine* e, const cdx_text_config* cfg, cdx_net** out);
void cdx_net_destroy(cdx_net* n);

/* Parameter inventory in the reference checkpoint's own key names (SURVEY.md Appendix C), so a
 * loader can walk torch.load(ckpt)["state_dict"] (txt2img.py:27-32; DW:378-379). */
int cdx_net_num_params(const cdx_net* n);
const char* cdx_net_param_name(const cdx_net* n, int i);
int cdx_net_param_shape(const cdx_net* n, int i, int64_t dims[4]); /* returns rank */
/* Copy one parameter (host or device fp32, dense, reference layout e.g. OIHW) into the engine. */
int cdx_net_load_param(cdx_net* n, const char* name, const float* data, int data_on_device,
                       const int64_t* dims, int rank);
/* All parameters present -> repack (conv3x3 OIHW -> O,kh,kw,I; split hi/lo planes for 3xTF32). */
int cdx_net_finalize(cdx_net* n);
/* The packed device blob holding every weight of this net; valid after the first load_param.
 * Multi-GPU: rank 0 loads + finalizes, every rank calls cdx_net_adopt_blob() after receiving the
 * blob with one ncclBroadcast (the only collective on the path; replaces the per-process
 * torch.load of txt2img.py:25-42 / DW:378-379). */
int cdx_net_weight_blob(cdx_net* n, void** dev_ptr, size_t* bytes);
int cdx_net_adopt_blob(cdx_net* n); /* mark a blob filled externally (broadcast) as finalized */
/* Sinusoid frequency table for timestep_embedding (util.py:152-172 / nn.py:103-121): the host
 * passes the table computed with the reference expression so that CPU oracle and engine agree
 * bit-for-bit on the frequencies; `half` must equal model_channels/2. */
int cdx_unet_set_time_freqs(cdx_net* n, const float* freqs_host, int half);

/* Output parameterisation of a CDX_UNET_OPENAI net (CDX_E_INVALID for any other kind).  CDX_PRED_EPS (the default): the U-Net
 * predicts the noise.  CDX_PRED_V (SD 2.x "-v" checkpoints, parameterization: "v"): it predicts v, and the latent loop drivers
 * (cdx_latent_encode / _decode, cdx_cycle_lockstep, cdx_latent_loop_ens, cdx_latent_cycle_fan) convert the guidance-combined output
 * of a step at timestep t as e_t = sa_v[t] v + s1_v[t] x_t, pred_x0 = sa_v[t] x_t - s1_v[t] v inside their fused step kernels.
 * sa_v / s1_v: host [T], fp32(sqrt(abar_t)) and fp32(sqrt(1 - abar_t)) of the float64 schedule; every loop timestep must be < T.
 * cdx_latent_cycle_pair rejects v nets; the single-op cdx_ddim_* kernels are eps-only. */
#define CDX_PRED_EPS 0
#define CDX_PRED_V 1
int cdx_unet_set_prediction(cdx_net* unet, int prediction, const float* sa_v_host, const float* s1_v_host, int T);

/* UNetModel.forward (OAI:710-742 via LatentDiffusion.apply_model ddpm.py:882-983 / IU:639-668).
 * x, out: [B, C, H, W] NCHW dev; t_dev: [B] float timesteps on device (the reference's int64
 * timesteps are cast with .float() at util.py:165); ctx_dev: [B, ctx_len, context_dim] or NULL
 * (IDDPM).  out has out_channels channels (IDDPM: 6 = eps | sigma). */
int cdx_unet_forward(cdx_net* n, const float* x_dev, const float* t_dev, const float* ctx_dev,
                     int ctx_len, float* out_dev, int B, int H, int W, void* stream);

/* AutoencoderKL.encode (autoencoder.py:324-328 + AEM:434-459): img [B,3,R,R] in [-1,1] ->
 * moments [B, 2*embed_dim, R/8, R/8] (mean | logvar), both NCHW dev. */
int cdx_vae_encode(cdx_net* n, const float* img_dev, float* moments_dev, int B, int R, void* stream);
/* The same for any image shape: img [B,3,H,W] -> moments [B, 2*embed_dim, H/f, W/f], f = 2^(len(ch_mult)-1).
 * H and W must be multiples of f (CDX_E_INVALID otherwise).  cdx_vae_encode(..., R, ...) is this call with H = W = R. */
int cdx_vae_encode_hw(cdx_net* n, const float* img_dev, float* moments_dev, int B, int H, int W, void* stream);
/* FrozenCLIPEmbedder.forward after tokenisation (ldm/modules/encoders/modules.py:140-158 -> transformer(input_ids=tokens)
 * .last_hidden_state; HF modeling_clip.py CLIPTextTransformer.forward, transformers==4.19.2 pinned by environment.yml:466):
 * token + position embedding, `layers` pre-LN blocks with causal self-attention and quick-GELU MLP, final LayerNorm.
 * ids_dev [B, L] int32 token ids (L <= max_len); out_dev [B, L, width] fp32.
 * kind XTRANSFORMER: BERTEmbedder.forward after tokenisation = transformer(tokens, return_embeddings=True)
 * (x_transformer.py:598-626, 481-523): parameter names transformer.token_emb.weight, transformer.attn_layers.layers.N.* ... */
int cdx_text_encode(cdx_net* n, const int* ids_dev, int B, int L, float* out_dev, void* stream);
/* AutoencoderKL.decode (autoencoder.py:330-333 + AEM:535-568): z [B,embed_dim,h,h] (already
 * divided by scale_factor) -> img [B, out_ch, 8h, 8h]. */
int cdx_vae_decode(cdx_net* n, const float* z_dev, float* img_dev, int B, int h, void* stream);
/* The same for any latent shape: z [B,embed_dim,h,w] -> img [B, out_ch, f*h, f*w], f = 2^(len(ch_mult)-1).
 * cdx_vae_decode(..., h, ...) is this call with w = h. */
int cdx_vae_decode_hw(cdx_net* n, const float* z_dev, float* img_dev, int B, int h, int w, void* stream);

/* ---------------------------------------------------------------- per-step kernels ---------- */
/* All element counts `n` are B*C*H*W of one NCHW tensor; scalars are the batch-uniform fp32
 * coefficients the reference broadcasts as [B,1,1,1] tensors.  Arithmetic is done op-by-op with
 * round-to-nearest (no FMA contraction) in the reference's evaluation order, so these are
 * bit-exact against the reference CPU path on identical inputs. */

/* out = a*x + b  (image normalisation SDW:176 / DW:470, post-process SDW:135-137, 1/scale_factor) */
int cdx_affine(cdx_engine* e, const float* x, float a, float b, float* out, size_t n, void* stream);
/* out = (x + b) * a   ((image - 0.5) * 2.0, exact reference order) */
int cdx_shift_scale(cdx_engine* e, const float* x, float b, float a, float* out, size_t n, void* stream);
/* x_t = sqrt_a*x0 + sqrt_1ma*noise  (DDIM:477-479 / DW:310-314) */
int cdx_q_sample(cdx_engine* e, const float* x0, const float* noise, float sqrt_a, float sqrt_1ma,
                 float* out, size_t n, void* stream);
/* DiagonalGaussianDistribution.sample * scale_factor (distributions.py:24-37, ddpm.py:536-543):
 * moments [B,2C,h,w]; noise [B,C,h,w] or NULL for the posterior mean (latentdiff copy). */
int cdx_vae_posterior(cdx_engine* e, const float* moments, const float* noise, float scale_factor,
                      float* out, int B, int C, int hw, void* stream);

typedef struct cdx_ddim_coef { /* one DDIM step, fp32 scalars exactly as ddim.py:570-573 builds them */
  float sqrt_at;        /* a_t.sqrt() */
  float sqrt_1m_at;     /* (1 - a_t).sqrt()                 -- sample_xt_next, ddim.py:597 */
  float sqrt_1m_at_tab; /* ddim_sqrt_one_minus_alphas[index] -- compute_eps, ddim.py:573 */
  float sqrt_aprev;     /* a_prev.sqrt() */
  float dir_coef;       /* (1 - a_prev - sigma_t**2).sqrt() */
  float sigma;          /* sigma_t */
} cdx_ddim_coef;

/* DDIMSampler.sample_xt_next (ddim.py:582-601): posterior sample x_{t-1} | x_t, x0 */
int cdx_ddim_posterior_sample(cdx_engine* e, const float* x0, const float* xt, const float* noise,
                              const cdx_ddim_coef* c, float* xt_next, size_t n, void* stream);
/* CFG combine + DDIMSampler.compute_eps tail (ddim.py:555-559, 575-579).  e_uc may be NULL
 * (scale 1 -> e_c only, ddim.py:550-551). */
int cdx_ddim_compute_eps(cdx_engine* e, const float* xt, const float* xt_next, const float* e_c,
                         const float* e_uc, float scale, const cdx_ddim_coef* c, float* eps_out,
                         size_t n, void* stream);
/* CFG combine + DDIMSampler.p_sample_ddim_with_eps tail (ddim.py:613-617, 634-645). */
int cdx_ddim_step_with_eps(cdx_engine* e, const float* x, const float* e_c, const float* e_uc,
                           float scale, const float* eps, const cdx_ddim_coef* c, float* x_prev,
                           size_t n, void* stream);

typedef struct cdx_pixel_coef { /* one step of the pixel-space samplers, DW:114-307 */
  int ddpm;           /* 1 = sample_type 'ddpm', 0 = 'ddim' */
  float sqrt_at;      /* at.sqrt() */
  float sqrt_1m_at;   /* (1 - at).sqrt() */
  float sqrt_at_next; /* at_next.sqrt() */
  float c1, c2;       /* ddim: eta*sqrt((1-at/at_next)(1-at_next)/(1-at)), sqrt((1-at_next)-c1^2) */
  float w0, wt, post_std;   /* ddpm posterior q(x_{t-1}|x_t,x0): DW:291-298 */
  float weight, inv_sqrt_1m_bt, std_model, mask; /* ddpm model mean / exp(0.5 logvar): DW:202-210 */
} cdx_pixel_coef;

/* sample_xt_next (DW:283-307) */
int cdx_pixel_posterior_sample(cdx_engine* e, const float* x0, const float* xt, const float* noise,
                               const cdx_pixel_coef* c, float* xt_next, size_t n, void* stream);
/* compute_eps (DW:230-280); et: U-Net output [B,Cnet,H,W] of which the first C channels are used
 * (learn_sigma split, DW:236-238); chw = C*H*W, net_chw = Cnet*H*W */
int cdx_pixel_compute_eps(cdx_engine* e, const float* xt, const float* xt_next, const float* et,
                          const cdx_pixel_coef* c, float* eps_out, int B, int chw, int net_chw,
                          void* stream);
/* denoising_step_with_eps / denoising_step (DW:114-227, diffusion_utils.py:23-136) */
int cdx_pixel_step_with_eps(cdx_engine* e, const float* xt, const float* et, const float* eps,
                            const cdx_pixel_coef* c, float* xt_next, int B, int chw, int net_chw,
                            void* stream);

/* ---------------------------------------------------------------- loop drivers -------------- */
/* DDIMSampler._ddpm_ddim_encoding (ddim.py:450-501), all refine steps on `stream`, no host sync.
 *   x0      [B,C,h,w]        clean latent
 *   c, uc   [B,L,D]          conditioning / unconditional conditioning (uc may be NULL if scale==1)
 *   coef    host[n_steps]    loop order (i = 0 is the noisiest step, index = n_steps-1)
 *   t_host  host[n_steps]    timestep value fed to the U-Net at iteration i
 *   n_rec                    number of steps that recover noise (min(n_steps, white_box-skip-1))
 *   noise   [n_rec(+1 incl. x_T draw), B,C,h,w] dev: noise[0] = x_T draw, noise[1+i] = draw of
 *                            iteration i (unused when index==0, ddim.py:583-584)
 *   sqrt_a_T, sqrt_1ma_T     at.sqrt(), (1-at).sqrt() of ddim.py:478-479
 *   z_out   [B, n_rec+1, C,h,w]  = stack(z_list, dim=1) (SDW:203)
 */
int cdx_latent_encode(cdx_net* unet, const float* x0, const float* c, const float* uc, int ctx_len,
                      float scale, const cdx_ddim_coef* coef, const float* t_host, int n_steps,
                      int n_rec, const float* noise, float sqrt_a_T, float sqrt_1ma_T, float* z_out,
                      int B, int C, int h, int w, void* stream);
/* DDIMSampler.ddim_sampling_with_eps (ddim.py:395-448): z [B, n_eps+1, C,h,w] (x_T first, SDW:150-154);
 * extra_noise [n_steps-n_eps, B,C,h,w] for steps without recovered noise (may be NULL if none). */
int cdx_latent_decode(cdx_net* unet, const float* z, int n_eps, const float* c, const float* uc,
                      int ctx_len, float scale, const cdx_ddim_coef* coef, const float* t_host,
                      int n_steps, const float* extra_noise, float* x_out, int B, int C, int h, int w,
                      void* stream);
/* Both chains in lock-step (SURVEY.md 7 step 8 / 8b; the loop shape of Diffusers' CycleDiffusionPipeline.__call__): the source chain
 * of _ddpm_ddim_encoding (ddim.py:450-501) under c_src / src_scale and the target chain of ddim_sampling_with_eps (ddim.py:395-448)
 * under c_tgt / tgt_scale advance together, ONE U-Net call per step on the batch [source segments | target segments] (B rows per
 * segment; a chain contributes [uncond, cond] when its scale is neither 0 nor 1), and the noise recovered at step i is consumed by the
 * target chain inside the same fused elementwise kernel: no z buffer.  Requires all n_steps noises to be recoverable
 * (white_box_steps > custom_steps - skip); noise [n_steps+1, B,C,h,w] as for cdx_latent_encode.  z_out (optional, may be NULL)
 * receives [B, n_steps+1, C,h,w] exactly as cdx_latent_encode would produce it.  Per-sample results equal the two-phase
 * cdx_latent_encode + cdx_latent_decode up to the summation order of split-K GEMMs (the batch size differs). */
int cdx_cycle_lockstep(cdx_net* unet, const float* x0, const float* c_src, const float* c_tgt, const float* uc,
                       int ctx_len, float src_scale, float tgt_scale, const cdx_ddim_coef* coef,
                       const float* t_host, int n_steps, const float* noise, float sqrt_a_T,
                       float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w,
                       void* stream);
/* Mask-guided local editing (Blended Latent Diffusion on the lock-step loop; diffusers' inpaint / DiffEdit `mask_image`):
 * cdx_cycle_lockstep with mask [B,1,h,w] in [0,1] at latent resolution, 1 = "may change".  After each step the target chain's
 * x_{t-1} becomes m * x_{t-1}(target) + (1 - m) * x_{t-1}(source), per latent pixel and broadcast over the C channels, where the
 * source chain's x_{t-1} is its posterior sample of q(x_{t-1} | x_t, x0) of the real image (x0 itself on the last step).  The
 * blended value is also the next U-Net input, so the edited region is denoised in the context of the real surroundings.
 * m == 1 keeps the target value and m == 0 takes the source value EXACTLY: a mask of ones gives cdx_cycle_lockstep's output bit for
 * bit, a mask of zeros gives x0.  The source chain reads no mask; its z_out moves only in the last bits, through the one U-Net
 * call the rows share (fp16-split operands take one exponent per tensor).  mask == NULL is cdx_cycle_lockstep. */
int cdx_cycle_lockstep_masked(cdx_net* unet, const float* x0, const float* c_src, const float* c_tgt, const float* uc,
                              int ctx_len, float src_scale, float tgt_scale, const cdx_ddim_coef* coef,
                              const float* t_host, int n_steps, const float* noise, float sqrt_a_T,
                              float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w,
                              void* stream, const float* mask);
/* Prompt-to-Prompt attention control (Hertz et al., 2022; "Cross Attention Control"), the "replace" edit, on the lock-step loop.
 * Only the target chain's cond row (the row under c_tgt[b]) is controlled; its uncond row and every source row run unchanged.  At
 * loop step i (0-based, of n_steps):
 *   - i < cross_steps, every cross-attention layer: the controlled row's probabilities are P_src . A_b, where P_src is the source
 *     row's softmax(Q K^T) under c_src[b] (same layer and head) and A_b = token_map[b] [L,L] (source token -> target token; NULL
 *     token_map: the identity).  Computed as softmax(Q_src K_src^T) . V', V' projected once per loop from A_b . c_tgt[b] (to_v has
 *     no bias), A_b . c_tgt[b] formed by the engine's exact-fp32 GEMM.
 *   - i < self_steps, self-attention layers of at most self_max_tokens tokens: the controlled row's probabilities are the source
 *     row's.
 * Inside the fused attention kernel the controlled row reads the source row's Q and K tiles: no score matrix is formed and no
 * launch is added.  Needs a source row: src_scale != 0 (and tgt_scale != 0 with uc).  Every controlled layer must run the fused
 * kernel: mma modes 0 and 2, and mode 3 at head width 160, are rejected (CDX_E_INVALID) rather than run uncontrolled. */
typedef struct cdx_attn_control {
  int cross_steps, self_steps, self_max_tokens;
  const float* token_map;            /* device [B,L,L] or NULL */
} cdx_attn_control;
/* cdx_cycle_lockstep_masked with attention control: ctl and mask may each be NULL (both NULL: cdx_cycle_lockstep).  With
 * cross_steps == self_steps == 0 the result is cdx_cycle_lockstep_masked's bit for bit, and so is it with an identity token_map. */
int cdx_cycle_lockstep_ctl(cdx_net* unet, const float* x0, const float* c_src, const float* c_tgt, const float* uc,
                           int ctx_len, float src_scale, float tgt_scale, const cdx_ddim_coef* coef,
                           const float* t_host, int n_steps, const float* noise, float sqrt_a_T,
                           float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w,
                           void* stream, const float* mask, const cdx_attn_control* ctl);
/* Prompt-to-Prompt's "refine" edit: cdx_cycle_lockstep_ctl with own_weight (device [B,L], finite, >= 0; NULL: exactly
 * cdx_cycle_lockstep_ctl, which calls this).  At a controlled cross-attention step the controlled row's probabilities for target
 * token j become
 *     attn[j] = P_src . A_b[:, j]  +  own_weight[b, j] . P_tgt[j]
 * P_tgt being the row's own softmax(Q K^T) under c_tgt[b].  With A_b[i, j] = alpha_j [m(j) = i] eq_j and own_weight[b, j] =
 * (1 - alpha_j) eq_j this is P2P's refine: a target token aligned to source token m(j) takes that token's map, an unaligned one
 * keeps its own (times the equalizer eq).  Computed as
 *     out = softmax(Q_src K_src^T) . V'  +  softmax(Q_tgt K_tgt^T) . V'',   V'' projected once per loop from diag(w_b) . c_tgt[b]
 * the second term by one more fused-attention launch over the controlled rows only, which adds into the output.  Range bound: the
 * output's range slot (it sets the fp16 exponent of the to_out projection's operand) is the first term's slot plus max |V''| over
 * the controlled rows -- |out| <= max |V'| + max |V''| -- formed on the device once per loop; own_weight == 0 leaves it, and the
 * result, bit for bit as without own_weight.  Self-attention control is unchanged (the source row's probabilities). */
int cdx_cycle_lockstep_refine(cdx_net* unet, const float* x0, const float* c_src, const float* c_tgt, const float* uc,
                              int ctx_len, float src_scale, float tgt_scale, const cdx_ddim_coef* coef,
                              const float* t_host, int n_steps, const float* noise, float sqrt_a_T,
                              float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w,
                              void* stream, const float* mask, const cdx_attn_control* ctl, const float* own_weight);
/* Mutual self-attention control (MasaCtrl, Cao et al., 2023) on the lock-step loop: cdx_cycle_lockstep_masked (mask may be NULL)
 * where the target chain's rows keep their own queries but attend over the source chain's keys and values in the decoder's
 * self-attention layers, so the layout can follow the target prompt while identity, texture and background are fetched from the
 * real image.  At loop step i (0-based, of n_steps) with i >= start_step, in every SpatialTransformer whose index (counted in
 * forward order over the input blocks, the middle block and the output blocks; SD v1 / 2.x and LDM text2img have 16) is
 * >= start_layer, each target row computes softmax(Q_own K_src^T * scale) . V_src, where for sample b
 *   - the target's cond row (under c_tgt[b]) reads the source chain's cond row (under c_src[b]), and
 *   - the target's uncond row (present when tgt_scale is neither 0 nor 1) reads the source chain's uncond row, or its cond row when
 *     the source runs without one (src_scale 0 or 1).
 * Source rows and every cross-attention layer run unchanged.  MasaCtrl's defaults are start_step = 4, start_layer = 10 (the last
 * six layers: the decoder's two finest levels).  Inside the fused attention kernel a controlled row reads the source row's K and
 * V^T tiles: no launch is added.  The output stays a convex combination of rows of the layer's V, so its range slot is unchanged.
 * start_step >= n_steps or start_layer >= the net's layer count gives cdx_cycle_lockstep_masked's result bit for bit; negative
 * values, nets without SpatialTransformers, and mma modes 0 and 2 (and mode 3 at head width 160) on a controlled layer are
 * CDX_E_INVALID. */
int cdx_cycle_lockstep_mutual(cdx_net* unet, const float* x0, const float* c_src, const float* c_tgt, const float* uc,
                              int ctx_len, float src_scale, float tgt_scale, const cdx_ddim_coef* coef,
                              const float* t_host, int n_steps, const float* noise, float sqrt_a_T,
                              float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w,
                              void* stream, const float* mask, int start_step, int start_layer);
/* Plug-and-Play diffusion features (PnP, Tumanyan et al., 2023) on the lock-step loop: cdx_cycle_lockstep_masked (mask may be NULL)
 * where the target chain's rows take the source chain's decoder ResBlock features and self-attention queries and keys, so the real
 * image's spatial layout is kept while the target prompt sets its appearance.  The source row runs in the same U-Net call at the
 * same timestep, so no feature cache or separate inversion pass is needed.  Rows are mapped as cdx_cycle_lockstep_mutual maps them:
 * for sample b the target's cond row r reads the source chain's cond row s, and the target's uncond row (present when tgt_scale is
 * neither 0 nor 1) reads the source's uncond row, or the source's only row when it has no uncond row.  src_scale 0 is allowed: the
 * source's only row is then its uncond row, PnP's own unconditional source branch.  At loop step i (0-based, of n_steps):
 *   - i < feature_steps, for each k of feature_blocks[0 .. n_feature_blocks) (host ints, indices of the net's output blocks): the
 *     ResBlock output_blocks.k.0 gives row r  skip_r + out_layers(h_s), skip_r row r's own skip path (identity or skip_connection)
 *     and h_s row s's in_layers output plus its embedding, out_layers(h) = conv3x3(SiLU(GroupNorm(h))).  The GroupNorm before the
 *     conv writes row r from row s's input and statistics, so the conv reads row s's operand and adds its bias and row r's skip in
 *     its epilogue: no launch or byte is added, and the norm's range slot stays the max over what it wrote.
 *   - i < attention_steps, in the self-attention of every SpatialTransformer whose index in forward order (16 in SD v1 / 2.x and the
 *     LDM text2img net: input 0-5, middle 6, output 7-15) is >= attention_start_layer: row r computes softmax(Q_s K_s^T * scale) . V_r,
 *     the fused attention kernel reading row s's Q and K tiles (as Prompt-to-Prompt's self-attention control does).
 * Cross-attention and the source rows run unchanged.  PnP's defaults are feature_steps = int(0.8 n), attention_steps = int(0.5 n),
 * feature_blocks = {4} (up_blocks[1].resnets[1]) and attention_start_layer = 8 (up_blocks[1].attentions[1]).
 * feature_steps = attention_steps = 0, or n_feature_blocks = 0 with attention_start_layer >= the net's layer count, gives
 * cdx_cycle_lockstep_masked's result bit for bit.  CDX_E_INVALID: negative values or step counts above n_steps, a block index
 * outside the net's output blocks or given twice, nets without SpatialTransformers or a context, and mma modes 0 and 2 (and mode 3
 * at head width 160) on a controlled attention layer. */
int cdx_cycle_lockstep_pnp(cdx_net* unet, const float* x0, const float* c_src, const float* c_tgt, const float* uc,
                           int ctx_len, float src_scale, float tgt_scale, const cdx_ddim_coef* coef,
                           const float* t_host, int n_steps, const float* noise, float sqrt_a_T,
                           float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w,
                           void* stream, const float* mask, int feature_steps, int attention_steps,
                           int attention_start_layer, const int* feature_blocks, int n_feature_blocks);
/* Semantic guidance (SEGA, Brack et al., 2023; LEDITS++'s editing term) on the lock-step loop: cdx_cycle_lockstep_masked (mask may
 * be NULL) where concepts are added to or removed from the target chain's image, each where its own guidance is strongest.  Each
 * target chain gets m concept rows (1 <= m <= CDX_SEMANTIC_MAX), appended after all target rows, that run the U-Net at the chain's
 * own x_t and timestep under c_edit[b, k] (device [B, m, L, D]).  At loop step i (0-based, of n_steps), with o_uc the chain's uncond
 * row output (at tgt_scale 1 the chain is given an uncond row; its eps-hat stays the cond row exactly) and o_k concept k's, every
 * operation one rounded fp32 op:
 *   psi_k = scale[k] * (o_k - o_uc)                 scale[k] signed: negative removes the concept
 *   theta = Q(threshold[k], |psi_k| over the h*w plane of each channel), per image: r = threshold*(hw - 1), the floor(r)-th and
 *           ceil(r)-th smallest values interpolated as torch.quantile does (w = r - floor(r); w < 0.5 ? lo + w*(hi - lo) :
 *           hi - (hi - lo)*(1 - w))
 *   g_k   = (i < cooldown[k] and |psi_k| >= theta) ? psi_k : 0;   S = g_0 + g_1 + ... (left to right)
 *   G     = S + momentum_scale * nu;   nu <- beta * nu + beta1 * G      (nu per target chain, zero at the first step)
 *   eps-hat += G when i >= warmup   (v nets: on the guidance-combined v, before the conversion)
 * beta1 = fp32(1 - beta) formed by the caller in double.  The source chain and z_out are untouched but for the last bits the shared
 * U-Net call moves (fp16-split operands take one exponent per tensor).  One more launch per step, the threshold stage, runs between
 * the U-Net call and the step kernel.  CDX_E_INVALID: m outside 1..CDX_SEMANTIC_MAX, a threshold outside [0, 1), nets without a
 * context, uc == NULL, and a row count whose U-Net call needs more GroupNorm statistics than the engine's pool holds. */
#define CDX_SEMANTIC_MAX 8
typedef struct cdx_semantic_guidance {
  int m;
  float scale[CDX_SEMANTIC_MAX];       /* signed: -edit_guidance_scale with reverse_editing_direction, else +edit_guidance_scale */
  float threshold[CDX_SEMANTIC_MAX];   /* percentile lambda in [0, 1) */
  int cooldown[CDX_SEMANTIC_MAX];      /* concept k guides at steps i < cooldown[k] */
  int warmup;                          /* G is added at steps i >= warmup (the momentum runs from step 0) */
  float momentum_scale, beta, beta1;
} cdx_semantic_guidance;
int cdx_cycle_lockstep_semantic(cdx_net* unet, const float* x0, const float* c_src, const float* c_tgt, const float* uc,
                                int ctx_len, float src_scale, float tgt_scale, const cdx_ddim_coef* coef,
                                const float* t_host, int n_steps, const float* noise, float sqrt_a_T,
                                float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w,
                                void* stream, const float* mask, const float* c_edit, const cdx_semantic_guidance* sg);
/* LEDITS++'s implicit masks (Brack et al., 2024) on cdx_cycle_lockstep_semantic: each concept's term is kept only where the concept's
 * own cross-attention points.  The concept rows' cross-attention probabilities are probed in every SpatialTransformer of the input
 * and output blocks (never the middle block) whose token count is (h/4)(w/4) -- for SD v1 / 2.x and LDM text2img input blocks 7, 8
 * and output blocks 3, 4, 5 -- from the operands the layer multiplied.  For concept k of target chain t at loop step i:
 *   A(p)   = sum over those layers, over heads, over j = 1..n_tokens[k] of softmax_j(scale q_p . k_j) over all L keys
 *   As     = 3x3 smoothing of A, reflect padding 1, weights fp32(g_a g_b / (sum g)^2), g = (e^-1, 1, e^-1) in double (diffusers'
 *            GaussianSmoothing(3, 0.5)); products row-major, each rounded, added left to right
 *   M1(y, x) = As(y/4, x/4) >= Q(threshold[k], As over the (h/4)(w/4) grid)   (the quantile of cdx_cycle_lockstep_semantic)
 *   intersect: s(y, x) = sum over c ascending of |psi_k(c, y, x)|, M = M1 and s >= Q(threshold[k], s over h*w); else M = M1
 *   g_k    = (i < cooldown[k] and M(y, x)) ? psi_k : 0     (SEGA's per-channel threshold is not applied)
 * The sum over concepts, the momentum and the warmup are cdx_cycle_lockstep_semantic's.  One probe launch per probed layer per step,
 * and the threshold stage stays one launch.  CDX_E_INVALID: everything cdx_cycle_lockstep_semantic rejects, n_tokens[k] outside
 * 1..L-2, h or w not a multiple of 4 or below 8, and a net with no cross-attention of (h/4)(w/4) tokens in its input or output
 * blocks. */
typedef struct cdx_semantic_attn_mask {
  int intersect;                        /* also the channel-summed mask of |psi_k| */
  int n_tokens[CDX_SEMANTIC_MAX];       /* concept k's own tokens: 1..n_tokens[k] of its context, after the start token */
} cdx_semantic_attn_mask;
int cdx_cycle_lockstep_semantic_attn(cdx_net* unet, const float* x0, const float* c_src, const float* c_tgt, const float* uc,
                                     int ctx_len, float src_scale, float tgt_scale, const cdx_ddim_coef* coef,
                                     const float* t_host, int n_steps, const float* noise, float sqrt_a_T,
                                     float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w,
                                     void* stream, const float* mask, const float* c_edit, const cdx_semantic_guidance* sg,
                                     const cdx_semantic_attn_mask* am);
/* Edit-friendly inversion (LEDITS++, Brack et al., 2024; the edit-friendly DDPM noise space of Huberman-Spiegelglas et al., 2024)
 * on the lock-step loop.  The source chain is not a posterior chain: its x at every loop step k is drawn from q(x_k | x0) on its own,
 *   x_k = qa[k]*x0 + q1[k]*noise[k]      (k = 0: x_T, qa[0] == sqrt_a_T and q1[0] == sqrt_1ma_T; the last step's next x is x0)
 * and each step's noise z is recovered from the pair (x_i, x_{i+1}) and the source row's output.  kind:
 *   CDX_SAMPLER_DDIM_POSTERIOR  cdx_cycle_lockstep's DPM-Encoder chain (qa, q1, dpm unused)
 *   CDX_SAMPLER_DDIM_DRAWS      the independent draws with coef's DDIM step (coef must be the eta = 1 table): z = (x_{i+1} -
 *                               sqrt_aprev*D - dir_coef*e_t) / sigma, the target y_{i+1} = sqrt_aprev*D_y + dir_coef*e_y + sigma*z
 *   CDX_SAMPLER_DPMSOLVER_DRAWS the independent draws with the second-order SDE-DPM-Solver++ step (diffusers' sde-dpmsolver++
 *                               midpoint update): with D a chain's x0-prediction (formed from coef as the DDIM step forms pred_x0) and
 *                               D_prev its previous step's, mu = a*x + b*D (+ c*(D - D_prev) when order == 2), one rounded op each;
 *                               z = (x_{i+1} - mu_src) / n, y_{i+1} = mu_y + n*z.  dpm host [n_steps]; order 2 on step 0 is rejected.
 * With identical prompts and scales on both chains the target returns x0 up to rounding: each step hands it the source's next x.
 * Every control of the lock-step loop acts on U-Net rows before the update and composes unchanged: mask (the blend partner is the
 * source's next x), ctl with own_weight (cdx_cycle_lockstep_refine), mutual (cdx_cycle_lockstep_mutual), pnp (cdx_cycle_lockstep_pnp),
 * sg with c_edit (cdx_cycle_lockstep_semantic) and am (cdx_cycle_lockstep_semantic_attn), each NULL when off and exclusive as there.
 * The noise draws are cdx_cycle_lockstep's: noise[0] gives x_T, noise[1 + i] the source's x at loop step i + 1.  With kind
 * CDX_SAMPLER_DDIM_POSTERIOR every result equals the matching cdx_cycle_lockstep* entry point's.  One launch per step, as there.
 * CDX_E_INVALID: an unknown kind, qa / q1 / dpm missing for their kinds, qa[0] or q1[0] other than the x_T scalars, a dpm entry with
 * n <= 0, an order other than 1 or 2, or order 2 on step 0, and everything the matching entry point rejects. */
#define CDX_SAMPLER_DDIM_POSTERIOR 0
#define CDX_SAMPLER_DDIM_DRAWS 1
#define CDX_SAMPLER_DPMSOLVER_DRAWS 2
typedef struct cdx_dpm_coef { /* one SDE-DPM-Solver++ step s -> t, each formed in double from fp32 abar and rounded once */
  float a;      /* (sigma_t / sigma_s) * exp(-h), h = lambda_t - lambda_s, lambda = log(alpha) - log(sigma) */
  float b;      /* alpha_t * -expm1(-2h) */
  float c;      /* order 2: 0.5 * b / r0, r0 = (lambda_s - lambda_prev) / h; order 1: 0 */
  float n;      /* sigma_t * sqrt(-expm1(-2h)) */
  int order;    /* 1 or 2 */
} cdx_dpm_coef;
typedef struct cdx_sampler {
  int kind;                      /* CDX_SAMPLER_* */
  const cdx_dpm_coef* dpm;       /* host [n_steps], kind CDX_SAMPLER_DPMSOLVER_DRAWS */
  const float* qa; const float* q1;   /* host [n_steps]: sqrt(abar) and sqrt(1 - abar) of loop step k's level, the draw kinds */
} cdx_sampler;
typedef struct cdx_mutual_control { int start_step, start_layer; } cdx_mutual_control;   /* cdx_cycle_lockstep_mutual's */
typedef struct cdx_pnp_control {                                                        /* cdx_cycle_lockstep_pnp's */
  int feature_steps, attention_steps, attention_start_layer;
  const int* feature_blocks; int n_feature_blocks;
} cdx_pnp_control;
int cdx_cycle_lockstep_sampler(cdx_net* unet, const float* x0, const float* c_src, const float* c_tgt, const float* uc,
                               int ctx_len, float src_scale, float tgt_scale, const cdx_ddim_coef* coef,
                               const float* t_host, int n_steps, const float* noise, float sqrt_a_T,
                               float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w,
                               void* stream, const cdx_sampler* sampler, const float* mask, const cdx_attn_control* ctl,
                               const float* own_weight, const cdx_mutual_control* mutual, const cdx_pnp_control* pnp,
                               const float* c_edit, const cdx_semantic_guidance* sg, const cdx_semantic_attn_mask* am);
/* Prompt-to-Prompt's LocalBlend (Hertz et al., 2022; its AttentionStore and LocalBlend.get_mask) on the lock-step loop of
 * cdx_cycle_lockstep_sampler (same arguments; sampler may be NULL, the DPM-Encoder chain; mutual, pnp, c_edit, sg and am must be
 * NULL): at each loop step the target chain is kept to where the blend words' cross-attention points.  K = 1: one source and one
 * target chain per image b.  The cond rows of both chains are probed (the attention probe of cdx_cycle_lockstep_semantic_attn, same
 * layers) with per-token weights, each map as the row attended with it:
 *   W_src,v(p) = sum over layers, heads, j of P_src(p, j) v_src[b, j]                       (v: alpha or sub, source prompt)
 *   W_tgt,v(p) = the same of P_src with weights A_b v_tgt[b]  (+ P_tgt with own_weight[b] * v_tgt[b] under refine)
 *                at steps i < ctl->cross_steps (A_b = ctl->token_map, identity when NULL), else of P_tgt with v_tgt[b]
 * and R_v += W_v from the loop's first step on.  On the (h/4) x (w/4) grid, per image:
 *   blend = OR over src, tgt of  maxpool3x3(R_alpha) / max(R_alpha) > th_blend      (stride 1, padding never wins)
 *   sub   = OR over src, tgt of  R_sub / max(R_sub) > th_sub                          (only with the subtract pair)
 *   m     = blend AND NOT sub, nearest x4 to h x w, times mask when given               (a map whose max is 0 adds nothing)
 * At steps i >= start_step the target's x_{t-1} is blended with the source's under m (cdx_cycle_lockstep_masked's blend); before,
 * the loop runs exactly as without LocalBlend.  Weight vectors: device [B, ctx_len], finite and >= 0 (not checked here).  One probe
 * launch per probed layer and one mask launch per step.  CDX_E_INVALID: a NULL blend or alpha vector, one subtract vector without
 * the other, start_step outside 0..n_steps, thresholds outside [0, 1), h or w not a multiple of 4, a source or target chain at
 * scale 0 with uc (no prompt row), and every control other than ctl / own_weight. */
typedef struct cdx_local_blend {
  const float* alpha_src;   /* device [B, ctx_len]: blend-word weights on the source prompt's tokens (P2P's alpha_layers) */
  const float* alpha_tgt;   /* device [B, ctx_len]: on the target prompt's tokens */
  const float* sub_src;     /* optional device [B, ctx_len]: subtract-word weights (P2P's substruct_layers), both or neither */
  const float* sub_tgt;
  int start_step;           /* loop steps i >= start_step blend: int(start_blend * n_steps) */
  float th_blend, th_sub;   /* in [0, 1) */
} cdx_local_blend;
int cdx_cycle_lockstep_blend(cdx_net* unet, const float* x0, const float* c_src, const float* c_tgt, const float* uc,
                             int ctx_len, float src_scale, float tgt_scale, const cdx_ddim_coef* coef,
                             const float* t_host, int n_steps, const float* noise, float sqrt_a_T,
                             float sqrt_1ma_T, float* x_out, float* z_out, int B, int C, int h, int w,
                             void* stream, const cdx_sampler* sampler, const float* mask, const cdx_attn_control* ctl,
                             const float* own_weight, const cdx_mutual_control* mutual, const cdx_pnp_control* pnp,
                             const float* c_edit, const cdx_semantic_guidance* sg, const cdx_semantic_attn_mask* am,
                             const cdx_local_blend* blend);
/* LocalBlend's mask stage alone (one launch): maps device [B*n_vec*n_terms, (h/4)(w/4)], entry (b*n_vec + v)*n_terms + t, vectors
 * v = 0, 1 the blend words of the source and target prompt, 2, 3 (n_vec == 4) the subtract words; run device [B*n_vec, (h/4)(w/4)]
 * += (term 0 + term 1 + ...) in fp32; mask_out device [B,1,h,w] <- cdx_cycle_lockstep_blend's m from run (times user_mask
 * [B,1,h,w] when given). */
int cdx_local_blend_mask(cdx_engine* e, const float* maps, int n_terms, int n_vec, float* run, const float* user_mask, float th_blend,
                         float th_sub, float* mask_out, int B, int h, int w, void* stream);
/* Helpers of masked editing (image resolution, one [B,1,H,W] mask broadcast over the channels):
 * cdx_mask_pool: mask [B,1,H,W] -> out [B,1,H/f,W/f], the mean of each f x f block (f = the first stage's factor: 8 for KL-f8,
 *   4 for VQ-f4), summed row by row then divided by f*f as torch.nn.functional.avg_pool2d(mask, f) does.  H, W multiples of f.
 * cdx_mask_composite: paste-back, out = m * clamp((dec + 1) * 0.5, 0, 1) + (1 - m) * image over [B,C,H,W] (dec the first stage's
 *   output in [-1,1], image in [0,1]); where m == 0 out is image exactly, where m == 1 the clamped decode exactly (the value of
 *   cdx_shift_scale(dec, 1, 0.5) followed by a clamp). */
int cdx_mask_pool(cdx_engine* e, const float* mask, float* out, int B, int H, int W, int f, void* stream);
int cdx_mask_composite(cdx_engine* e, const float* dec, const float* image, const float* mask, float* out, int B, int C, int H,
                       int W, void* stream);
/* Edit masks from two prompts (DiffEdit, Couairon et al., 2022): where the source and target predictions of the noised image
 * disagree is where the edit goes.  x0 [B,C,h,w] the encoded latent, c_src / c_tgt [B,ctx_len,D], noise [B,n_maps,C,h,w].
 * For image b and map k (k = 0 .. n_maps-1):
 *   x_t  = sqrt_a * x0[b] + sqrt_1ma * noise[b,k]               (cdx_q_sample's op order)
 *   d    = e(x_t, t, c_tgt[b]) - e(x_t, t, c_src[b])            per element, two U-Net rows, no uncond row
 *          (v-prediction nets: d = sa_v[t] * (v_tgt - v_src), so the map is in eps units; t must index the net's tables)
 *   s[p] = sum over c ascending of |d[c,p]|                       fp32
 *   acc[b,p] += s[p]                                              fp32, k ascending: one add per map
 * cdx_edit_map: the whole computation.  acc_out [B,h,w] is zeroed first.  The (map, image) pairs are walked map-major, as many
 *   whole pairs per U-Net call as rows_per_call (>= 2) allows, two rows per pair; the result does not depend on rows_per_call.  A
 *   call whose GroupNorm statistics would exceed the engine's pool (a 96-row SD call does; 48 rows fit) is rejected by the
 *   sizing pass, before anything runs.
 *   t, sqrt_a, sqrt_1ma: the first timestep of DDIMSchedule(S, eta, S - int(S*strength)) and that schedule's sqrt_a_T /
 *   sqrt_1ma_T.  Text-conditioned latent U-Nets only.
 * cdx_edit_map_from_eps: the accumulation alone, on given predictions e_src / e_tgt [B,n_maps,C,h,w], vscale multiplying each
 *   difference (1: eps nets, exactly), maps_per_launch maps per launch; acc_out [B,h,w] is zeroed first and is bit-identical for
 *   any maps_per_launch.
 * cdx_edit_mask: per image, map = acc / (n_maps*C) -> map_out [B,1,h,w]; mean = fp32(sum_p map in fp64 / (h*w)) (fixed
 *   summation order); M = ratio * mean (ratio > 0); mask_out [B,1,h,w] = (min(map, M) / M > 0.5) ? 1 : 0 when M > 0, all 0 when
 *   M == 0 (the two prompts predict the same: nothing to edit).  mask_img_out (nullable) [B,1,f*h,f*w]: the mask nearest-upsampled
 *   by f, which cdx_mask_pool(.., f) turns back into mask_out exactly.
 * Unlike diffusers' StableDiffusionDiffEditPipeline.generate_mask: the mean is per image (a mask never depends on its batch-mates),
 * two rows per map (the guidance scale cancels in the normalisation), and an all-zero map gives an empty mask. */
int cdx_edit_map(cdx_net* unet, const float* x0, const float* c_src, const float* c_tgt, int ctx_len, float t, float sqrt_a,
                 float sqrt_1ma, const float* noise, int n_maps, int rows_per_call, float* acc_out, int B, int C, int h,
                 int w, void* stream);
int cdx_edit_map_from_eps(cdx_engine* e, const float* e_src, const float* e_tgt, float vscale, int n_maps,
                          int maps_per_launch, float* acc_out, int B, int C, int h, int w, void* stream);
int cdx_edit_mask(cdx_engine* e, const float* acc, int n_maps, float ratio, float* map_out, float* mask_out,
                  float* mask_img_out, int f, int B, int C, int h, int w, void* stream);
/* The same three loops with PER-SAMPLE guidance scales (device arrays of B floats): the ensemble driver of the text wrappers
 * (SDW:146-165 generate, :189-204 encode -- the reference loops trial x encoder-scale x skip, then x decoder-scale, one chain at a
 * time, recomputing the conditioning and every context K/V projection per member).  Members that share a schedule are batched
 * along B: mode 1 = encode (x0, c_src, src_scales, noise -> z_out), 2 = decode (z_in, c_tgt, tgt_scales -> x_out), 3 = lock-step.
 * Both CFG segments run for every member; a member whose scale is 1 (0) takes eps-hat(c) (eps-hat(uc)) unchanged, exactly the
 * reference's single-forward branch (ddim.py:550-551), so each member equals its own cdx_latent_encode / _decode call.  The context
 * K / V projections are computed once per loop for the whole batch. */
int cdx_latent_loop_ens(cdx_net* unet, int mode, const float* x0, const float* c_src, const float* c_tgt, const float* uc,
                        int ctx_len, const float* src_scales, const float* tgt_scales, const cdx_ddim_coef* coef,
                        const float* t_host, int n_steps, int n_rec, const float* noise, float sqrt_a_T,
                        float sqrt_1ma_T, const float* z_in, int n_eps, const float* extra_noise, float* z_out,
                        float* x_out, int B, int C, int h, int w, void* stream);
/* ---- Directional-CLIP ranking and the evaluation metrics on the device (SURVEY 8f-3)
 * clip_preprocess: clean_clip.py:14-17 = Resize(size, bicubic) + CenterCrop(size) + Normalize(mean, std) on a float image batch in
 *   [0,1] (square inputs; torch bicubic, A = -0.75, align_corners = False, no antialias -- the tensor path of the torchvision release
 *   the reference pins).  img [B,3,R,R] -> out [B,3,size,size].
 * cdx_clip_image_features: CLIP.encode_image = ViT tower -> ln_post(class token) @ proj  -> [B, proj_dim] (net kind CDX_CLIP_VISION).
 * cdx_text_features: CLIP.encode_text = final-LN state at the EOT token (argmax of the ids) @ text_projection -> [B, proj_dim].
 * cdx_dclip_scores: clean_clip.py:24-39: L2-normalise the four feature sets, clip = <img, dec_text>, dclip = <unit(img - orig),
 *   unit(dec_text - enc_text)>.  All [B, D] device arrays; clip_out / dclip_out [B].
 * cdx_image_metrics: evaluation/translate_text.py:76-89 per image pair after clamp(0,1): PSNR = 10 log10(1 / mse) (100 when equal;
 *   evaluation/utils.py:60-66), L2 = sqrt(sum sq diff), SSIM of the x255 images (11x11 Gaussian sigma 1.5, valid region, per channel,
 *   mean of 3; evaluation/utils.py:35-57).  a, b [B,3,H,W] -> out [B,3] = {psnr, ssim, l2} (fp32). */
int cdx_clip_preprocess(cdx_engine* e, const float* img, int B, int R, int size, float* out, void* stream);
int cdx_clip_image_features(cdx_net* vision, const float* pixels, int B, float* out, void* stream);
int cdx_text_features(cdx_net* text, const int* ids_dev, int B, int L, float* out, void* stream);
int cdx_dclip_scores(cdx_engine* e, const float* img_f, const float* orig_f, const float* enc_f, const float* dec_f, int B, int D,
                     float* clip_out, float* dclip_out, void* stream);
int cdx_image_metrics(cdx_engine* e, const float* a, const float* b, int B, int H, int W, float* out, void* stream);
/* DDPMDDIMWrapper.encode loop (DW:483-521): coef/t_host have n_rec entries (loop order);
 * noise[0] = x_T draw, noise[1+i] = draw of iteration i; z_out [B, n_rec+1, C,R,R]. */
int cdx_pixel_encode(cdx_net* unet, const float* x0, const cdx_pixel_coef* coef, const float* t_host,
                     int n_rec, const float* noise, float sqrt_a_T, float sqrt_1ma_T, float* z_out,
                     int B, int C, int R, void* stream);
/* DDPMDDIMWrapper.generate main loop (DW:415-429): n_steps = n_eps + 1 (the last step's noise is
 * multiplied by 0 in the reference; pass it in last_noise or NULL). */
int cdx_pixel_decode(cdx_net* unet, const float* z, int n_eps, const cdx_pixel_coef* coef,
                     const float* t_host, int n_steps, const float* last_noise, float* x_out, int B,
                     int C, int R, void* stream);

/* ---- Unpaired translation in lock-step: the source model's DPM-Encoder chain and the target model's decode chain advance
 * together, so z is never written.  Replaces source.encode(image) -> z -> target(z) of UnsupervisedTranslation.forward
 * (unsupervised_translation.py:44-49).  The two schedules must be identical.  The two U-Net calls of a step are independent: when
 * the nets belong to different engines the target's call runs on the target engine's own non-blocking stream, forked from and
 * joined into `stream` once per step; nets of one engine run in order on `stream`.  Results are bit-identical to the two-phase
 * calls either way.
 *
 * cdx_pixel_cycle_lockstep: DDPMDDIMWrapper.encode (DW:472-523) under `src` with the first es_steps - 1 steps of .generate
 * (DW:392-429) under `tgt`, steps [i0, i1) of that loop.  Per step: both U-Net calls, then one fused kernel that draws the source
 * chain's x_{t-1} (DW:291-303), recovers the step's noise (DW:264-276) and advances the target chain with it (DW:202-222).
 * state [2, B,C,R,R] = (source x_t, target x_t), caller-owned, carried from call to call; coef / t_host: the loop's n_rec = es_steps-1
 * steps (loop order, indexed by i).  noise: this range's draws [i1 - i0, B,C,R,R], preceded by the x_T draw when i0 == 0 (which
 * also initialises state).  Walking [0, n_rec) in chunks keeps device memory at one chunk of noise.  The final target-only step
 * (t = 0, with the `last` draw) is cdx_pixel_decode on state[1] with n_eps = 0. */
int cdx_pixel_cycle_lockstep(cdx_net* src, cdx_net* tgt, const float* x0, const cdx_pixel_coef* coef, const float* t_host,
                             int i0, int i1, const float* noise, float sqrt_a_T, float sqrt_1ma_T, float* state, int B,
                             int C, int R, void* stream);
/* cdx_latent_cycle_pair: LatentDiffStochasticWrapper.encode under `src` and .generate's sampler under `tgt`
 * (latentdiff_stochastic_wrapper.py:253-311), unconditional U-Nets, scale 1.  noise [n_rec+1, B,C,h,w] as for cdx_latent_encode;
 * with n_rec < n_steps the target chain continues alone for the last n_steps - n_rec steps with extra_noise [n_steps-n_rec,
 * B,C,h,w] (ddim.py:640).  x_out [B,C,h,w]: the decoded latent, before any refine pass. */
int cdx_latent_cycle_pair(cdx_net* src, cdx_net* tgt, const float* x0, const cdx_ddim_coef* coef, const float* t_host,
                          int n_steps, int n_rec, const float* noise, float sqrt_a_T, float sqrt_1ma_T,
                          const float* extra_noise, float* x_out, int B, int C, int h, int w, void* stream);

/* ---- The ensemble search of the text wrappers in lock-step (SURVEY 8f-2).  Replaces encode's loop over trial x encoder scale x
 * skip (SDW:189-204), generate's loop over each z x decoder scale (SDW:146-165) and the Directional-CLIP argmax (SDW:219-249).
 *
 * cdx_latent_cycle_fan: n_src source chains -- _ddpm_ddim_encoding (ddim.py:450-501) of one (member, sample) pair under c_src[j] at
 * src_scales[j] -- each driving K target chains -- ddim_sampling_with_eps (ddim.py:395-448) under c_tgt[j] at tgt_scales[j*K + k] --
 * with the noise it recovers at each step (ddim.py:575-579, consumed at :603-646 in registers).  Every step is ONE U-Net call over
 * exactly the rows the chains need (a chain at scale 1 runs its cond row only, at scale 0 its uncond row only, else both,
 * ddim.py:550-559) and one fused elementwise launch.  The scales are host arrays: the row layout is derived from them, with no
 * device read.  Each chain computes what cdx_latent_encode / cdx_latent_decode compute for it, up to the summation order of
 * split-K GEMMs at a different batch size.  All steps recovered (eta > 0, white_box_steps > custom_steps - skip).
 *   x0 [n_src,C,h,w]; c_src, c_tgt, uc [n_src,L,D]; noise [n_steps+1, n_src,C,h,w] as for cdx_latent_encode;
 *   x_out [n_src*K, C,h,w]: target chain j*K + k's final latent; z_out optional [n_src, n_steps+1, C,h,w] (test hook).
 *
 * cdx_ensemble_select: running per-sample best over candidates that arrive in chunks, in any order.  Chunk entry c: score scores[c],
 * image images[c] [3,H,W], index cand_idx[c] in the reference's candidate order (column of the [B, n_total] score matrix of
 * SDW:225), sample sample_idx[c] in [0, B).  The state best_score [B], best_idx [B] (int64; < 0 = empty), best_img [B,3,H,W]
 * reproduces torch.argmax over the score matrix (larger wins; NaN beats any number; ties and NaNs go to the lower index); an
 * image is copied only when it becomes its sample's best.  score_mat [B, n_total] receives the chunk's scores. */
int cdx_latent_cycle_fan(cdx_net* unet, int n_src, int K, const float* x0, const float* c_src, const float* c_tgt,
                         const float* uc, int ctx_len, const float* src_scales_host, const float* tgt_scales_host,
                         const cdx_ddim_coef* coef, const float* t_host, int n_steps, const float* noise, float sqrt_a_T,
                         float sqrt_1ma_T, float* x_out, float* z_out, int C, int h, int w, void* stream);
/* cdx_latent_cycle_fan with mask [n_src,1,h,w]: source chain j's K target chains are blended with its x_{t-1} under mask[j] as in
 * cdx_cycle_lockstep_masked (m == 1 / m == 0 exact).  mask == NULL is cdx_latent_cycle_fan. */
int cdx_latent_cycle_fan_masked(cdx_net* unet, int n_src, int K, const float* x0, const float* c_src, const float* c_tgt,
                                const float* uc, int ctx_len, const float* src_scales_host, const float* tgt_scales_host,
                                const cdx_ddim_coef* coef, const float* t_host, int n_steps, const float* noise, float sqrt_a_T,
                                float sqrt_1ma_T, float* x_out, float* z_out, int C, int h, int w, void* stream,
                                const float* mask);
int cdx_ensemble_select(cdx_engine* e, int n, const float* scores, const int64_t* cand_idx, const int* sample_idx,
                        const float* images, float* best_score, int64_t* best_idx, float* best_img, float* score_mat, int B,
                        int n_total, int H, int W, void* stream);

/* ---------------------------------------------------------------- unit-test hooks ----------- */
/* Individual ops exported for per-op parity tests (tests/test_ops_gpu.py).  NHWC = [B,H,W,C]. */
int cdx_op_conv3x3(cdx_engine* e, const float* x_nhwc, const float* w_oihw, const float* bias,
                   float* y_nhwc, int B, int H, int W, int Cin, int Cout, int stride, int pad_lo,
                   int upsample, void* stream);
int cdx_op_linear(cdx_engine* e, const float* x, const float* w, const float* bias, float* y, int M,
                  int K, int N, void* stream);
int cdx_op_groupnorm(cdx_engine* e, const float* x_nhwc, const float* gamma, const float* beta,
                     float eps, int silu, float* y_nhwc, int B, int HW, int C, void* stream);
int cdx_op_layernorm(cdx_engine* e, const float* x, const float* gamma, const float* beta, float* y,
                     int M, int C, void* stream);
/* softmax(q k^T * scale) v with q [B,Nq,heads*d], k/v [B,Nk,heads*d] -> [B,Nq,heads*d] */
int cdx_op_attention(cdx_engine* e, const float* q, const float* k, const float* v, float* out, int B,
                     int Nq, int Nk, int heads, int d, float scale, void* stream);
/* cdx_op_attention with a row table: image b attends with image qk_rows[b]'s q and k and its own v (qk_rows: host [B], each in
 * [0, B)).  Fused kernel only: a shape or mode that would take another route is CDX_E_INVALID. */
int cdx_op_attention_rows(cdx_engine* e, const float* q, const float* k, const float* v, float* out, int B,
                          int Nq, int Nk, int heads, int d, float scale, const int* qk_rows, void* stream);
/* cdx_op_attention with a key / value row table: image b attends with its own q over image kv_rows[b]'s k and v (kv_rows: host
 * [B], each in [0, B)).  Fused kernel only, as cdx_op_attention_rows. */
int cdx_op_attention_kv_rows(cdx_engine* e, const float* q, const float* k, const float* v, float* out, int B,
                             int Nq, int Nk, int heads, int d, float scale, const int* kv_rows, void* stream);
/* The fused kernel's accumulating launch: out[r] += softmax(q[r] k[r]^T * scale) v[r] for each image r of acc_rows (host [n_acc],
 * each in [0, B)); the other images of out are not touched.  Fused kernel only, as cdx_op_attention_rows. */
int cdx_op_attention_accum(cdx_engine* e, const float* q, const float* k, const float* v, float* out, int B,
                           int Nq, int Nk, int heads, int d, float scale, const int* acc_rows, int n_acc, void* stream);
/* One attention with its operands prepared as the network executors prepare them after the projection
 * (tests/test_attention_bound_gpu.py).  C = heads * d, out [B*N, C].
 *   kind 0, self (the U-Net SpatialTransformer): qkv [B*N, 3C], one q|k|v projection with ONE range slot for all three operands
 *     (`slot` > 0: that value, else max |qkv|); K at the per-image key stride N, V^T padded per image.  TF32 planes (mma mode 3):
 *     q|k and V^T as the projection epilogues write them, on both of the network's V^T routes (N % 4 == 0 or not).
 *   kind 1, cross: q [B*N, C] (its own slot, `q_slot` > 0 or max |q|) over a context padded to ctx_lp >= L rows per image,
 *     kv [B*ctx_lp, 2C] one K | V projection with one slot (`slot` > 0 or max |kv|); keys >= L masked.
 *   kind 2, generic (text towers, VAE): q [B*N, C], k / v [B*L, C], two contractions around the row softmax; causal: query i sees
 *     keys j <= i.
 * qk_rows / kv_rows (host [B]) and acc_rows (host [n_acc], out += for those images only) as cdx_op_attention_rows / _kv_rows /
 * _accum; fused routes only.  plan_out (host int[7], optional): route (0 generic, 1 unfused tensor-core, 2 fused fp16 three-term,
 * 3 fused TF32, 4 fused one-term), the fused kernel's queries per CTA, ragged query tile, key split, ring depth, and the K and V^T
 * per-image key strides Nks, Nvs (zero where not fused). */
typedef struct cdx_attention_net_desc {
  int kind, causal;
  const float* qkv;
  const float* q; const float* kv; const float* k; const float* v;
  int B, N, L, ctx_lp, heads, d;
  float scale;
  const int* qk_rows; const int* kv_rows; const int* acc_rows; int n_acc;
  float slot, q_slot;
  float* out;
  /* kind 1 only, optional: LEDITS++'s probe on the operands the route multiplied (cdx_cycle_lockstep_semantic_attn), probe_map
   * [n_probe, N] <- for image probe_rows[i], sum over heads of sum over j = 1..probe_spans[i] of softmax_j (host lists) */
  const int* probe_rows; const int* probe_spans; int n_probe;
  float* probe_map;
} cdx_attention_net_desc;
int cdx_op_attention_net(cdx_engine* e, const cdx_attention_net_desc* desc, int* plan_out, void* stream);
/* cdx_op_attention_net with LocalBlend's weighted probe (cdx_cycle_lockstep_blend): probe_spans must be NULL and probe_weights (host
 * [n_probe, L], finite) gives probe_map[i] <- sum over heads of sum over j of probe_weights[i, j] softmax_j of image probe_rows[i]. */
int cdx_op_attention_net_weighted(cdx_engine* e, const cdx_attention_net_desc* desc, const float* probe_weights, int* plan_out,
                                  void* stream);
int cdx_op_nchw_to_nhwc(cdx_engine* e, const float* x, float* y, int B, int C, int HW, void* stream);
int cdx_op_nhwc_to_nchw(cdx_engine* e, const float* x, float* y, int B, int C, int HW, void* stream);
/* The normalisation kernels in the forms the network executors call them, with their side outputs (tests/test_norms_gpu.py).
 * cdx_op_groupnorm_ex: GroupNorm(32) over the channel concat [x1 | x2] (NHWC [B,HW,C1] and [B,HW,C2]; x2 NULL when C2 == 0), then
 *   optionally * (1 + scale) + shift (scale / shift [B, ld_ss] or NULL) and SiLU -> y [B,HW,C1+C2].  amax_out (optional, device
 *   float): the tracked range slot of y as the norm left it.  ab_out (optional, device [B, C1+C2, 2] floats): the (a, o) table
 *   the norm applies, y = silu?(x * a + o).
 * cdx_op_layernorm_ex: cdx_op_layernorm plus the tracked range slot of y in amax_out (optional, device float).
 * cdx_op_softmax_rows: in-place softmax over `rows` rows of length L (row stride ld); causal_nq > 0: row r sees only columns
 *   j <= r % causal_nq, the others become exactly 0.
 * cdx_op_produce_norm: a producer GEMM with its GroupNorm side outputs, then the GroupNorm that trusts them.  conv == 0: linear,
 *   x [B*H*W, Cin] @ w[Cout, Cin]^T + bias; conv == 1: stride-1 pad-1 conv3x3 of NHWC x [B,H,W,Cin] with w OIHW [Cout,Cin,3,3].
 *   y [B*H*W, Cout] receives the product, amax_out (device float) its range slot, stats_out (device [B, Cout, 2] doubles) its
 *   per-(image, channel) {sum, sum of squares} -- from the epilogue or, where it cannot, the standalone pass -- and yn (device
 *   [B*H*W, Cout]) GroupNorm(32)(y) with those statistics (eps, no SiLU).  *path_out (host): how the statistics were made --
 *   0 FFMA tiles + standalone pass, 1 fused into the tensor-core epilogue, 2 tensor cores + standalone pass, 3 split-K reduce +
 *   standalone pass. */
int cdx_op_groupnorm_ex(cdx_engine* e, const float* x1, int C1, const float* x2, int C2, const float* gamma, const float* beta,
                        float eps, int silu, const float* scale, const float* shift, int ld_ss, float* y, float* amax_out,
                        float* ab_out, int B, int HW, void* stream);
/* cdx_op_groupnorm_rows: cdx_op_groupnorm_ex's norm twice from ONE set of statistics: y [B,HW,C] plain, and y_rows [B,HW,C] with a
 *   row table (src_rows: host [B], each in [0, B)), image b of y_rows being image src_rows[b]'s norm -- bit for bit y[src_rows[b]].
 *   amax_out / amax_rows_out (optional, device floats): the tracked range slots of y and y_rows. */
int cdx_op_groupnorm_rows(cdx_engine* e, const float* x1, int C1, const float* x2, int C2, const float* gamma, const float* beta,
                          float eps, int silu, const float* scale, const float* shift, int ld_ss, const int* src_rows, float* y,
                          float* amax_out, float* y_rows, float* amax_rows_out, int B, int HW, void* stream);
int cdx_op_layernorm_ex(cdx_engine* e, const float* x, const float* gamma, const float* beta, float* y, float* amax_out, int M,
                        int C, void* stream);
int cdx_op_softmax_rows(cdx_engine* e, float* x, int64_t rows, int L, int ld, int causal_nq, void* stream);
int cdx_op_produce_norm(cdx_engine* e, const float* x, const float* w, const float* bias, int conv, int B, int H, int W, int Cin,
                        int Cout, const float* gamma, const float* beta, float eps, float* y, float* amax_out, double* stats_out,
                        float* yn, int* path_out, void* stream);

/* One contraction through the engine's production GEMM with every epilogue term the network executors use
 * (tests/test_gemm_epilogue_gpu.py):
 *   C[m, n] = alpha * sum_k A(m, k) W(n, k) (+ bias[n]) (+ rowvec[m / rows_per_batch, n]) (+ residual[m, n])
 * mode 0: dense; A(m, k) = A[m * lda + k] for k < C1, else A2[m * lda2 + k - C1] (K = C1 + C2); W [N][K] with row stride ldb
 *   (b_kn == 1: [K][N], FFMA only); batch * heads > 1: blockIdx.z-batched products with the s*_b / s*_h element strides (FFMA only).
 * mode 1: conv3x3 of NHWC A [B, Hin, Win, C1] (pixel stride lda) to an [B, Hout, Wout] grid, stride 1 or 2, low-side padding pad;
 *   w OIHW [N, C1, 3, 3], repacked here (K = 9 C1, ldb ignored).
 * Outputs, caller-allocated with caller strides: C [M, ldc] (geglu: [M, N/2] of value * gelu(gate) over [32 value | 32 gate] row
 * blocks of w; out_nchw: [M / rows_per_img, N, rows_per_img]); C_lo optional: C <- rn_tf32(result), C_lo <- rn_tf32(result - C);
 * Ct_hi / Ct_lo optional: columns n >= t_col0 go transposed as TF32 planes to Ct[(n - t_col0) * ldt + m]; c_amax (device float)
 * <- max(c_amax, max |stored C|); c_stats (device [M / rows_per_batch, N, 2] doubles) += per-(image, channel) {sum, sum sq}.
 * a_amax / a2_amax: tracked range slots of A / A2 (device floats), or NULL (measured here).  w_range > 0: the fp16 weight planes
 * take the exponent of max(w_range, max |w|), as in a net whose weight exponent comes from a larger weight elsewhere.
 * up (trailing field; 0 reads as 1): 2 folds a nearest-2x upsample of A into the conv3x3 gather (Hin, Win: the stored map; the FFMA
 * tiles run it, as the networks' Upsample convs on that path).
 * *plan_out (host): how the call ran -- bit 3 tensor cores; bits 0-2 range fused, statistics fused, split-K; bits 4-5 operand kind
 * (0 SS, 1 TS, 2 fp16 split, 3 one-term fp16); bits 8-15 tile width (FFMA: tile side); bits 16-23 split-K factor. */
typedef struct cdx_gemm_desc {
  int mode, M, N, K;
  const float* A; int lda; int C1;
  const float* A2; int lda2; int C2;
  int Hin, Win, Hout, Wout, stride, pad;
  const float* w; int ldb; int b_kn;
  const float* bias;
  const float* rowvec; int ld_rowvec; int rows_per_batch;
  const float* residual; int ldr;
  float alpha;
  int geglu;
  int out_nchw, rows_per_img;
  float* C; int ldc;
  float* C_lo;
  float* Ct_hi; float* Ct_lo; int t_col0; int64_t ldt;
  const float* a_amax; const float* a2_amax;
  float* c_amax; double* c_stats;
  float w_range;
  int batch, heads;
  int64_t sA_b, sA_h, sB_b, sB_h, sC_b, sC_h;
  int up;
} cdx_gemm_desc;
int cdx_op_gemm(cdx_engine* e, const cdx_gemm_desc* desc, int* plan_out, void* stream);

/* One launch of the latent loops' fused step kernels, the production latent_chains_init (stage 0), latent_chains_step (stage 1) or
 * semantic guidance's threshold stage (stage 2) every latent loop driver runs (tests/test_step_kernels_gpu.py).  n_src element groups of chw elements; group j has a source chain
 * (when src) and K target chains j*K + k.  chains: host [n_src + n_src*K] {row, row2, scale}, the source chains first, staged to the
 * device as the drivers stage theirs: `row` is the chain's cond row of xin / eout ([rows, chw]), `row2` its uncond row or -1; a
 * chain on two rows at scale 1 (0) reads its cond (uncond) row unchanged, else eps-hat = e(row2) + scale * (e(row) - e(row2)).
 * Every other field is a device pointer or a scalar with the meaning of the loop drivers' per-step arguments:
 *   init, src:    x_T = sa*x0 + s1*noise0 -> xt, z_out[j*z_stride + r] (optional), xin rows of every chain, yt; next == 1:
 *                 xn = posterior sample of (x0, x_T, noise_next) under cnext, next == 2: xn = x0
 *   init, no src: x_T = eps_in[j*eps_stride + r] -> yt and the target chains' xin rows
 *   step, src:    the noise recovered from e(source rows), xt, xn under c -> z_out (optional); xn -> the source chain's xin rows;
 *                 next == 1: xn2 = posterior sample of (x0, xn, noise_next) under cnext, next == 2: xn2 = x0
 *   step, no src: the noise <- eps_in[j*eps_stride + r]
 *   step:         each target chain from yt with that noise -> y_out and its xin rows; pred == 1: the output is v, converted with
 *                 (vsa, vs1); mask (src only) [n_src, hw], broadcast over the chw / hw channels: y_out = m*y + (1 - m)*xn
 *   sg_m > 0:     semantic guidance (cdx_cycle_lockstep_semantic).  sg_rows: host [n_src*K*sg_m], the concept rows of target chain
 *                 t at t*sg_m + k (staged as chains are); a target chain's uncond row is row2, or row when row2 < 0.  Stage 2 (the
 *                 threshold stage) writes sg_thr [n_src*K*sg_m*C] (C = chw / hw, plane (t*sg_m + k)*C + c) from eout under
 *                 sg_scale and sg_lambda; stage 1 then adds G to each target chain's eps-hat when sg_apply, from the concepts whose
 *                 bit is set in sg_active, updates the momentum sg_nu [n_src*K, chw] in place with (sg_mu, sg_beta, sg_beta1), and
 *                 writes the chain's next x_t to its concept rows too (as does stage 0).
 *   sg_mask > 0:  LEDITS++'s masks (cdx_cycle_lockstep_semantic_attn) instead of the per-channel thresholds: stage 2 writes sg_thr
 *                 [n_src*K*sg_m, 2], the threshold of the smoothed map and (sg_mask == 2) of the channel-summed |psi_k|; stage 1
 *                 keeps psi_k where both masks hold.
 * Row indices, counts, strides and the stage are checked on the host; buffer extents are the caller's. */
typedef struct cdx_latent_chain { int row, row2; float scale; } cdx_latent_chain;
typedef struct cdx_latent_chains_desc {
  int chw, n_src, K, rows;
  const cdx_latent_chain* chains;
  int src;
  const float* x0;
  const float* eout;
  cdx_ddim_coef c;
  const float* noise0; float sa, s1;
  float* xt; float* xn;
  int next;
  const float* noise_next; cdx_ddim_coef cnext;
  float* xn2;
  float* z_out; int64_t z_stride;
  const float* eps_in; int64_t eps_stride;
  float* yt; float* y_out;
  float* xin;
  int pred; float vsa, vs1;
  const float* mask; int hw;
  int sg_m;
  const int* sg_rows;
  float* sg_thr; float* sg_nu;
  float sg_scale[CDX_SEMANTIC_MAX]; float sg_lambda[CDX_SEMANTIC_MAX];
  unsigned sg_active; int sg_apply;
  float sg_mu, sg_beta, sg_beta1;
  const float* sg_map;          /* [n_src*K*sg_m, sg_gh*sg_gw]: the raw attention maps of the concept rows */
  int sg_mask;                  /* 0 SEGA's thresholds, 1 LEDITS++'s attention mask, 2 with its channel-summed mask */
  int sg_gh, sg_gw;             /* the map grid: h/4 x w/4 */
  int w;                        /* latent width (hw = h*w = 16*sg_gh*sg_gw) */
  /* edit-friendly inversion (cdx_cycle_lockstep_sampler): solver 0 the DDIM step on the posterior chain (next 0, 1, 2), 1 the DDIM
   * step on independent draws, 2 the SDE-DPM-Solver++ step under dc on independent draws (next 0, 2, 3).  next == 3: xn (stage 0) /
   * xn2 (stage 1) = qa*x0 + q1*noise_next.  solver 2, stage 1: d_src [n_src, chw] and d_tgt [n_src*K, chw] hold each chain's
   * previous x0-prediction, read when dc.order == 2 and overwritten with this step's. */
  int solver;
  cdx_dpm_coef dc;
  float* d_src; float* d_tgt;
  float qa, q1;
} cdx_latent_chains_desc;
int cdx_op_latent_chains(cdx_engine* e, const cdx_latent_chains_desc* desc, int stage, void* stream);
/* One launch of the two-model pixel loop's fused step (pixel_lockstep_step, which cdx_pixel_cycle_lockstep runs): xs / ys [B, chw]
 * (source x_t, target x_t) advanced in place from x0, the source and target U-Net outputs et_src [B, net_chw_src] / et_tgt
 * [B, net_chw_tgt] (first chw elements of each row used: the learned-variance split) and noise [B, chw]. */
int cdx_op_pixel_lockstep(cdx_engine* e, const float* x0, float* xs, float* ys, const float* et_src, const float* et_tgt,
                          const float* noise, const cdx_pixel_coef* c, int B, int chw, int net_chw_src, int net_chw_tgt,
                          void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CDX_H_ */
