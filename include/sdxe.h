/* sdxe — H100-native (sm_90a) denoising engine for AUTOMATIC1111/stable-diffusion-webui's hot path.
 *
 * C-ABI of libsdxe.so. Plain pointers and sizes only; every pointer named "device" is a CUDA device pointer on
 * the current device, `stream` is a cudaStream_t (0 = legacy default stream). No call synchronises the host
 * unless stated. All entry points return 0 on success and a negative code on failure; the message is available
 * from sdxe_last_error() (thread local). There is no CPU fallback: without a CUDA device every compute call fails.
 *
 * Reference interfaces replaced (paths relative to the reference tree, v1.10.1):
 *   sdxe_unet_forward   <- modules/sd_unet.py:75-77      SdUnet.forward(x, timesteps, context, *args, **kwargs)
 *                          called from modules/sd_unet.py:87-91 (UNetModel_forward)
 *   sdxe_attention      <- modules/sd_hijack_optimizations.py:535-537  F.scaled_dot_product_attention(q, k, v)
 *                          inside scaled_dot_product_attention_forward (:508-546) and sdp_attnblock_forward (:637-655)
 *   sdxe_vae_decode     <- modules/sd_samplers_common.py:58   model.decode_first_stage(z)  (AutoencoderKL.decode)
 *   sdxe_cfg_combine    <- modules/sd_samplers_cfg_denoiser.py:74-82   CFGDenoiser.combine_denoised
 *   sdxe_cfg_combine_affine
 *                       <- the same combine behind CFGDenoiserTimesteps (modules/sd_samplers_timesteps.py: raw eps,
 *                          get_pred_x0, CFG++'s last_noise_uncond) and CFGDenoiserLCM (modules/sd_samplers_lcm.py:50-63)
 *   sdxe_denoiser_in    <- k_diffusion/external.py DiscreteEpsDDPMDenoiser.forward (c_in scaling; its x + eps*c_out runs
 *                          inside sdxe_cfg_combine; un-vendored dependency pinned at modules/launch_utils.py:357)
 *   sdxe_euler_ancestral_step / sdxe_dpmpp_2m_step
 *                       <- k_diffusion/sampling.py sample_euler_ancestral / sample_dpmpp_2m loop bodies
 *                          (called through modules/sd_samplers_kdiffusion.py:230)
 *   sdxe_set_circular  <- modules/sd_hijack.py:311-318  StableDiffusionModelHijack.apply_circular(enable) (padding_mode
 *                          'circular' on every Conv2d of the model), driven by the Tiling setting at
 *                          modules/processing.py:879-880,895
 *   sdxe_create / sdxe_set_weight / sdxe_finalize
 *                       <- modules/sd_unet.py:63-72 SdUnetOption.create_unet() + SdUnet.activate(): the plugin owns
 *                          its weights (the stock UNet is moved to the CPU, modules/sd_unet.py:54)
 */
#ifndef SDXE_H_
#define SDXE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 16-bit storage / compute input format of activations and weights (accumulation is always fp32). */
enum sdxe_dtype { SDXE_F16 = 0, SDXE_BF16 = 1, SDXE_F32 = 2 };

enum sdxe_model_kind { SDXE_MODEL_UNET = 0, SDXE_MODEL_VAE_DECODER = 1, SDXE_MODEL_VAE_ENCODER = 2, SDXE_MODEL_CLIP_TEXT = 3 };

#define SDXE_MAX_LEVELS 8

/* Architecture description (ldm / sgm UNetModel constructor arguments; configs/v1-inference.yaml:29-44,
 * configs/sd_xl_inpaint.yaml:19-37) or the KL-VAE decoder (configs/v1-inference.yaml:46-65). */
typedef struct sdxe_config {
  int32_t kind;                 /* sdxe_model_kind */
  int32_t dtype;                /* SDXE_F16 or SDXE_BF16 */
  /* UNet */
  int32_t in_channels;          /* 4 */
  int32_t out_channels;         /* 4 */
  int32_t model_channels;       /* 320 */
  int32_t num_levels;           /* len(channel_mult) */
  int32_t channel_mult[SDXE_MAX_LEVELS];
  int32_t num_res_blocks;       /* 2 */
  int32_t transformer_depth[SDXE_MAX_LEVELS]; /* per level; 0 = no attention at that level */
  int32_t num_heads;            /* > 0: fixed head count (SD1.x: 8); else use num_head_channels */
  int32_t num_head_channels;    /* SDXL: 64 */
  int32_t context_dim;          /* 768 / 2048 */
  int32_t use_linear_in_transformer; /* 0: conv1x1 proj_in/out (SD1.x), 1: Linear (SDXL) */
  int32_t adm_in_channels;      /* 0 or 2816 (SDXL label_emb) */
  int32_t transformer_depth_middle; /* middle block depth (SD1.x: 1, SDXL: 10) */
  /* VAE decoder */
  int32_t vae_ch;               /* 128 */
  int32_t vae_z_channels;       /* 4 */
  int32_t vae_out_ch;           /* 3 */
  /* SDXE_MODEL_CLIP_TEXT (transformers CLIPTextModel / open_clip text tower; CLIP-L: 49408, 768, 3072, 12, 12, 77, 0) */
  int32_t clip_vocab;
  int32_t clip_hidden;
  int32_t clip_intermediate;
  int32_t clip_layers;
  int32_t clip_heads;
  int32_t clip_positions;
  int32_t clip_act;             /* 0 = quick_gelu (CLIP-L), 1 = erf GELU (OpenCLIP bigG) */
  int32_t reserved[1];
} sdxe_config;

typedef struct sdxe_engine sdxe_engine;

/* ---- lifecycle ------------------------------------------------------------------------------------------- */
const char* sdxe_last_error(void);
int sdxe_version(void);
/* Number of kernels launched by this library so far in this process (monotonic; for bench `gpu_launches`). */
int64_t sdxe_launch_count(void);

int sdxe_create(const sdxe_config* cfg, sdxe_engine** out);
void sdxe_destroy(sdxe_engine* e);
/* Copy one state-dict tensor (ldm key layout, e.g. "input_blocks.1.0.in_layers.2.weight", VAE:
 * "decoder.mid.attn_1.q.weight", "post_quant_conv.weight") into the engine. `data` is a contiguous device or
 * host pointer of element type `dtype`; the engine converts and repacks at sdxe_finalize. */
int sdxe_set_weight(sdxe_engine* e, const char* key, const void* data, int dtype, int ndim, const int64_t* shape);
/* Number of parameters ingested so far (for the parameter-count known-answer test). */
int64_t sdxe_param_count(const sdxe_engine* e);
/* Verify that every key the architecture needs is present, repack into kernel layouts. Synchronises. */
int sdxe_finalize(sdxe_engine* e);
/* Bytes of the packed weight blob and its device address (for the one NCCL broadcast at load). */
int sdxe_weight_blob(sdxe_engine* e, void** device_ptr, int64_t* bytes);

/* ---- hot path -------------------------------------------------------------------------------------------- */
/* eps = UNet(x, t, context[, y]).  x, out: [n,4,h,w] NCHW; t: [n]; ctx: [n, ctx_len, context_dim];
 * y: [n, adm_in_channels] or NULL. io_dtype is the element type of x/t/ctx/y/out (SDXE_F16/BF16/F32). */
int sdxe_unet_forward(sdxe_engine* e, const void* x, const void* t, const void* ctx, const void* y, void* out,
                      int n, int h, int w, int ctx_len, int io_dtype, void* stream);
/* image = AutoencoderKL.decode(z): z [n, 4, h, w] (already divided by scale_factor) -> [n, 3, 8h, 8w] NCHW. */
int sdxe_vae_decode(sdxe_engine* e, const void* z, void* out, int n, int h, int w, int io_dtype, void* stream);
/* moments = quant_conv(AutoencoderKL.encoder(x)): x [n, 3, H, W] in [-1, 1] NCHW -> [n, 2*z_channels, H/8, W/8]
 * (mean | logvar, the input of DiagonalGaussianDistribution). Replaces model.encode_first_stage(image) in
 * modules/sd_samplers_common.py:87-112 (images_tensor_to_samples), used by img2img init (modules/processing.py:1602-1757).
 * Engine kind SDXE_MODEL_VAE_ENCODER, weights "encoder.*" and "quant_conv.*". H, W multiples of 2^(num_levels-1) (8). */
int sdxe_vae_encode(sdxe_engine* e, const void* x, void* out, int n, int h, int w, int io_dtype, void* stream);

/* CLIP text transformer (row N4): hidden_states[layer] of the causal text transformer, optionally through final_layer_norm
 * — what `encode_with_transformers` needs (modules/sd_hijack_clip.py:351-360: last_hidden_state, or hidden_states[-skip]
 * + final_layer_norm for CLIP_stop_at_last_layers; sgm for SDXL: hidden_states[11] / "penultimate", no final norm).
 * tokens: int32 [n, T] (device), T <= clip_positions; layer in 1 .. clip_layers counts transformer layers applied;
 * out: [n, T, clip_hidden] in io_dtype (the engine's 16-bit type or SDXE_F32). Engine kind SDXE_MODEL_CLIP_TEXT, weights
 * with the Hugging Face names "text_model.embeddings.token_embedding.weight", "text_model.encoder.layers.N.*", ... */
int sdxe_clip_forward(sdxe_engine* e, const int32_t* tokens, void* out, int n, int T, int layer, int final_norm, int io_dtype,
                      void* stream);

/* The same with textual-inversion "fixes" (modules/sd_hijack.py:340-366 EmbeddingsWithFixes.forward, fed by
 * modules/sd_hijack_clip.py:162-176, 219): before the position embedding is added, row fix_rows[i] (= batch * T + position) of
 * the token embedding is replaced by the learned vector fix_vecs[i, :] (engine 16-bit type, [n_fix, clip_hidden]); when a row
 * is named more than once the last entry wins (fixes apply in order). fix_rows / fix_vecs are device pointers; n_fix = 0 is
 * sdxe_clip_forward. */
int sdxe_clip_forward_fixes(sdxe_engine* e, const int32_t* tokens, void* out, int n, int T, int layer, int final_norm, int io_dtype,
                            const int32_t* fix_rows, const void* fix_vecs, int n_fix, void* stream);

/* Cross-attention K / V cache. The context of a job does not change between sampler steps (CFGDenoiser.forward re-sends the
 * same cond_in every step, modules/sd_samplers_cfg_denoiser.py:236-249), but its k | v projections (one GEMM over all
 * transformer blocks) would be recomputed by every sdxe_unet_forward call. A non-zero `key` set before a call promises that
 * whatever context is passed under this key has identical contents each time; calls whose plan last projected the context
 * under the same key skip the cast + GEMM. key = 0 (default) disables the cache. */
int sdxe_unet_set_context_key(sdxe_engine* e, int64_t key);

/* Hypertile for the next sdxe_unet_forward only (extensions-builtin/hypertile/hypertile.py:269-313): one row
 * (h', w', nh, nw, max_tiles) of int32 per attn1 (self-attention) layer, in execution order (input blocks, middle block,
 * output blocks; transformer blocks in order). A row with max_tiles > 0 tiles that layer: its h' * w' tokens, taken as
 * a row-major h' x w' grid, are regrouped `b (nh h nw w) c -> (b nh nw) (h w) c` and attention runs inside each of the
 * nh * nw tiles (nh | h', nw | w', nh * nw <= max_tiles). max_tiles = 0 leaves the layer untiled (nh = nw = 1).
 * The plan is keyed on (h', w', max_tiles) of every row; (nh, nw) change per call without a new plan or graph.
 * n_layers = 0: no Hypertile (also the state after every forward). */
int sdxe_unet_set_hypertile(sdxe_engine* e, const int32_t* layers, int n_layers);

/* Tiling (seamless images): with enable != 0, every 3x3 convolution with padding 1 of a UNet, VAE decoder or VAE encoder
 * engine pads circularly, as torch's padding_mode='circular' (F.pad(x, (1,1,1,1), mode='circular'), then the convolution
 * without padding): out-of-range taps wrap around the image instead of reading zeros. 1x1 convolutions and the VAE
 * encoder's stride-2 Downsample (padding 0 after an explicit constant pad) are unchanged. Sticky until changed. The
 * setting is part of the plan key: enabling builds (once) a plan of its own per shape, disabling returns to the plan
 * without it. Fails for CLIP engines. */
int sdxe_set_circular(sdxe_engine* e, int enable);

/* Execution-plan cache. A plan (buffers from the engine's pool, tensor maps, one CUDA graph) is built per input shape
 * (n, h, w, ctx_len) on first use and replayed afterwards; at most `max_plans` (default 8) are kept, least recently used
 * evicted, and after an eviction free pool memory beyond `pool_limit_mb` (default 6144; < 0 = keep) returns to the
 * driver. An allocation failure during a plan build drops every cached plan and retries once; if that fails the call
 * returns -1 ("out of device memory ...") with nothing leaked. All calls on one engine must use one stream at a time. */
int sdxe_set_plan_cache(sdxe_engine* e, int max_plans, int64_t pool_limit_mb);
/* bytes held by the engine's activation pool (cached plans + free list); *n_plans = cached plans. */
int64_t sdxe_pool_bytes(sdxe_engine* e, int64_t* n_plans);

/* Per-kernel-class timing: while enabled, forward / decode calls run their plan eagerly with a CUDA event pair
 * around every launch on the launching stream. kind: 0 GEMM (wgmma), 1 conv3x3 implicit GEMM (wgmma),
 * 2 attention, 3 GroupNorm, 4 LayerNorm, 5 other. flops / bytes are ALGORITHMIC totals of the timed launches. */
int sdxe_profile(sdxe_engine* e, int enable);
int sdxe_profile_read(sdxe_engine* e, int kind, double* ms, double* flops, double* bytes, int64_t* launches);

/* out[b, q, h*D + j] = softmax(q k^T * scale) v.  q: [B,H,Nq,D], k,v: [B,H,Nk,D] contiguous, 16-bit `dtype`;
 * out: [B, Nq, H*D]. D multiple of 8, D <= 512. */
int sdxe_attention(const void* q, const void* k, const void* v, void* out, int B, int H, int Nq, int Nk, int D,
                   float scale, int dtype, void* stream);
/* Hypertile self-attention of one layer: qkv [B, hp*wp, 3*H*D] (q | k | v, heads contiguous inside each), the tokens a
 * row-major hp x wp grid cut into nh x nw tiles with (nh, nw) = draw[0], draw[1] (device int32[2], nh | hp, nw | wp,
 * nh * nw <= max_tiles). qkv_tiled: scratch of qkv's size (the tile-major copy). out: [B, hp*wp, H*D], each token's
 * attention over the keys of its own tile at the token's own row. */
int sdxe_hypertile_attention(const void* qkv, void* qkv_tiled, const int32_t* draw, void* out, int B, int H, int hp,
                             int wp, int D, int max_tiles, float scale, int dtype, void* stream);

/* out[M,N] = A[M,K] W[N,K]^T (+bias[N] fp32) (+residual[M,N]); 16-bit `dtype`; K % 8 == 0, N % 8 == 0.
 * flags: bit0 = GEGLU epilogue (W/bias rows = [value ; gate], out is [M, N/2]). */
int sdxe_gemm(const void* A, const void* W, void* out, int M, int N, int K, const float* bias, const void* residual,
              int flags, int dtype, void* stream);
/* 3x3 stride-1 pad-1 convolution, NHWC activations, weight [Cout, 3, 3, Cin] (tap-major), Cin % 64 == 0. */
int sdxe_conv3x3_nhwc(const void* x, const void* w, void* out, int n, int h, int wd, int cin, int cout,
                      const float* bias, int dtype, void* stream);
/* GroupNorm(32 groups) [+ SiLU] over NHWC 16-bit activations, fp32 statistics. */
int sdxe_group_norm_nhwc(const void* x, const float* gamma, const float* beta, void* out, int n, int hw, int c,
                         int groups, float eps, int silu, int dtype, void* stream);
/* LayerNorm over the last dim of [rows, c]. */
int sdxe_layer_norm(const void* x, const float* gamma, const float* beta, void* out, int rows, int c, float eps,
                    int dtype, void* stream);

/* ---- sampler-step elementwise fusions (fp32 latents [n,4,h,w]) -------------------------------------------- */
/* x_in[r] = x[src[r]] * c_in[r] cast to 16-bit: builds the 2B CFG batch (sd_samplers_cfg_denoiser.py:203) and applies
 * CompVisDenoiser's c_in in one pass. src: int32[rows], c_in: fp32[rows] (device). */
int sdxe_denoiser_in(const float* x, const int32_t* src, const float* c_in, void* x_in, int rows, int64_t elems,
                     int out_dtype, void* stream);
/* denoised[i] = u + sum_k w_k*s*(c_k - u) with c = x_in + eps*c_out (k-diffusion x + eps * (-sigma)), for the
 * common one-cond-per-image case: rows [0,B) cond, [B,2B) uncond. eps is 16-bit or fp32. */
int sdxe_cfg_combine(const float* x, const void* eps, const float* sigma, float cond_scale, float* denoised, int B,
                     int64_t elems, int eps_dtype, void* stream);
/* General form of the same combine (AND-composed prompts, per-cond weights): image b owns eps rows
 * cond_rows[row_ptr[b] .. row_ptr[b+1]) with weights cond_w[k] (= weight_k * cond_scale) and uncond row uncond_rows[b]
 * (when the uncond pass is skipped, s_min_uncond, the reference substitutes the image's first cond row, :272-275):
 * denoised[b] = den_u + sum_k cond_w[k] * (den_k - den_u), den_r = x[b] + eps[r] * (-sigma[b]).
 * row_ptr: int32[B+1], cond_rows: int32[nnz], cond_w: fp32[nnz], uncond_rows: int32[B] (device). */
int sdxe_cfg_combine_multi(const float* x, const void* eps, const float* sigma, const int32_t* row_ptr,
                           const int32_t* cond_rows, const float* cond_w, const int32_t* uncond_rows, float* denoised,
                           int B, int64_t elems, int eps_dtype, void* stream);
/* Combine for denoisers whose per-row output is affine in (x[b], eps[r]) with per-image coefficients (DDIM / PLMS / UniPC:
 * raw eps, cx = 0, ce = 1; LCM: c_out'(x - sigma eps) + c_skip' x). With the CSR rows of sdxe_cfg_combine_multi:
 *   out[b] = cx[b] x[b] + ce[b] (e_u + sum_k cond_w[k] (e_k - e_u)),  e_u = eps[uncond_rows[b]].
 * Optional, in the same pass (NULL to skip): x0_out[b] = x0_coef[2b] x[b] + x0_coef[2b+1] eps[cond_rows[row_ptr[b]]]
 * (the timestep samplers' pred_x0 of the first cond, returned by an interrupted job) and uncond_out[b] = e_u as fp32
 * (DDIM CFG++). cx, ce: fp32[B], x0_coef: fp32[2B] (device). eps is 16-bit or fp32. */
int sdxe_cfg_combine_affine(const float* x, const void* eps, const int32_t* row_ptr, const int32_t* cond_rows,
                            const float* cond_w, const int32_t* uncond_rows, const float* cx, const float* ce, float* out,
                            const float* x0_coef, float* x0_out, float* uncond_out, int B, int64_t elems, int eps_dtype,
                            void* stream);
/* out = c0 p0 + c1 p1 + c2 p2 + c3 p3 over fp32 latents (p1..p3 may be NULL, out may alias an input): the step update of
 * the remaining k-diffusion samplers (Euler, Heun, DPM2, DPM2 a, DPM++ 2S a, LMS, Restart; selected at
 * modules/sd_samplers_kdiffusion.py:11-27), of DDIM / DDIM CFG++ / PLMS / UniPC / LCM, with the step's scalars computed on
 * the host. */
int sdxe_lincomb(float* out, const float* p0, float c0, const float* p1, float c1, const float* p2, float c2, const float* p3,
                 float c3, int64_t total, void* stream);
/* x <- x + (x - denoised)/sigma * (sigma_down - sigma) + noise * sigma_up  (noise may be NULL when sigma_up == 0). */
int sdxe_euler_ancestral_step(float* x, const float* denoised, const float* noise, float sigma, float sigma_down,
                              float sigma_up, int64_t total, void* stream);
/* x <- (sigma_next/sigma) x - expm1(-h) * (c0*denoised + c1*old_denoised)  (old may be NULL when c1 == 0). */
int sdxe_dpmpp_2m_step(float* x, const float* denoised, const float* old_denoised, float ratio, float neg_expm1,
                       float c0, float c1, int64_t total, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SDXE_H_ */
