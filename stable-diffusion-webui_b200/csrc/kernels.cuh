// Bandwidth-bound kernels of the engine (norms, layout changes, embeddings, sampler-step fusions, weight repack).
#pragma once
#include "common.cuh"

namespace sdxe {

// ---- normalisation ---------------------------------------------------------------------------------------
// GroupNorm over NHWC 16-bit activations; the input may be the channel-concatenation of two tensors
// (x1: [n,hw,c1], x2: [n,hw,c2] or null) — this is how the UNet's skip-concat is consumed without a torch.cat.
// scratch: fp32 [group_norm_scratch_floats(n, groups)] (block partials + final mean / rstd); no atomics, deterministic.
size_t group_norm_scratch_floats(int n, int groups);
int kernels_init();  // one-time kernel attribute setup (before any stream capture)
int group_norm_launch(const void* x1, int c1, const void* x2, int c2, const float* gamma, const float* beta, void* out,
                      float* scratch, int n, int hw, int groups, float eps, bool silu, bool bf16, cudaStream_t s);
int layer_norm_launch(const void* x, const float* gamma, const float* beta, void* out, int rows, int c, float eps,
                      bool bf16, cudaStream_t s);

// ---- layout / gather ---------------------------------------------------------------------------------------
// 3x3 im2col of NHWC 16-bit input -> A[n*Ho*Wo, kpad], column = tap*C + c, zero padded. pad_lo = top/left padding.
// circular: taps outside the image wrap around (index mod H, W) instead of reading zero (pad_lo = 1 only).
int im2col3x3_launch(const void* x, void* A, int n, int H, int W, int C, int Ho, int Wo, int stride, int pad_lo,
                     int kpad, bool circular, bool bf16, cudaStream_t s);
// same, stride 1 pad 1, reading an NCHW tensor of `io_dtype` (the UNet / VAE entry convolution on the caller's latent).
int im2col3x3_nchw_launch(const void* x, int io_dtype, void* A, int n, int C, int H, int W, int kpad, bool circular,
                          bool bf16, cudaStream_t s);
// [n, H, W, C] -> [n, H+2, W+2, C] with the wrapped rows, columns and corners of circular padding (C % 8 == 0): the
// operand of the implicit convolution under circular padding, which then reads every tap in bounds.
int circular_pad_nhwc_launch(const void* x, void* out, int n, int H, int W, int C, cudaStream_t s);
int upsample2x_launch(const void* x, void* out, int n, int H, int W, int C, cudaStream_t s);
// out[n, c, h, w] (io_dtype) = in[(n*hw + p) * ld + c], c < C
int nhwc_to_nchw_launch(const void* in, int ld, void* out, int io_dtype, int n, int C, int hw, bool bf16, cudaStream_t s);
// generic cast of a contiguous [rows, cols] (src dtype) into 16-bit [rows, ldo] (pad columns untouched)
int cast_rows_launch(const void* src, int src_dtype, void* dst, int64_t rows, int cols, int ldo, bool bf16, cudaStream_t s);

// ---- embeddings --------------------------------------------------------------------------------------------
// modules/sd_hijack_unet.py:58-78: emb[m, :] = [cos(t*f) , sin(t*f)], rounded through the 16-bit type; fp32 out.
int timestep_embedding_launch(const void* t, int t_dtype, float* out, int m, int dim, bool bf16, cudaStream_t s);
// out[m, n] = act(round16(sum_k in[m,k] * W[n,k] + b[n]) (+ add[m,n])), act = SiLU (rounded) if silu_out; in/out fp32; W 16-bit [N,K]
int skinny_linear_launch(const float* in, int ldi, const void* W, const float* b, const float* add, float* out, int ldo,
                         int M, int N, int K, bool silu_out, bool bf16, cudaStream_t s);
int lincomb_launch(float* out, const float* p0, float c0, const float* p1, float c1, const float* p2, float c2, const float* p3, float c3,
                   int64_t total, cudaStream_t s);
// CLIP text encoder pieces (kernels.cu)
int clip_embed_launch(const int32_t* ids, const void* tok, const void* pos, void* x, float2* stat, int M, int T, int C, int vocab,
                      bool bf16, cudaStream_t s);
int clip_fix_launch(const int32_t* rows, const void* vec, const void* pos, void* x, float2* stat, int n_fix, int M, int T, int C,
                    bool bf16, cudaStream_t s);
int causal_attn_small_launch(const void* qkv, void* out, int B, int T, int H, int d, float scale, bool bf16, cudaStream_t s);
int act_inplace_launch(void* x, int64_t n, int mode, bool bf16, cudaStream_t s);
int cast_to_f32_launch(const void* src, int src_dtype, float* dst, int64_t n, bool round16, bool bf16, cudaStream_t s);

// ---- weight repack (run once at finalize) -------------------------------------------------------------------
enum : int { PACK_PLAIN = 0, PACK_CONV3 = 1, PACK_GEGLU = 2 };
// PLAIN: dst[r, c] = src[r, c] (cols -> ld).  CONV3: src [Cout, Cin, 3, 3] -> dst[Cout, tap*Cin + c].
// GEGLU: PLAIN with rows permuted so that every `tile` rows hold tile/2 value rows then the matching gate rows.
int pack_weight_launch(const void* src, int src_dtype, void* dst, int mode, int rows, int cols, int ld, int tile,
                       bool bf16, cudaStream_t s);
// fold a LayerNorm's affine into the packed weight that consumes its output (see gemm.cuh); bias must be allocated (zeroed if the
// layer has none), c1 receives the row sums of the folded weight
int ln_fold_launch(void* w, int rows, int K, int ld, const float* gamma, const float* beta, float* bias, float* c1, bool bf16,
                   cudaStream_t s);
int pack_vector_launch(const void* src, int src_dtype, float* dst, int n, int geglu_tile, bool round16, bool bf16,
                       cudaStream_t s);

// ---- sampler-step fusions -----------------------------------------------------------------------------------
int denoiser_in_launch(const float* x, const int32_t* src, const float* c_in, void* x_in, int rows, int64_t elems,
                       int out_dtype, cudaStream_t s);
int cfg_combine_launch(const float* x, const void* eps, const float* sigma, float cond_scale, float* denoised, int B,
                       int64_t elems, int eps_dtype, cudaStream_t s);
int cfg_combine_multi_launch(const float* x, const void* eps, const float* sigma, const int32_t* row_ptr,
                             const int32_t* cond_rows, const float* cond_w, const int32_t* uncond_rows, float* denoised,
                             int B, int64_t elems, int eps_dtype, cudaStream_t s);
int cfg_combine_affine_launch(const float* x, const void* eps, const int32_t* row_ptr, const int32_t* cond_rows,
                              const float* cond_w, const int32_t* uncond_rows, const float* cx, const float* ce, float* out,
                              const float* x0_coef, float* x0_out, float* uncond_out, int B, int64_t elems, int eps_dtype,
                              cudaStream_t s);
int euler_a_step_launch(float* x, const float* den, const float* noise, float sigma, float sigma_down, float sigma_up,
                        int64_t total, cudaStream_t s);
int dpmpp_2m_step_launch(float* x, const float* den, const float* old, float ratio, float neg_expm1, float c0, float c1,
                         int64_t total, cudaStream_t s);

}  // namespace sdxe
