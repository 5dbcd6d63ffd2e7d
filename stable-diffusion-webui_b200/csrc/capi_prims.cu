// C-ABI entry points for the stand-alone primitives (include/sdxe.h): attention, GEMM, conv3x3, norms and the
// sampler-step fusions. The model-level entry points live in engine.cu.
#include "../../include/sdxe.h"
#include "attention.cuh"
#include "gemm.cuh"
#include "kernels.cuh"
#include <cmath>
#include <cstring>
#include <vector>

using namespace sdxe;

static inline bool is16(int dt) { return dt == SDXE_F16 || dt == SDXE_BF16; }

extern "C" {

const char* sdxe_last_error(void) { return last_error(); }
int sdxe_version(void) { return 1; }
int64_t sdxe_launch_count(void) { return launch_count(); }

int sdxe_attention(const void* q, const void* k, const void* v, void* out, int B, int H, int Nq, int Nk, int D,
                   float scale, int dtype, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (!is16(dtype) || D % 8 != 0 || D > 512 || D <= 0) { set_last_error(__FILE__, __LINE__, "sdxe_attention: dtype/D"); return -2; }
  // [B, H, N, D] contiguous; heads are interleaved in the output as h*D + j
  const int64_t sq = (int64_t)Nq * D, sk = (int64_t)Nk * D;
  std::vector<AttnArgs> passes;
  if (attention_args(passes, {q, D, sq, H * sq}, {k, D, sk, H * sk}, {v, D, sk, H * sk}, B, H, Nq, Nk, D, D, scale, out,
                     H * D, D))
    return -1;
  for (const AttnArgs& a : passes)
    if (int rc = attention_launch(a, dtype == SDXE_BF16, stream)) return rc;
  return 0;
}

int sdxe_hypertile_attention(const void* qkv, void* qkv_tiled, const int32_t* draw, void* out, int B, int H, int hp,
                             int wp, int D, int max_tiles, float scale, int dtype, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (!is16(dtype) || D % 8 != 0 || D > 512 || D <= 0 || B < 1 || H < 1 || hp < 1 || wp < 1 || max_tiles < 1 || !draw) {
    set_last_error(__FILE__, __LINE__, "sdxe_hypertile_attention: bad argument");
    return -2;
  }
  const int N = hp * wp, ld = 3 * H * D;
  std::vector<AttnArgs> passes;
  const char* t = (const char*)qkv_tiled;
  if (attention_args(passes, {t, ld, D, (int64_t)N * ld}, {t + 2 * H * D, ld, D, (int64_t)N * ld},
                     {t + 4 * H * D, ld, D, (int64_t)N * ld}, B, H, N, N, D, D, scale, out, H * D, D))
    return -1;
  if (int rc = hypertile_gather_launch(qkv, qkv_tiled, B, hp, wp, ld, draw, stream)) return rc;
  for (AttnArgs& a : passes) {
    a.seg = draw; a.seg_h = hp; a.seg_w = wp; a.seg_max_tiles = max_tiles;
    if (int rc = attention_launch(a, dtype == SDXE_BF16, stream)) return rc;
  }
  return 0;
}

int sdxe_gemm(const void* A, const void* W, void* out, int M, int N, int K, const float* bias, const void* residual,
              int flags, int dtype, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (!is16(dtype) || K % 8 || N % 8) { set_last_error(__FILE__, __LINE__, "sdxe_gemm: dtype / alignment"); return -2; }
  const bool bf16 = dtype == SDXE_BF16;
  const bool geglu = flags & 1;
  void* scratch = nullptr;
  GemmW w;
  w.w = W; w.rows = N; w.ld = K; w.N = N; w.K = K; w.bias = bias;
  if (geglu) {
    // value / gate rows interleaved per tile, so that both land in the same accumulator tile (packed below, once the
    // tile width is chosen)
    SDXE_CUDA_CHECK(cudaMallocAsync(&scratch, (size_t)N * K * 2 + (size_t)N * 4, stream));
    w.w = scratch;
    if (bias) w.bias = (const float*)((char*)scratch + (size_t)N * K * 2);
  }
  GemmEpi o;
  o.epi = geglu ? EPI_GEGLU : EPI_PLAIN;
  o.residual = residual;
  o.ldr = N;
  GemmArgs a;
  int rc = gemm_args(a, GemmA::matrix(A, M, K), w, out, o, flags >> 8);  // flags >> 8: test hook forcing the tile width
  if (rc == 0 && geglu) {
    rc = pack_weight_launch(W, dtype, scratch, PACK_GEGLU, N, K, K, a.BN, bf16, stream);
    if (rc == 0 && bias) rc = pack_vector_launch(bias, SDXE_F32, (float*)w.bias, N, a.BN, false, bf16, stream);
  }
  if (rc == 0) rc = gemm_launch(a, bf16, stream);
  if (scratch) cudaFreeAsync(scratch, stream);
  return rc;
}

int sdxe_conv3x3_nhwc(const void* x, const void* w, void* out, int n, int h, int wd, int cin, int cout,
                      const float* bias, int dtype, void* stream_) {
  int bw, bh, bn;
  if (!is16(dtype) || cin % 64 || cout % 8) { set_last_error(__FILE__, __LINE__, "sdxe_conv3x3: alignment"); return -2; }
  if (!conv_tile_shape(h, wd, &bw, &bh, &bn)) { set_last_error(__FILE__, __LINE__, "sdxe_conv3x3: unsupported H x W tile"); return -2; }
  GemmW W;
  W.w = w; W.rows = cout; W.ld = 9 * cin; W.N = cout; W.K = 9 * cin; W.bias = bias;
  GemmArgs a;
  if (gemm_args(a, GemmA::nhwc(x, n, h, wd, cin), W, out, GemmEpi())) return -1;
  return gemm_launch(a, dtype == SDXE_BF16, (cudaStream_t)stream_);
}

int sdxe_group_norm_nhwc(const void* x, const float* gamma, const float* beta, void* out, int n, int hw, int c,
                         int groups, float eps, int silu, int dtype, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (!is16(dtype)) { set_last_error(__FILE__, __LINE__, "group_norm: dtype"); return -2; }
  float* stats = nullptr;
  SDXE_CUDA_CHECK(cudaMallocAsync((void**)&stats, sizeof(float) * group_norm_scratch_floats(n, groups), stream));
  int rc = group_norm_launch(x, c, nullptr, 0, gamma, beta, out, stats, n, hw, groups, eps, silu != 0, dtype == SDXE_BF16, stream);
  cudaFreeAsync(stats, stream);
  return rc;
}

int sdxe_layer_norm(const void* x, const float* gamma, const float* beta, void* out, int rows, int c, float eps,
                    int dtype, void* stream) {
  if (!is16(dtype)) { set_last_error(__FILE__, __LINE__, "layer_norm: dtype"); return -2; }
  return layer_norm_launch(x, gamma, beta, out, rows, c, eps, dtype == SDXE_BF16, (cudaStream_t)stream);
}

int sdxe_denoiser_in(const float* x, const int32_t* src, const float* c_in, void* x_in, int rows, int64_t elems,
                     int out_dtype, void* stream) {
  return denoiser_in_launch(x, src, c_in, x_in, rows, elems, out_dtype, (cudaStream_t)stream);
}
int sdxe_cfg_combine(const float* x, const void* eps, const float* sigma, float cond_scale, float* denoised, int B,
                     int64_t elems, int eps_dtype, void* stream) {
  return cfg_combine_launch(x, eps, sigma, cond_scale, denoised, B, elems, eps_dtype, (cudaStream_t)stream);
}
int sdxe_lincomb(float* out, const float* p0, float c0, const float* p1, float c1, const float* p2, float c2, const float* p3,
                 float c3, int64_t total, void* stream) {
  if (!out || !p0 || total < 0) { set_last_error(__FILE__, __LINE__, "sdxe_lincomb: bad argument"); return -1; }
  return lincomb_launch(out, p0, c0, p1, c1, p2, c2, p3, c3, total, (cudaStream_t)stream);
}
int sdxe_cfg_combine_multi(const float* x, const void* eps, const float* sigma, const int32_t* row_ptr,
                           const int32_t* cond_rows, const float* cond_w, const int32_t* uncond_rows, float* denoised,
                           int B, int64_t elems, int eps_dtype, void* stream) {
  return cfg_combine_multi_launch(x, eps, sigma, row_ptr, cond_rows, cond_w, uncond_rows, denoised, B, elems, eps_dtype,
                                  (cudaStream_t)stream);
}
int sdxe_cfg_combine_affine(const float* x, const void* eps, const int32_t* row_ptr, const int32_t* cond_rows,
                            const float* cond_w, const int32_t* uncond_rows, const float* cx, const float* ce, float* out,
                            const float* x0_coef, float* x0_out, float* uncond_out, int B, int64_t elems, int eps_dtype,
                            void* stream) {
  if (!x || !eps || !row_ptr || !cond_rows || !cond_w || !uncond_rows || !cx || !ce || !out || (x0_out && !x0_coef) ||
      B < 0 || elems < 0 || (eps_dtype != SDXE_F32 && !is16(eps_dtype))) {
    set_last_error(__FILE__, __LINE__, "sdxe_cfg_combine_affine: bad argument");
    return -1;
  }
  return cfg_combine_affine_launch(x, eps, row_ptr, cond_rows, cond_w, uncond_rows, cx, ce, out, x0_coef, x0_out,
                                   uncond_out, B, elems, eps_dtype, (cudaStream_t)stream);
}
int sdxe_euler_ancestral_step(float* x, const float* denoised, const float* noise, float sigma, float sigma_down,
                              float sigma_up, int64_t total, void* stream) {
  return euler_a_step_launch(x, denoised, noise, sigma, sigma_down, sigma_up, total, (cudaStream_t)stream);
}
int sdxe_dpmpp_2m_step(float* x, const float* denoised, const float* old_denoised, float ratio, float neg_expm1,
                       float c0, float c1, int64_t total, void* stream) {
  return dpmpp_2m_step_launch(x, denoised, old_denoised, ratio, neg_expm1, c0, c1, total, (cudaStream_t)stream);
}

}  // extern "C"
