// C-ABI entry points for the stand-alone primitives (include/sdxe.h): attention, GEMM, conv3x3, norms and the
// sampler-step fusions. The model-level entry points live in engine.cu.
#include "../../include/sdxe.h"
#include "attention.cuh"
#include "gemm.cuh"
#include "kernels.cuh"
#include <cmath>
#include <cstring>

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
  const bool bf16 = dtype == SDXE_BF16;
  const int Dpad = (D + 63) / 64 * 64;
  // value dim is processed in passes of at most ATTN_MAX_DV columns (the O accumulator lives in registers)
  int rc = 0;
  for (int v0 = 0; v0 < D && rc == 0; v0 += ATTN_MAX_DV) {
    const int dv = std::min(ATTN_MAX_DV, D - v0);
    AttnArgs a;
    memset(&a, 0, sizeof(a));
    // [B, H, N, D] contiguous seen as (d, token, head, batch); boxes reaching past D are zero-filled by TMA
    if (make_tmap_heads(&a.tmQ, q, D, Nq, H, B, D, (int64_t)Nq * D, (int64_t)H * Nq * D, ATTN_Q_BOX_ROWS)) return -1;
    if (make_tmap_heads(&a.tmK, k, D, Nk, H, B, D, (int64_t)Nk * D, (int64_t)H * Nk * D, ATTN_KV_BOX_ROWS)) return -1;
    const int dvpad = (dv + 63) / 64 * 64;
    if (make_tmap_heads(&a.tmV, (const uint16_t*)v + v0, dv, Nk, H, B, D, (int64_t)Nk * D, (int64_t)H * Nk * D, ATTN_KV_BOX_ROWS)) return -1;
    a.B = B; a.H = H; a.Nq = Nq; a.Nk = Nk;
    a.dqk_slabs = Dpad / 64;
    a.dv_slabs = dvpad / 64;
    a.dv = dv;
    a.dqk = D;
    a.scale_log2 = scale * 1.4426950408889634f;
    a.out = out;
    a.ldo = H * D;
    a.out_col0 = v0;
    a.out_hstride = D;  // heads are interleaved in the output as h*D + j, whatever slice of the value dim a pass covers
    rc = attention_launch(a, bf16, stream);
    count_launch();
  }
  return rc;
}

int sdxe_gemm(const void* A, const void* W, void* out, int M, int N, int K, const float* bias, const void* residual,
              int flags, int dtype, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (!is16(dtype) || K % 8 || N % 8) { set_last_error(__FILE__, __LINE__, "sdxe_gemm: dtype / alignment"); return -2; }
  const bool bf16 = dtype == SDXE_BF16;
  const bool geglu = flags & 1;
  void* scratch = nullptr;
  const void* Wp = W;
  const float* bp = bias;
  GemmArgs a;
  memset(&a, 0, sizeof(a));
  a.M = M; a.N = N; a.K = K; a.K1 = K;
  a.epi = geglu ? EPI_GEGLU : EPI_PLAIN;
  a.BN = gemm_pick_bn(M, N, K, a.epi);
  if (flags >> 8) a.BN = flags >> 8;  // test hook: force the tile width
  if (geglu) {
    // interleave value / gate rows per tile so that both land in the same accumulator tile
    SDXE_CUDA_CHECK(cudaMallocAsync(&scratch, (size_t)N * K * 2 + (size_t)N * 4, stream));
    if (pack_weight_launch(W, dtype, scratch, PACK_GEGLU, N, K, K, a.BN, bf16, stream)) { cudaFreeAsync(scratch, stream); return -1; }
    Wp = scratch;
    if (bias) {
      float* b2 = (float*)((char*)scratch + (size_t)N * K * 2);
      if (pack_vector_launch(bias, SDXE_F32, b2, N, a.BN, false, bf16, stream)) { cudaFreeAsync(scratch, stream); return -1; }
      bp = b2;
    }
  }
  if (make_tmap_2d(&a.tmA, A, M, K, K, 128)) { if (scratch) cudaFreeAsync(scratch, stream); return -1; }
  a.tmA2 = a.tmA;
  a.bias = bp;
  a.residual = residual;
  a.ldr = N;
  a.out = out;
  a.ldo = geglu ? N / 2 : N;
  a.rows_per_sample = 1;
  if (gemm_finish_args(a, Wp, N, K)) { if (scratch) cudaFreeAsync(scratch, stream); return -1; }
  int rc = gemm_launch(a, bf16, stream);
  count_launch();
  if (scratch) cudaFreeAsync(scratch, stream);
  return rc;
}

int sdxe_conv3x3_nhwc(const void* x, const void* w, void* out, int n, int h, int wd, int cin, int cout,
                      const float* bias, int dtype, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (!is16(dtype) || cin % 64 || cout % 8) { set_last_error(__FILE__, __LINE__, "sdxe_conv3x3: alignment"); return -2; }
  const bool bf16 = dtype == SDXE_BF16;
  int bw, bh, bn;
  if (!conv_tile_shape(h, wd, &bw, &bh, &bn)) { set_last_error(__FILE__, __LINE__, "sdxe_conv3x3: unsupported H x W tile"); return -2; }
  GemmArgs a;
  memset(&a, 0, sizeof(a));
  a.M = n * h * wd; a.N = cout; a.K = 9 * cin; a.K1 = a.K;
  a.conv = 1; a.cblocks = cin / 64; a.H = h; a.W = wd; a.bh = bh; a.bn = bn;
  a.epi = EPI_PLAIN;
  a.BN = gemm_pick_bn(a.M, a.N, a.K, a.epi);
  if (make_tmap_nhwc(&a.tmA, x, n, h, wd, cin, bw, bh, bn)) return -1;
  a.tmA2 = a.tmA;
  a.bias = bias;
  a.out = out;
  a.ldo = cout;
  a.rows_per_sample = 1;
  if (gemm_finish_args(a, w, cout, a.K)) return -1;
  int rc = gemm_launch(a, bf16, stream);
  count_launch();
  return rc;
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
  count_launch();
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
