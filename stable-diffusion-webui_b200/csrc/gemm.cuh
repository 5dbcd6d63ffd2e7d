// Argument block of the wgmma GEMM / implicit-GEMM convolution kernel (gemm.cu).
#pragma once
#include "common.cuh"
#include <functional>

namespace sdxe {

enum : int {
  EPI_PLAIN = 0,  // out[m, n] = acc (+bias +rowvec +residual)
  EPI_GEGLU = 1,  // out[m, j] = (acc[j] + b[j]) * gelu(acc[BN/2 + j] + b[BN/2 + j]); weights pre-interleaved per tile
};

struct alignas(64) GemmArgs {
  CUtensorMap tmA;   // 2D: [M, K1] 16-bit, box 64 x 128.  conv: NHWC [N,H,W,C], box 64 x bw x bh x bn
  CUtensorMap tmA2;  // optional second K segment (skip-concat read as two K-segments), 2D only
  CUtensorMap tmB;   // weights [N, K] K-contiguous, box 64 x BN
  int M, N, K;       // problem (conv: K = 9 * Cin, M = N_img * H * W)
  int K1;            // K elements sourced from tmA (== K when there is no second segment)
  int BN;            // tile width (multiple of 16, <= 256)
  int num_stages;
  int conv;          // 0 = plain GEMM, 1 = 3x3 stride-1 pad-1 NHWC implicit GEMM, 2 = 3x3 stride-2 (tmA = make_tmap_nhwc_s2)
  int pad_lo;        // conv == 2: zero rows / columns before the image (1: ldm UNet Downsample, 0: VAE encoder pad (0,1,0,1))
  int cblocks;       // conv: Cin / 64
  int H, W;          // conv: OUTPUT image size; tile = bn images x bh rows x bw pixels (bw == W, or 128 | W)
  int bh, bn;
  int epi;
  int ldrv;          // row pitch (elements) of rowvec
  const float* bias;    // [N] (EPI_GEGLU: interleaved like the weights) or null
  const float* rowvec;  // [M / rows_per_sample, N] per-sample vector added to every row of the sample, or null
  int rows_per_sample;
  int ldr;
  const void* residual;  // [M, ldr] 16-bit or null
  void* out;             // [M, ldo] 16-bit
  int ldo;
  // LayerNorm folded into this GEMM (A is the UN-normalised activation, W already carries gamma):
  //   out[m, n] = rstd[m] * (acc[m, n] - mean[m] * c1[n]) + bias[n]      c1[n] = sum_k W'[n, k], bias includes beta W^T
  // mean / rstd of row m come from the per-row partial (sum, sum of squares) the PRODUCING GEMM wrote (stat_out there).
  const float* c1;          // [N] (GEGLU: interleaved like the bias) or null = no fold
  const float2* ln_part;    // [ln_parts][M] partial (sum, sumsq) of the A rows
  int ln_parts;
  float ln_inv_c, ln_eps;   // 1 / K (the normalised width), epsilon
  // emit per-row partial statistics of the (rounded) output for a consumer's LayerNorm fold:
  float2* stat_out;         // [num_n][M]: part n_blk; null = off. Needs EPI_PLAIN, no rowvec.
};

// A operand: a row-major matrix [M, K1] with row pitch ld, optionally followed along K by a second contiguous matrix
// A2 [M, K - K1] (the skip-concat read as two K segments); or an NHWC image [n, h, w, c] read by the implicit 3x3
// convolution, stride 1 with padding 1, or stride 2 with pad_lo zero rows / columns before the image (output h/2 x w/2).
struct GemmA {
  const void* p = nullptr;
  int64_t M = 0, ld = 0;
  const void* A2 = nullptr;
  int K1 = 0;
  int conv = 0;  // GemmArgs::conv
  int n = 0, h = 0, w = 0, c = 0, pad_lo = 1;
  static GemmA matrix(const void* p, int64_t M, int64_t ld, const void* A2 = nullptr, int K1 = 0) {
    GemmA a;
    a.p = p; a.M = M; a.ld = ld; a.A2 = A2; a.K1 = K1;
    return a;
  }
  static GemmA nhwc(const void* x, int n, int h, int w, int c, int stride = 1, int pad_lo = 1) {
    GemmA a;
    a.p = x; a.conv = stride == 2 ? 2 : 1; a.n = n; a.h = h; a.w = w; a.c = c; a.pad_lo = pad_lo;
    return a;
  }
};
// Packed weight [rows, ld] 16-bit, K-contiguous; rows >= N (zero rows keep a TMA box inside the tensor). c1: the row sums
// of a weight with a LayerNorm folded in (then the epilogue needs the row statistics of A).
struct GemmW {
  const void* w = nullptr;
  int64_t rows = 0, ld = 0;
  int N = 0, K = 0;
  const float* bias = nullptr;
  const float* c1 = nullptr;
};
struct GemmEpi {
  int epi = EPI_PLAIN;
  int ldo = 0;  // 0: N rounded up to 8 (EPI_GEGLU: N / 2)
  const float* rowvec = nullptr;
  int ldrv = 0, rows_per_sample = 1;
  const void* residual = nullptr;
  int ldr = 0;
  const float2* ln_part = nullptr;  // statistics of the A rows, for a weight with a folded LayerNorm
  int ln_parts = 0;
  // set: emit per-row partial statistics of the output (stat_out) into the [parts][M] buffer this returns, parts = the
  // number of column tiles of the chosen BN
  std::function<float2*(int parts)> stat_out;
};
// Fills `a` for out = A W^T with epilogue `o`: tensor maps, tile width (bn > 0 forces it), stage count. Returns 0 / -1.
int gemm_args(GemmArgs& a, const GemmA& A, const GemmW& W, void* out, const GemmEpi& o, int bn = 0);
// Launch on `stream`. bf16 selects the 16-bit format of A/B/out/residual. Returns 0 / -1.
int gemm_launch(const GemmArgs& a, bool bf16, cudaStream_t stream);
int gemm_init();  // one-time kernel attribute setup (call before any stream capture)
// 128-pixel tile of the implicit-GEMM conv as a TMA box (bw x bh x bn); false if (H, W) needs the im2col path.
bool conv_tile_shape(int H, int W, int* bw, int* bh, int* bn);

}  // namespace sdxe
