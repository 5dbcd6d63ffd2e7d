// Argument block of the wgmma GEMM / implicit-GEMM convolution kernel (gemm.cu).
#pragma once
#include "common.cuh"

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

// Launch on `stream`. bf16 selects the 16-bit format of A/B/out/residual. Returns 0 / -1.
int gemm_launch(const GemmArgs& a, bool bf16, cudaStream_t stream);
int gemm_init();  // one-time kernel attribute setup (call before any stream capture)
// Tile-width heuristic: pick BN for an [M, N] output (geglu needs BN % 32 == 0 and N % BN == 0).
int gemm_pick_bn(int M, int N, int K, int epi);
int gemm_pick_stages(int BN);
// After M/N/K/K1/BN/epi/tmA/out/ldo/residual/ldr are set: picks the stage count and builds tmB over the packed
// weights W [w_rows, K] (row pitch w_ld).
int gemm_finish_args(GemmArgs& a, const void* W, int64_t w_rows, int64_t w_ld);
// 128-pixel tile of the implicit-GEMM conv as a TMA box (bw x bh x bn); false if (H, W) needs the im2col path.
bool conv_tile_shape(int H, int W, int* bw, int* bh, int* bn);

}  // namespace sdxe
