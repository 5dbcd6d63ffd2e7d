// wgmma GEMM / implicit-GEMM 3x3 convolution for sm_90a.
//
//   out[M, N] = A[M, K] * W[N, K]^T  (+ bias + per-sample vector + residual | GEGLU)
//
// Replaces, on the UNet / VAE hot path of the reference (all PyTorch library dispatch there):
//   * ResBlock / Upsample / VAE conv3x3      (ldm openaimodel.py ResBlock; SURVEY K5/K6/K10) -> conv mode
//   * conv1x1 proj_in/proj_out/skip, Linear q/k/v/out/FF (SURVEY K7)                          -> plain mode
//   * GEGLU (ldm attention.py GEGLU: x * gelu(gate))                                         -> EPI_GEGLU
//   * nn.LayerNorm in front of q/k/v, cross-attention q and the feed-forward (BasicTransformerBlock norm1-3)
//     -> folded: the producing GEMM emits per-row (sum, sum of squares) (STAT), the consuming GEMM normalises in its
//        epilogue (LNF) with gamma / beta pre-multiplied into its packed weight / bias (gemm.cuh)
//
// Structure (one CTA per SM, persistent over output tiles of 128 x BN):
//   warp 8      : TMA producer. A tile = 128 rows x 64 K (16 KB, 128B swizzle). In conv mode the A tile is a
//                 4D NHWC box (64 ch x W x bh x bn) fetched at the tap's (dx-1, dy-1) offset: TMA's out-of-bounds
//                 zero fill IS the convolution padding, so no im2col buffer ever exists. Circular padding cannot come
//                 from TMA: there the input carries a materialised one-pixel halo and tap (dy, dx) starts at the pixel.
//   warps 0-7   : two warpgroups, each owning 64 rows of the tile. wgmma m64nBNk16 straight from the swizzled stages,
//                 fp32 accumulators in registers (one k-block group in flight while the next is issued), then the
//                 fused epilogue (bias / LayerNorm fold / timestep-embedding vector / residual / GEGLU / row
//                 statistics) from registers to global memory. The producer keeps prefetching the next tile meanwhile.
#include "gemm.cuh"
#include "wgmma.cuh"
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <utility>

namespace sdxe {

static constexpr int BLOCK_M = 128;
static constexpr int BLOCK_K = 64;
static constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;
static constexpr int GEMM_THREADS = 288;  // warpgroups 0-1: MMA + epilogue, warp 8: TMA producer
static constexpr int CONSUMER_WARPS = 8;
static constexpr int SMEM_BUDGET = 227 * 1024;

template <int BN, bool BF16>
__global__ void __launch_bounds__(GEMM_THREADS, 1) gemm_kernel(const __grid_constant__ GemmArgs a) {
  using T = T16<BF16>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t smem_base = (raw + 1023u) & ~1023u;

  const int S = a.num_stages;
  constexpr uint32_t stage_bytes = A_STAGE_BYTES + BN * 128;  // multiple of 1024: every stage keeps the swizzle phase
  const uint32_t bar_base = smem_base + S * stage_bytes;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (S + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_m = (a.M + BLOCK_M - 1) / BLOCK_M;
  const int num_n = (a.N + BN - 1) / BN;
  const int num_kb = (a.K + BLOCK_K - 1) / BLOCK_K;
  const int num_tiles = num_m * num_n;

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), CONSUMER_WARPS);
    }
    fence_mbar_init();
    tma_prefetch_desc(&a.tmA);
    tma_prefetch_desc(&a.tmB);
  }
  __syncthreads();

  if (warp == CONSUMER_WARPS) {
    // ------------------------------------------------------------------ TMA producer (converged warp, elected issue)
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int n_blk = tile % num_n;
      const int m0 = (tile / num_n) * BLOCK_M;
      int img0 = 0, h0 = 0, w0 = 0;
      if (a.conv) {
        const int hw = a.H * a.W;
        img0 = m0 / hw;
        const int rem = m0 - img0 * hw;
        h0 = rem / a.W;
        w0 = rem - h0 * a.W;
      }
      int tap = 0, cb = 0;  // conv: k-block -> (tap, channel block) without divisions
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(empty_bar(stage), phase ^ 1u);
        if (elect_one()) {
          const uint32_t sA = smem_base + stage * stage_bytes;
          const uint32_t sB = sA + A_STAGE_BYTES;
          const uint32_t fb = full_bar(stage);
          mbar_expect_tx(fb, stage_bytes);
          if (a.conv == 2) {  // stride 2: (pixel pair, parity) addressing of the 5-D view, see make_tmap_nhwc_s2
            const int dy = tap / 3, dx = tap - dy * 3;
            const int ty = dy - a.pad_lo, tx = dx - a.pad_lo;
            tma_load_5d(sA, &a.tmA, fb, (tx & 1) * (a.cblocks * BLOCK_K) + cb * BLOCK_K, w0 + (tx >> 1), ty & 1, h0 + (ty >> 1), img0);
          } else if (a.conv) {
            const int dy = tap / 3, dx = tap - dy * 3;
            tma_load_4d(sA, &a.tmA, fb, cb * BLOCK_K, w0 + dx - a.pad_lo, h0 + dy - a.pad_lo, img0);
          } else {
            const int k0 = kb * BLOCK_K;
            if (k0 < a.K1) tma_load_2d(sA, &a.tmA, fb, k0, m0);
            else tma_load_2d(sA, &a.tmA2, fb, k0 - a.K1, m0);
          }
          tma_load_2d(sB, &a.tmB, fb, kb * BLOCK_K, n_blk * BN);
        }
        __syncwarp();
        if (++cb == a.cblocks) { cb = 0; ++tap; }
        if (++stage == S) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- MMA + epilogue warpgroups
  // Accumulator fragment of wgmma m64nN (per warp 16 rows): acc[4 i + 2 h + e] is row (lane / 4 + 8 h) of the warp's
  // band, column 8 i + 2 (lane % 4) + e.
  const int wg = warp >> 2;
  const int band = (warp & 3) * 16 + (lane >> 2);  // row inside this warpgroup's 64
  const int cq = 2 * (lane & 3);
  const int M = a.M, N = a.N;
  const uint64_t adesc0 = gmma_desc_sw128(smem_base + (uint32_t)wg * (64 * 128), 16, 1024);
  const uint64_t bdesc0 = gmma_desc_sw128(smem_base + A_STAGE_BYTES, 16, 1024);
  constexpr uint32_t stage_inc = stage_bytes >> 4;
  float acc[BN / 2];
  int stage = 0;
  uint32_t phase = 0;
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int n_blk = tile % num_n;
    const int m_blk = tile / num_n;
    int prev = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(full_bar(stage), phase);
      wgmma_fence();
      const uint64_t ad = adesc0 + (uint64_t)(stage * stage_inc);
      const uint64_t bd = bdesc0 + (uint64_t)(stage * stage_inc);
      // +32 bytes along K inside the 128B swizzle atom = +2 in the (addr >> 4) field
      wgmma_ss<BN, BF16>(acc, ad, bd, kb != 0);
      wgmma_ss<BN, BF16>(acc, ad + 2, bd + 2, 1);
      wgmma_ss<BN, BF16>(acc, ad + 4, bd + 4, 1);
      wgmma_ss<BN, BF16>(acc, ad + 6, bd + 6, 1);
      wgmma_commit();
      if (prev >= 0) {  // the previous k-block's group is complete: its stage may be refilled
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(empty_bar(prev));
      }
      prev = stage;
      if (++stage == S) { stage = 0; phase ^= 1u; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);
    if (lane == 0 && prev >= 0) mbar_arrive(empty_bar(prev));

    // ---------------------------------------------------------------- epilogue
    const int row0 = m_blk * BLOCK_M + wg * 64 + band;
    float ln_mu[2] = {0.f, 0.f}, ln_rs[2] = {1.f, 1.f};
    if (a.c1) {  // LayerNorm fold: this row's mean / rstd from the producer's partial sums (fixed order: deterministic)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = row0 + 8 * h;
        float ps = 0.f, pq = 0.f;
        if (m < M) {
          for (int pp = 0; pp < a.ln_parts; ++pp) {
            const float2 t = __ldg(a.ln_part + (size_t)pp * M + m);
            ps += t.x;
            pq += t.y;
          }
        }
        ln_mu[h] = ps * a.ln_inv_c;
        ln_rs[h] = rsqrtf(fmaxf(pq * a.ln_inv_c - ln_mu[h] * ln_mu[h], 0.f) + a.ln_eps);
      }
    }
    if (a.epi == EPI_GEGLU) {
      // PACK_GEGLU weights / bias / c1: tile n_blk's rows are [BN/2 value rows | the matching BN/2 gate rows]; N % BN == 0.
      // Value column j and gate column BN/2 + j sit in the same thread's fragment.
      constexpr int HALF = BN / 2;
      const int ldo = a.ldo;
#pragma unroll
      for (int i = 0; i < HALF / 8; ++i) {
        const int jl = 8 * i + cq;
        const int cv = n_blk * BN + jl, cg = cv + HALF;
        float bv[2] = {0.f, 0.f}, bg[2] = {0.f, 0.f}, kv[2] = {0.f, 0.f}, kg[2] = {0.f, 0.f};
        if (a.bias) { bv[0] = __ldg(a.bias + cv); bv[1] = __ldg(a.bias + cv + 1); bg[0] = __ldg(a.bias + cg); bg[1] = __ldg(a.bias + cg + 1); }
        if (a.c1) { kv[0] = __ldg(a.c1 + cv); kv[1] = __ldg(a.c1 + cv + 1); kg[0] = __ldg(a.c1 + cg); kg[1] = __ldg(a.c1 + cg + 1); }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = row0 + 8 * h;
          float o[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float v = acc[4 * i + 2 * h + e], g = acc[4 * (i + HALF / 8) + 2 * h + e];
            if (a.c1) {
              v = fmaf(ln_rs[h], v - ln_mu[h] * kv[e], bv[e]);
              g = fmaf(ln_rs[h], g - ln_mu[h] * kg[e], bg[e]);
            } else {
              v += bv[e];
              g += bg[e];
            }
            o[e] = v * gelu_fast_f(g);
          }
          if (m < M) *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(a.out) + (size_t)m * ldo + n_blk * HALF + jl) = T::pack(o[0], o[1]);
        }
      }
    } else {
      // columns N .. N rounded up to 8 (inside the output pitch) are written as zeros (+ residual), like a padded weight row
      const int n_store = std::min((N + 7) / 8 * 8, a.ldo);
      const int n_res = a.residual ? std::min((N + 7) / 8 * 8, a.ldr) : 0;
      const float* rv[2] = {nullptr, nullptr};
      bool row_ok[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = row0 + 8 * h;
        row_ok[h] = m < M;
        if (a.rowvec && row_ok[h]) rv[h] = a.rowvec + (size_t)(m / a.rows_per_sample) * a.ldrv;
      }
      float st_s[2] = {0.f, 0.f}, st_q[2] = {0.f, 0.f};
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const int col = n_blk * BN + 8 * i + cq;  // even; n_store is a multiple of 8, so col + 1 is stored with col
        if (col >= n_store) continue;
        const bool in0 = col < N, in1 = col + 1 < N;
        float b[2] = {0.f, 0.f}, k[2] = {0.f, 0.f};
        if (a.bias) { b[0] = in0 ? __ldg(a.bias + col) : 0.f; b[1] = in1 ? __ldg(a.bias + col + 1) : 0.f; }
        if (a.c1) { k[0] = in0 ? __ldg(a.c1 + col) : 0.f; k[1] = in1 ? __ldg(a.c1 + col + 1) : 0.f; }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!row_ok[h]) continue;
          const size_t m = (size_t)(row0 + 8 * h);
          float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
          if (a.c1) {
            v0 = fmaf(ln_rs[h], v0 - ln_mu[h] * k[0], b[0]);
            v1 = fmaf(ln_rs[h], v1 - ln_mu[h] * k[1], b[1]);
          } else {
            v0 += b[0];
            v1 += b[1];
          }
          if (rv[h]) {
            if (in0) v0 += __ldg(rv[h] + col);
            if (in1) v1 += __ldg(rv[h] + col + 1);
          }
          if (col < n_res) {
            const uint32_t r = __ldg(reinterpret_cast<const unsigned int*>(reinterpret_cast<const uint16_t*>(a.residual) + m * a.ldr + col));
            const float2 f = T::unpack(r);
            v0 += f.x;
            v1 += f.y;
          }
          const uint32_t pk = T::pack(v0, v1);
          *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(a.out) + m * a.ldo + col) = pk;
          if (a.stat_out) {  // statistics of the values as stored (rounded to 16 bit), like a LayerNorm reading them back
            const float2 f = T::unpack(pk);
            const float x0 = in0 ? f.x : 0.f, x1 = in1 ? f.y : 0.f;
            st_s[h] += x0 + x1;
            st_q[h] = fmaf(x0, x0, fmaf(x1, x1, st_q[h]));
          }
        }
      }
      if (a.stat_out) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {  // the four threads of a quad hold one row's columns
          st_s[h] += __shfl_xor_sync(0xffffffffu, st_s[h], 1);
          st_q[h] += __shfl_xor_sync(0xffffffffu, st_q[h], 1);
          st_s[h] += __shfl_xor_sync(0xffffffffu, st_s[h], 2);
          st_q[h] += __shfl_xor_sync(0xffffffffu, st_q[h], 2);
          if ((lane & 3) == 0 && row_ok[h]) a.stat_out[(size_t)n_blk * M + row0 + 8 * h] = make_float2(st_s[h], st_q[h]);
        }
      }
    }
  }
}

bool conv_tile_shape(int H, int W, int* bw, int* bh, int* bn) {
  if (W >= 128) {
    if (W % 128) return false;
    *bw = 128; *bh = 1; *bn = 1;
    return true;
  }
  if (128 % W) return false;
  const int rows = 128 / W;
  if (H >= rows) {
    if (H % rows) return false;
    *bw = W; *bh = rows; *bn = 1;
    return true;
  }
  if (rows % H) return false;
  *bw = W; *bh = H; *bn = rows / H;
  return true;
}

static size_t gemm_smem_fixed(int num_stages) {  // everything but the operand stages
  return 1024 /*base alignment*/ + 16 * (size_t)num_stages;
}
static size_t gemm_smem(int BN, int num_stages) { return (size_t)num_stages * (A_STAGE_BYTES + BN * 128) + gemm_smem_fixed(num_stages); }

static int gemm_pick_stages(int BN) {
  const int stage_bytes = A_STAGE_BYTES + BN * 128;
  const int s = (int)((SMEM_BUDGET - gemm_smem_fixed(8)) / stage_bytes);
  return std::max(2, std::min(s, 8));
}

// Tile-width heuristic: pick BN for an [M, N] output (geglu needs BN % 32 == 0 and N % BN == 0).
static int gemm_pick_bn(int M, int N, int epi) {
  const int sms = num_sms();
  const int num_m = (M + BLOCK_M - 1) / BLOCK_M;
  double best = 1e30;
  int best_bn = 16;
  for (int bn = 16; bn <= 256; bn += 16) {
    if (epi == EPI_GEGLU && (bn % 32 != 0 || N % bn != 0)) continue;
    const int num_n = (N + bn - 1) / bn;
    const long tiles = (long)num_m * num_n;
    const long waves = (tiles + sms - 1) / sms;
    // cycles per 64-deep k-block: tensor pipe (128 x BN x 64 MACs at ~2 k MACs / clk / SM) vs. operand fetch through L2
    // (~32 B/clk/SM) + fixed issue / barrier overhead
    const double kb = std::max(4.0 * bn, (A_STAGE_BYTES + 128.0 * bn) / 32.0) + 64.0;
    const double cost = waves * kb;
    if (cost < best - 1e-9) { best = cost; best_bn = bn; }
  }
  return best_bn;
}

int gemm_args(GemmArgs& a, const GemmA& A, const GemmW& W, void* out, const GemmEpi& o, int bn) {
  memset(&a, 0, sizeof(a));
  a.N = W.N; a.K = W.K;
  if (A.conv) {
    const int Ho = (A.h - 2 * A.halo) / A.conv, Wo = (A.w - 2 * A.halo) / A.conv;
    int bw;
    if (A.c % 64 || !conv_tile_shape(Ho, Wo, &bw, &a.bh, &a.bn)) { set_last_error(__FILE__, __LINE__, "gemm: conv geometry"); return -1; }
    a.M = A.n * Ho * Wo; a.K1 = a.K;
    a.conv = A.conv; a.pad_lo = A.pad_lo; a.cblocks = A.c / 64; a.H = Ho; a.W = Wo;
    if ((A.conv == 2 ? make_tmap_nhwc_s2 : make_tmap_nhwc)(&a.tmA, A.p, A.n, A.h, A.w, A.c, bw, a.bh, a.bn)) return -1;
    a.tmA2 = a.tmA;
  } else {
    a.M = (int)A.M;
    a.K1 = A.A2 ? A.K1 : W.K;
    if (make_tmap_2d(&a.tmA, A.p, A.M, a.K1, A.ld, 128)) return -1;
    if (A.A2) { if (make_tmap_2d(&a.tmA2, A.A2, A.M, W.K - A.K1, W.K - A.K1, 128)) return -1; }
    else a.tmA2 = a.tmA;
  }
  a.epi = o.epi;
  a.BN = bn ? bn : gemm_pick_bn(a.M, a.N, o.epi);
  a.num_stages = gemm_pick_stages(a.BN);
  a.bias = W.bias;
  a.rowvec = o.rowvec; a.ldrv = o.ldrv; a.rows_per_sample = std::max(1, o.rows_per_sample);
  a.residual = o.residual; a.ldr = o.ldr;
  a.out = out;
  a.ldo = o.ldo ? o.ldo : (o.epi == EPI_GEGLU ? W.N / 2 : (W.N + 7) / 8 * 8);
  if (W.c1) {  // a weight with a LayerNorm folded in can only be applied with the row statistics of A
    if (!o.ln_part || A.A2) { set_last_error(__FILE__, __LINE__, "gemm: folded LayerNorm weight without row statistics"); return -1; }
    a.c1 = W.c1; a.ln_part = o.ln_part; a.ln_parts = o.ln_parts;
    a.ln_inv_c = 1.0f / (float)W.K; a.ln_eps = 1e-5f;
  }
  if (o.stat_out) a.stat_out = o.stat_out((a.N + a.BN - 1) / a.BN);
  if (a.ldo % 8 || (a.residual && a.ldr % 8)) { set_last_error(__FILE__, __LINE__, "gemm: ldo / ldr must be multiples of 8"); return -1; }
  return make_tmap_2d(&a.tmB, W.w, W.rows, a.K, W.ld, a.BN);
}

typedef void (*GemmKernel)(const GemmArgs);
static constexpr int GEMM_NUM_BN = 16;  // BN = 16, 32, ..., 256
template <std::size_t... I>
static GemmKernel gemm_variant_impl(int i, bool bf16, std::index_sequence<I...>) {
  static const GemmKernel k16[] = {gemm_kernel<16 * (int)(I + 1), false>...};
  static const GemmKernel kb16[] = {gemm_kernel<16 * (int)(I + 1), true>...};
  return bf16 ? kb16[i] : k16[i];
}
static GemmKernel gemm_variant(int BN, bool bf16) {
  return gemm_variant_impl(BN / 16 - 1, bf16, std::make_index_sequence<GEMM_NUM_BN>{});
}

int gemm_init() {
  static bool done = false;
  if (!done) {
    for (int bn = 16; bn <= 256; bn += 16)
      for (int b = 0; b < 2; ++b)
        SDXE_CUDA_CHECK(cudaFuncSetAttribute(gemm_variant(bn, b != 0), cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BUDGET));
    done = true;
  }
  return 0;
}

int gemm_launch(const GemmArgs& a, bool bf16, cudaStream_t stream) {
  if (a.BN % 16 != 0 || a.BN < 16 || a.BN > 256) { set_last_error(__FILE__, __LINE__, "gemm: bad BN"); return -1; }
  if (a.K1 != a.K && (a.K1 % BLOCK_K) != 0) { set_last_error(__FILE__, __LINE__, "gemm: K1 % 64"); return -1; }
  if (a.epi == EPI_GEGLU && (a.BN % 32 != 0 || a.N % a.BN != 0)) { set_last_error(__FILE__, __LINE__, "gemm: geglu tile"); return -1; }
  if ((a.epi != EPI_PLAIN) && (a.residual || a.rowvec || a.stat_out)) { set_last_error(__FILE__, __LINE__, "gemm: residual / rowvec / statistics need EPI_PLAIN"); return -1; }
  if ((a.c1 && (a.residual || a.stat_out || a.rowvec)) || (a.stat_out && a.rowvec)) {
    set_last_error(__FILE__, __LINE__, "gemm: unsupported LayerNorm-fold / statistics combination");
    return -1;
  }
  if (a.num_stages < 2) { set_last_error(__FILE__, __LINE__, "gemm: stages (fill the arguments with gemm_args)"); return -1; }
  const size_t smem = gemm_smem(a.BN, a.num_stages);
  if (smem > (size_t)SMEM_BUDGET) { set_last_error(__FILE__, __LINE__, "gemm: shared memory budget"); return -1; }
  const int num_m = (a.M + BLOCK_M - 1) / BLOCK_M, num_n = (a.N + a.BN - 1) / a.BN;
  const int tiles = num_m * num_n;
  if (tiles <= 0) return 0;
  if (gemm_init() != 0) return -1;
  const int grid = std::min(tiles, num_sms());
  const GemmKernel kern = gemm_variant(a.BN, bf16);
  kern<<<grid, GEMM_THREADS, smem, stream>>>(a);
  SDXE_LAUNCH_CHECK();
  return 0;
}

}  // namespace sdxe
