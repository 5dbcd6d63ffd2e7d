// Bandwidth-bound kernels: GroupNorm / LayerNorm, layout gathers, embeddings, weight repack, sampler-step fusions.
// All activation tensors are 16-bit NHWC ([n, h*w, c]); vectors of 8 channels (16 B) per thread access.
#include "kernels.cuh"
#include <algorithm>

namespace sdxe {

SDXE_DEVINL float load_any(const void* p, int dtype, int64_t i) {
  if (dtype == DT_F16) return __half2float(reinterpret_cast<const __half*>(p)[i]);
  if (dtype == DT_BF16) return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[i]);
  return reinterpret_cast<const float*>(p)[i];
}
SDXE_DEVINL void store_any(void* p, int dtype, int64_t i, float v) {
  if (dtype == DT_F16) reinterpret_cast<__half*>(p)[i] = __float2half_rn(v);
  else if (dtype == DT_BF16) reinterpret_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
  else reinterpret_cast<float*>(p)[i] = v;
}
template <bool BF16>
SDXE_DEVINL void unpack8(const uint4& u, float* v) {
  float2 f;
  f = T16<BF16>::unpack(u.x); v[0] = f.x; v[1] = f.y;
  f = T16<BF16>::unpack(u.y); v[2] = f.x; v[3] = f.y;
  f = T16<BF16>::unpack(u.z); v[4] = f.x; v[5] = f.y;
  f = T16<BF16>::unpack(u.w); v[6] = f.x; v[7] = f.y;
}
template <bool BF16>
SDXE_DEVINL uint4 pack8(const float* v) {
  uint4 u;
  u.x = T16<BF16>::pack(v[0], v[1]);
  u.y = T16<BF16>::pack(v[2], v[3]);
  u.z = T16<BF16>::pack(v[4], v[5]);
  u.w = T16<BF16>::pack(v[6], v[7]);
  return u;
}
template <bool BF16>
SDXE_DEVINL float round16(float v) { return T16<BF16>::to_f(T16<BF16>::from_f(v)); }

// =============================================================================================================
// GroupNorm (ldm GroupNorm32: statistics in fp32 — modules/devices.py:284-295 states the upcast)
// =============================================================================================================
// Deterministic two-level reduction (no atomics: the same input always gives bit-identical statistics, as the
// reference's torch.group_norm does): block partials [n, chunk, group, 2] -> finalize -> (mean, rstd) per (n, group).
template <bool BF16>
__global__ void gn_stats_kernel(const uint4* __restrict__ x1, int c1, const uint4* __restrict__ x2, int c2,
                                float* __restrict__ partial, int hw, int groups, int pix_per_block) {
  extern __shared__ float sh[];  // [rpi][C] sums, then [rpi][C] sums of squares
  const int C = c1 + c2, V = C >> 3, cpg = C / groups;
  const int n = blockIdx.y;
  const int vec = threadIdx.x % V, prow = threadIdx.x / V, rpi = blockDim.x / V;
  float* sh_s = sh;
  float* sh_q = sh + rpi * C;
  const int p0 = blockIdx.x * pix_per_block, p1 = min(hw, p0 + pix_per_block);
  float s[8], ss[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = ss[j] = 0.f;
  const int c = vec * 8;
  const uint4* src = (c < c1) ? x1 : x2;
  const int cs = (c < c1) ? c1 : c2, co = (c < c1) ? c : c - c1;
#pragma unroll 4
  for (int p = p0 + prow; p < p1; p += rpi) {
    const size_t pix = (size_t)n * hw + p;
    const uint4 u = __ldg(src + (pix * cs + co) / 8);
    float v[8];
    unpack8<BF16>(u, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) { s[j] += v[j]; ss[j] += v[j] * v[j]; }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) { sh_s[prow * C + c + j] = s[j]; sh_q[prow * C + c + j] = ss[j]; }
  __syncthreads();
  for (int g = threadIdx.x; g < groups; g += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int r = 0; r < rpi; ++r)
      for (int cc = g * cpg; cc < (g + 1) * cpg; ++cc) { a += sh_s[r * C + cc]; b += sh_q[r * C + cc]; }
    float* dst = partial + (((size_t)n * gridDim.x + blockIdx.x) * groups + g) * 2;
    dst[0] = a;
    dst[1] = b;
  }
}

__global__ void gn_finalize_kernel(const float* __restrict__ partial, float* __restrict__ stats, int n_img, int chunks,
                                   int groups, float inv_cnt, float eps) {
  // one warp per (image, group): lanes stride over the block partials, fixed-order tree reduce (deterministic)
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n_img * groups) return;
  const int n = i / groups, g = i - n * groups;
  float a = 0.f, b = 0.f;
  for (int ch = lane; ch < chunks; ch += 32) {
    const float2 v = __ldg(reinterpret_cast<const float2*>(partial + (((size_t)n * chunks + ch) * groups + g) * 2));
    a += v.x;
    b += v.y;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  if (lane == 0) {
    const float mean = a * inv_cnt;
    const float var = fmaxf(b * inv_cnt - mean * mean, 0.f);
    stats[2 * i] = mean;
    stats[2 * i + 1] = rsqrtf(var + eps);
  }
}

// Apply: same thread -> (8-channel vector, pixel row) mapping as the statistics kernel, so the per-channel
// scale = rstd*gamma and shift = beta - mean*scale are computed once per thread and the pixel loop is
// load -> 8 x (FMA [+ SiLU]) -> store with no index arithmetic.
template <bool BF16, bool SILU>
__global__ void gn_apply_kernel(const uint4* __restrict__ x1, int c1, const uint4* __restrict__ x2, int c2,
                                const float* __restrict__ stats, const float* __restrict__ gamma,
                                const float* __restrict__ beta, uint4* __restrict__ out, int hw, int groups,
                                int pix_per_block) {
  const int C = c1 + c2, V = C >> 3, cpg = C / groups;
  const int n = blockIdx.y;
  const int vec = threadIdx.x % V, prow = threadIdx.x / V, rpi = blockDim.x / V;
  const int c = vec * 8;
  float sc[8], sh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int g = (c + j) / cpg;
    const float2 mr = __ldg(reinterpret_cast<const float2*>(stats + ((size_t)n * groups + g) * 2));
    sc[j] = mr.y * __ldg(gamma + c + j);
    sh[j] = __ldg(beta + c + j) - mr.x * sc[j];
  }
  const uint4* src = (c < c1) ? x1 : x2;
  const int cs = (c < c1) ? c1 : c2, co = (c < c1) ? c : c - c1;
  const int p0 = blockIdx.x * pix_per_block, p1 = min(hw, p0 + pix_per_block);
#pragma unroll 4
  for (int p = p0 + prow; p < p1; p += rpi) {
    const size_t pix = (size_t)n * hw + p;
    float v[8];
    unpack8<BF16>(__ldg(src + (pix * cs + co) / 8), v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float y = fmaf(v[j], sc[j], sh[j]);
      if (SILU) y = silu_f(y);
      v[j] = y;
    }
    out[pix * V + vec] = pack8<BF16>(v);
  }
}

// One-pass GroupNorm for the UNet's shapes: one CTA per (sample, group) keeps the group's [hw, C/groups] strip in shared
// memory — one global read, fp32 two-pass statistics (mean, then centred second moment) from smem, one global write.
// Replaces stats + finalize + apply (2 reads, 1 write, 3 launches) for the small tensors (strip hw * cpg * 2 B <= 48 KB:
// the 8x8 / 16x16 and narrow 32x32 levels, where the three launches are latency-bound); larger tensors keep the
// three-kernel streaming path.
// Thread -> (pixel lane, channel pair): the channel pair is fixed per thread, so gamma / beta / source pointer live in
// registers and the loops carry no divisions. Fixed reduction order: bit-identical on replay.
template <bool BF16, bool SILU>
__global__ void __launch_bounds__(512) gn_onepass_kernel(const uint32_t* __restrict__ x1, int c1, const uint32_t* __restrict__ x2, int c2,
                                  const float* __restrict__ gamma, const float* __restrict__ beta,
                                  uint32_t* __restrict__ out, int hw, int groups, float eps) {
  extern __shared__ uint32_t gn_tile[];  // [hw][W] packed channel pairs
  __shared__ float red[16];
  __shared__ float bcast;
  const int C = c1 + c2, cpg = C / groups, W = cpg >> 1;
  const int g = blockIdx.x, n = blockIdx.y;
  const int R = blockDim.x / W;                 // pixels per sweep
  const int pl = threadIdx.x / W, w = threadIdx.x - pl * W;
  const bool active = pl < R;
  const int c = g * cpg + 2 * w;                // first channel of this thread's pair
  const uint32_t* src = (c < c1) ? x1 : x2;
  const int cs = (c < c1) ? c1 : c2, co = (c < c1) ? c : c - c1;
  const size_t pix0 = (size_t)n * hw;
  auto block_sum = [&](float v) -> float {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();  // red / bcast reusable
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
      float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if (threadIdx.x == 0) bcast = t;
    }
    __syncthreads();
    return bcast;
  };
  float s = 0.f;
  if (active) {
#pragma unroll 4
    for (int p = pl; p < hw; p += R) {
      const uint32_t u = __ldg(src + (((pix0 + p) * cs + co) >> 1));
      gn_tile[p * W + w] = u;
      const float2 f = T16<BF16>::unpack(u);
      s += f.x + f.y;
    }
  }
  const float inv_cnt = 1.f / ((float)hw * (float)cpg);
  const float mean = block_sum(s) * inv_cnt;
  float q = 0.f;
  if (active) {
#pragma unroll 4
    for (int p = pl; p < hw; p += R) {  // own elements only: no cross-thread smem dependency
      const float2 f = T16<BF16>::unpack(gn_tile[p * W + w]);
      const float a = f.x - mean, b = f.y - mean;
      q += a * a + b * b;
    }
  }
  const float rstd = rsqrtf(block_sum(q) * inv_cnt + eps);
  if (active) {
    const float sc0 = rstd * __ldg(gamma + c), sc1 = rstd * __ldg(gamma + c + 1);
    const float sh0 = __ldg(beta + c) - mean * sc0, sh1 = __ldg(beta + c + 1) - mean * sc1;
    uint32_t* dst = out + ((pix0 * C + c) >> 1);
    const int Ch = C >> 1;
#pragma unroll 4
    for (int p = pl; p < hw; p += R) {
      const float2 f = T16<BF16>::unpack(gn_tile[p * W + w]);
      float y0 = fmaf(f.x, sc0, sh0), y1 = fmaf(f.y, sc1, sh1);
      if (SILU) { y0 = silu_f(y0); y1 = silu_f(y1); }
      dst[(size_t)p * Ch] = T16<BF16>::pack(y0, y1);
    }
  }
}

static int skinny_linear_init();
int kernels_init() {
  static bool done = false;
  if (!done) {
    SDXE_CUDA_CHECK(cudaFuncSetAttribute(gn_stats_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    SDXE_CUDA_CHECK(cudaFuncSetAttribute(gn_stats_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    SDXE_CUDA_CHECK(cudaFuncSetAttribute(gn_onepass_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    SDXE_CUDA_CHECK(cudaFuncSetAttribute(gn_onepass_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    SDXE_CUDA_CHECK(cudaFuncSetAttribute(gn_onepass_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    SDXE_CUDA_CHECK(cudaFuncSetAttribute(gn_onepass_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    if (skinny_linear_init() != 0) return -1;
    done = true;
  }
  return 0;
}

size_t group_norm_scratch_floats(int n, int groups) { return (size_t)n * groups * 2 * ((size_t)num_sms() * 4 + 2); }

int group_norm_launch(const void* x1, int c1, const void* x2, int c2, const float* gamma, const float* beta, void* out,
                      float* scratch, int n, int hw, int groups, float eps, bool silu, bool bf16, cudaStream_t s) {
  if (x2 == nullptr) c2 = 0;
  const int C = c1 + c2;
  if (C % 8 || c1 % 8 || C % groups) { set_last_error(__FILE__, __LINE__, "group_norm: channel alignment"); return -1; }
  if (kernels_init() != 0) return -1;
  {
    const int cpg = C / groups;
    const size_t strip = (size_t)hw * cpg * 2;
    // crossover: one CTA per strip wins up to ~48 KB (enough CTAs per SM to hide its serial passes); the
    // wide 64x64 / 32x32 tensors are faster through the three streaming kernels
    if (cpg % 2 == 0 && cpg / 2 <= 256 && strip <= 48 * 1024) {
      const int threads = strip >= 32 * 1024 ? 512 : 256;
      dim3 grid(groups, n);
#define GN_ONE(B, S) gn_onepass_kernel<B, S><<<grid, threads, strip, s>>>((const uint32_t*)x1, c1, (const uint32_t*)x2, c2, gamma, beta, (uint32_t*)out, hw, groups, eps)
      if (bf16) { if (silu) GN_ONE(true, true); else GN_ONE(true, false); }
      else { if (silu) GN_ONE(false, true); else GN_ONE(false, false); }
#undef GN_ONE
      SDXE_LAUNCH_CHECK();
      return 0;
    }
  }
  const int V = C / 8;
  if (V > 1024) { set_last_error(__FILE__, __LINE__, "group_norm: too many channels"); return -1; }
  int rpi = std::max(1, 256 / V);
  while (rpi > 1 && (size_t)rpi * C * 8 > 96 * 1024) --rpi;
  const int threads = V * rpi;
  int chunks = std::max(1, std::min((num_sms() * 4 + n - 1) / n, (hw + rpi * 4 - 1) / (rpi * 4)));
  const int ppb = (hw + chunks - 1) / chunks;
  chunks = (hw + ppb - 1) / ppb;
  float* stats = scratch;                          // [n, groups, 2] (mean, rstd)
  float* partial = scratch + (size_t)n * groups * 2;  // [n, chunks, groups, 2]
  dim3 grid(chunks, n);
  const size_t sm = sizeof(float) * 2 * rpi * C;
  if (kernels_init() != 0) return -1;
  if (bf16)
    gn_stats_kernel<true><<<grid, threads, sm, s>>>((const uint4*)x1, c1, (const uint4*)x2, c2, partial, hw, groups, ppb);
  else
    gn_stats_kernel<false><<<grid, threads, sm, s>>>((const uint4*)x1, c1, (const uint4*)x2, c2, partial, hw, groups, ppb);
  SDXE_LAUNCH_CHECK();
  const float inv_cnt = 1.f / ((float)hw * (float)(C / groups));
  gn_finalize_kernel<<<(n * groups + 3) / 4, 128, 0, s>>>(partial, stats, n, chunks, groups, inv_cnt, eps);
  SDXE_LAUNCH_CHECK();
  // apply: finer pixel chunks than the statistics pass (pure streaming, wants every SM busy several times over)
  int achunks = std::max(1, std::min((num_sms() * 8 + n - 1) / n, (hw + rpi * 2 - 1) / (rpi * 2)));
  const int appb = (hw + achunks - 1) / achunks;
  achunks = (hw + appb - 1) / appb;
  dim3 agrid(achunks, n);
#define GN_APPLY(B, S)                                                                                                \
  gn_apply_kernel<B, S><<<agrid, threads, 0, s>>>((const uint4*)x1, c1, (const uint4*)x2, c2, stats, gamma, beta, (uint4*)out, \
                                                  hw, groups, appb)
  if (bf16) { if (silu) GN_APPLY(true, true); else GN_APPLY(true, false); }
  else { if (silu) GN_APPLY(false, true); else GN_APPLY(false, false); }
#undef GN_APPLY
  SDXE_LAUNCH_CHECK();
  return 0;
}

// =============================================================================================================
// LayerNorm (fp32 statistics, as torch autocast runs layer_norm in fp32) — one warp per row
// =============================================================================================================
template <bool BF16, int MAXV>  // MAXV x 32 x 8 channels held in registers (one global read of the row)
__global__ void __launch_bounds__(256) layer_norm_kernel(const uint4* __restrict__ x, const float* __restrict__ gamma,
                                  const float* __restrict__ beta, uint4* __restrict__ out, int rows, int C, float eps) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const int V = C >> 3;
  const uint4* xr = x + (size_t)warp * V;
  float f[MAXV][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int v = lane + 32 * i;
    if (v < V) {
      unpack8<BF16>(__ldg(xr + v), f[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += f[i][j];
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / (float)C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    if (lane + 32 * i < V) {
#pragma unroll
      for (int j = 0; j < 8; ++j) { const float d = f[i][j] - mean; sq += d * d; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / (float)C + eps);
  uint4* orow = out + (size_t)warp * V;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int v = lane + 32 * i;
    if (v < V) {
      const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + v * 8)), gb = __ldg(reinterpret_cast<const float4*>(gamma + v * 8 + 4));
      const float4 ba = __ldg(reinterpret_cast<const float4*>(beta + v * 8)), bb = __ldg(reinterpret_cast<const float4*>(beta + v * 8 + 4));
      const float gm[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
      const float bt[8] = {ba.x, ba.y, ba.z, ba.w, bb.x, bb.y, bb.z, bb.w};
      float y[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = (f[i][j] - mean) * rstd * gm[j] + bt[j];
      orow[v] = pack8<BF16>(y);
    }
  }
}

// C = 40 * G channels (the UNet's 320 / 640 / 1280): G = 8 / 16 / 32 lanes per row, five 8-channel vectors per lane, so
// every lane of the warp is busy (the generic kernel leaves 3/8 of its lanes idle at C = 320) and a warp covers 32 / G rows.
template <bool BF16, int G>
__global__ void __launch_bounds__(256) layer_norm5_kernel(const uint4* __restrict__ x, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, uint4* __restrict__ out, int rows, float eps) {
  constexpr int RPW = 32 / G, V = 5 * G, C = 8 * V;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int row = warp * RPW + lane / G, gl = lane % G;
  const bool ok = row < rows;
  const uint4* xr = x + (size_t)row * V;
  float f[5][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    if (ok) unpack8<BF16>(__ldg(xr + gl + G * i), f[i]);
    else {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[i][j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) sum += f[i][j];
  }
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum * (1.f / (float)C);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < 5; ++i) {
#pragma unroll
    for (int j = 0; j < 8; ++j) { const float d = f[i][j] - mean; sq += d * d; }
  }
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq * (1.f / (float)C) + eps);
  if (!ok) return;
  uint4* orow = out + (size_t)row * V;
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    const int v = gl + G * i;
    const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + v * 8)), gb = __ldg(reinterpret_cast<const float4*>(gamma + v * 8 + 4));
    const float4 ba = __ldg(reinterpret_cast<const float4*>(beta + v * 8)), bb = __ldg(reinterpret_cast<const float4*>(beta + v * 8 + 4));
    const float gm[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
    const float bt[8] = {ba.x, ba.y, ba.z, ba.w, bb.x, bb.y, bb.z, bb.w};
    float y[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) y[j] = (f[i][j] - mean) * rstd * gm[j] + bt[j];
    orow[v] = pack8<BF16>(y);
  }
}

int layer_norm_launch(const void* x, const float* gamma, const float* beta, void* out, int rows, int c, float eps,
                      bool bf16, cudaStream_t s) {
  if (c % 8 || c > 2048) { set_last_error(__FILE__, __LINE__, "layer_norm: C % 8 != 0 or C > 2048"); return -1; }
  if (c == 320 || c == 640 || c == 1280) {
    const int G = c / 40, rpb = 8 * (32 / G);  // rows per 256-thread block
    const int nb = (rows + rpb - 1) / rpb;
#define LN5(B, GG) layer_norm5_kernel<B, GG><<<nb, 256, 0, s>>>((const uint4*)x, gamma, beta, (uint4*)out, rows, eps)
    if (bf16) { if (G == 8) LN5(true, 8); else if (G == 16) LN5(true, 16); else LN5(true, 32); }
    else { if (G == 8) LN5(false, 8); else if (G == 16) LN5(false, 16); else LN5(false, 32); }
#undef LN5
    SDXE_LAUNCH_CHECK();
    return 0;
  }
  const int blocks = (rows + 7) / 8;  // 8 warps (rows) per block
  const int nv = (c / 8 + 31) / 32;   // vectors per lane
#define LN_LAUNCH(B, MV) layer_norm_kernel<B, MV><<<blocks, 256, 0, s>>>((const uint4*)x, gamma, beta, (uint4*)out, rows, c, eps)
  if (bf16) { if (nv <= 2) LN_LAUNCH(true, 2); else if (nv <= 3) LN_LAUNCH(true, 3); else if (nv <= 5) LN_LAUNCH(true, 5); else LN_LAUNCH(true, 8); }
  else { if (nv <= 2) LN_LAUNCH(false, 2); else if (nv <= 3) LN_LAUNCH(false, 3); else if (nv <= 5) LN_LAUNCH(false, 5); else LN_LAUNCH(false, 8); }
#undef LN_LAUNCH
  SDXE_LAUNCH_CHECK();
  return 0;
}

// =============================================================================================================
// gathers
// =============================================================================================================
__global__ void im2col3x3_kernel(const uint4* __restrict__ x, uint4* __restrict__ A, int n, int H, int W, int C, int Ho,
                                 int Wo, int stride, int pad_lo, int kpad) {
  const int KV = kpad >> 3;
  const size_t total = (size_t)n * Ho * Wo * KV;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int kv = (int)(idx % KV);
    const size_t m = idx / KV;
    const int k = kv * 8;
    const int tap = k / C, c = k - tap * C;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (tap < 9) {
      const int wo = (int)(m % Wo);
      const int ho = (int)((m / Wo) % Ho);
      const int img = (int)(m / ((size_t)Wo * Ho));
      const int dy = tap / 3, dx = tap - dy * 3;
      const int hi = ho * stride + dy - pad_lo, wi = wo * stride + dx - pad_lo;
      if (hi >= 0 && hi < H && wi >= 0 && wi < W) val = __ldg(x + (((size_t)img * H + hi) * W + wi) * (C >> 3) + (c >> 3));
    }
    A[idx] = val;
  }
}

int im2col3x3_launch(const void* x, void* A, int n, int H, int W, int C, int Ho, int Wo, int stride, int pad_lo,
                     int kpad, bool, cudaStream_t s) {
  if (C % 8 || kpad % 8) { set_last_error(__FILE__, __LINE__, "im2col: alignment"); return -1; }
  const size_t total = (size_t)n * Ho * Wo * (kpad / 8);
  const int blocks = (int)std::min<size_t>((total + 255) / 256, (size_t)num_sms() * 16);
  im2col3x3_kernel<<<blocks, 256, 0, s>>>((const uint4*)x, (uint4*)A, n, H, W, C, Ho, Wo, stride, pad_lo, kpad);
  SDXE_LAUNCH_CHECK();
  return 0;
}

template <bool BF16>
__global__ void im2col3x3_nchw_kernel(const void* __restrict__ x, int io_dtype, uint4* __restrict__ A, int n, int C,
                                      int H, int W, int kpad) {
  const size_t M = (size_t)n * H * W;
  const size_t m = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (m >= M) return;
  const int w = (int)(m % W), h = (int)((m / W) % H), img = (int)(m / ((size_t)W * H));
  for (int k0 = 0; k0 < kpad; k0 += 8) {
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = k0 + j;
      const int tap = k / C, c = k - tap * C;
      float val = 0.f;
      if (tap < 9) {
        const int dy = tap / 3, dx = tap - dy * 3;
        const int hi = h + dy - 1, wi = w + dx - 1;
        if (hi >= 0 && hi < H && wi >= 0 && wi < W) val = load_any(x, io_dtype, (((int64_t)img * C + c) * H + hi) * W + wi);
      }
      v[j] = val;
    }
    A[m * (kpad >> 3) + (k0 >> 3)] = pack8<BF16>(v);
  }
}

int im2col3x3_nchw_launch(const void* x, int io_dtype, void* A, int n, int C, int H, int W, int kpad, bool bf16,
                          cudaStream_t s) {
  const size_t M = (size_t)n * H * W;
  const int blocks = (int)((M + 127) / 128);
  if (bf16) im2col3x3_nchw_kernel<true><<<blocks, 128, 0, s>>>(x, io_dtype, (uint4*)A, n, C, H, W, kpad);
  else im2col3x3_nchw_kernel<false><<<blocks, 128, 0, s>>>(x, io_dtype, (uint4*)A, n, C, H, W, kpad);
  SDXE_LAUNCH_CHECK();
  return 0;
}

__global__ void upsample2x_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int n, int H, int W, int V) {
  const size_t total = (size_t)n * 2 * H * 2 * W * V;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int v = (int)(idx % V);
    size_t p = idx / V;
    const int wo = (int)(p % (2 * W));
    p /= 2 * W;
    const int ho = (int)(p % (2 * H));
    const int img = (int)(p / (2 * H));
    out[idx] = __ldg(x + (((size_t)img * H + (ho >> 1)) * W + (wo >> 1)) * V + v);
  }
}

int upsample2x_launch(const void* x, void* out, int n, int H, int W, int C, cudaStream_t s) {
  const size_t total = (size_t)n * 4 * H * W * (C / 8);
  const int blocks = (int)std::min<size_t>((total + 255) / 256, (size_t)num_sms() * 16);
  upsample2x_kernel<<<blocks, 256, 0, s>>>((const uint4*)x, (uint4*)out, n, H, W, C / 8);
  SDXE_LAUNCH_CHECK();
  return 0;
}

template <bool BF16>
__global__ void nhwc_to_nchw_kernel(const typename T16<BF16>::type* __restrict__ in, int ld, void* __restrict__ out,
                                    int io_dtype, int n, int C, int hw) {
  const size_t total = (size_t)n * C * hw;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int p = (int)(idx % hw);
    const int c = (int)((idx / hw) % C);
    const int img = (int)(idx / ((size_t)hw * C));
    store_any(out, io_dtype, (int64_t)idx, T16<BF16>::to_f(in[((size_t)img * hw + p) * ld + c]));
  }
}

int nhwc_to_nchw_launch(const void* in, int ld, void* out, int io_dtype, int n, int C, int hw, bool bf16, cudaStream_t s) {
  const size_t total = (size_t)n * C * hw;
  const int blocks = (int)std::min<size_t>((total + 255) / 256, (size_t)num_sms() * 16);
  if (bf16) nhwc_to_nchw_kernel<true><<<blocks, 256, 0, s>>>((const __nv_bfloat16*)in, ld, out, io_dtype, n, C, hw);
  else nhwc_to_nchw_kernel<false><<<blocks, 256, 0, s>>>((const __half*)in, ld, out, io_dtype, n, C, hw);
  SDXE_LAUNCH_CHECK();
  return 0;
}

template <bool BF16>
__global__ void cast_rows_kernel(const void* __restrict__ src, int src_dtype, typename T16<BF16>::type* __restrict__ dst,
                                 int64_t rows, int cols, int ldo) {
  const int64_t total = rows * cols;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / cols;
    const int c = (int)(idx - r * cols);
    dst[r * ldo + c] = T16<BF16>::from_f(load_any(src, src_dtype, idx));
  }
}

int cast_rows_launch(const void* src, int src_dtype, void* dst, int64_t rows, int cols, int ldo, bool bf16, cudaStream_t s) {
  const int64_t total = rows * cols;
  if (total == 0) return 0;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)num_sms() * 16);
  if (bf16) cast_rows_kernel<true><<<blocks, 256, 0, s>>>(src, src_dtype, (__nv_bfloat16*)dst, rows, cols, ldo);
  else cast_rows_kernel<false><<<blocks, 256, 0, s>>>(src, src_dtype, (__half*)dst, rows, cols, ldo);
  SDXE_LAUNCH_CHECK();
  return 0;
}


// =============================================================================================================
// embeddings
// =============================================================================================================
template <bool BF16>
__global__ void timestep_embedding_kernel(const void* __restrict__ t, int t_dtype, float* __restrict__ out, int m, int dim) {
  const int half = dim / 2;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= m * half) return;
  const int row = idx / half, j = idx - row * half;
  const float tv = load_any(t, t_dtype, row);
  const float freq = expf(-logf(10000.f) * (float)j / (float)half);
  const float arg = tv * freq;
  out[(size_t)row * dim + j] = round16<BF16>(cosf(arg));
  out[(size_t)row * dim + half + j] = round16<BF16>(sinf(arg));
}

int timestep_embedding_launch(const void* t, int t_dtype, float* out, int m, int dim, bool bf16, cudaStream_t s) {
  const int total = m * (dim / 2);
  const int blocks = (total + 127) / 128;
  if (bf16) timestep_embedding_kernel<true><<<blocks, 128, 0, s>>>(t, t_dtype, out, m, dim);
  else timestep_embedding_kernel<false><<<blocks, 128, 0, s>>>(t, t_dtype, out, m, dim);
  SDXE_LAUNCH_CHECK();
  return 0;
}

// Skinny linear (a handful of rows against a wide weight matrix: time_embed, label_emb, all emb_layers in one launch):
// out[M <= 16 per pass, N] = in[M, K] (fp32 holding 16-bit values) x W[N, K]^T. Sixteen rows are exactly one m16n8k16
// warp-MMA tile — far below wgmma's 64-row minimum, so this one op uses mma.sync: the kernel only has to stream the
// weight matrix once at HBM speed. A block stages its 16 input rows in shared memory as 16-bit (lossless: every producer
// rounds to the model dtype); each warp owns 8 output features; per 32 k a lane reads ONE 16-byte weight vector (its
// feature gid, k = 32 s + 8 tig .. + 7) and two 16-byte activation vectors (rows gid, gid + 8, same k) and issues two
// MMAs — the k index inside a 32-block is permuted identically for both operands, which a dot product does not see.
constexpr int SKL_WARPS = 8;
template <bool BF16>
SDXE_DEVINL void mma_16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  if (BF16)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
template <bool BF16>
__global__ void __launch_bounds__(SKL_WARPS * 32)
skinny_linear_kernel(const float* __restrict__ in, int ldi, const uint4* __restrict__ W, const float* __restrict__ b,
                     const float* add, float* out, int ldo, int M, int N, int K, int silu_out) {
  extern __shared__ __align__(16) uint8_t skl_in[];  // [16][row_bytes] 16-bit activations, K zero-padded to a multiple of 32
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gid = lane >> 2, tig = lane & 3;
  const int n0 = (blockIdx.x * SKL_WARPS + warp) * 8;
  const int Kp = (K + 31) & ~31;
  const int row_bytes = ((Kp * 2 + 127) & ~127) + 64;  // = 64 mod 128: the 8 lanes of an LDS.128 phase (2 rows x 4 pieces) hit 8 distinct 16-byte bank groups
  const int KV = K >> 3;
  for (int m0 = 0; m0 < M; m0 += 16) {
    __syncthreads();  // the previous row tile is no longer read
    for (int idx = threadIdx.x; idx < 16 * (Kp >> 2); idx += blockDim.x) {
      const int r = idx / (Kp >> 2), c = idx - r * (Kp >> 2);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m0 + r < M && c * 4 < K) v = __ldg(reinterpret_cast<const float4*>(in + (size_t)(m0 + r) * ldi) + c);
      uint2 u;
      u.x = T16<BF16>::pack(v.x, v.y);
      u.y = T16<BF16>::pack(v.z, v.w);
      *reinterpret_cast<uint2*>(skl_in + (size_t)r * row_bytes + c * 8) = u;
    }
    __syncthreads();
    if (n0 < N) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      const bool col_ok = n0 + gid < N;
      const uint4* wrow = W + (size_t)(col_ok ? n0 + gid : n0) * KV;
      const uint8_t* a_lo = skl_in + (size_t)gid * row_bytes + tig * 16;
      const uint8_t* a_hi = a_lo + 8 * (size_t)row_bytes;
      const int steps = Kp >> 5;
#pragma unroll 4
      for (int s = 0; s < steps; ++s) {
        const int kv = s * 4 + tig;  // this lane's 16-byte weight vector (8 k) of the 32-k block
        uint4 w = make_uint4(0u, 0u, 0u, 0u);
        if (kv < KV) w = __ldg(wrow + kv);
        const uint4 lo = *reinterpret_cast<const uint4*>(a_lo + s * 64);
        const uint4 hi = *reinterpret_cast<const uint4*>(a_hi + s * 64);
        mma_16816<BF16>(acc, lo.x, hi.x, lo.y, hi.y, w.x, w.y);
        mma_16816<BF16>(acc, lo.z, hi.z, lo.w, hi.w, w.z, w.w);
      }
      // c0, c1: (row gid, features n0 + 2 tig, + 1); c2, c3: row gid + 8
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int r = m0 + gid + (q >> 1) * 8, n = n0 + tig * 2 + (q & 1);
        if (r < M && n < N) {
          float v = round16<BF16>(acc[q] + (b ? __ldg(b + n) : 0.f));
          if (add) v = round16<BF16>(v + add[(size_t)r * ldo + n]);
          if (silu_out) v = round16<BF16>(silu_f(v));  // the only consumer applies SiLU first (emb_layers / time_embed)
          out[(size_t)r * ldo + n] = v;
        }
      }
    }
  }
}

static int skinny_linear_init() {
  SDXE_CUDA_CHECK(cudaFuncSetAttribute(skinny_linear_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  SDXE_CUDA_CHECK(cudaFuncSetAttribute(skinny_linear_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  return 0;
}

int skinny_linear_launch(const float* in, int ldi, const void* W, const float* b, const float* add, float* out, int ldo,
                         int M, int N, int K, bool silu_out, bool bf16, cudaStream_t s) {
  if (K % 8 || ldi % 4) { set_last_error(__FILE__, __LINE__, "skinny_linear: K % 8"); return -1; }
  if (kernels_init() != 0) return -1;
  const int Kp = (K + 31) & ~31;
  const size_t smem = 16 * (size_t)(((Kp * 2 + 127) & ~127) + 64);
  if (smem > 200 * 1024) { set_last_error(__FILE__, __LINE__, "skinny_linear: K too large for the activation stage"); return -1; }
  const int blocks = (N + 8 * SKL_WARPS - 1) / (8 * SKL_WARPS);
  if (bf16)
    skinny_linear_kernel<true><<<blocks, SKL_WARPS * 32, smem, s>>>(in, ldi, (const uint4*)W, b, add, out, ldo, M, N, K, silu_out ? 1 : 0);
  else
    skinny_linear_kernel<false><<<blocks, SKL_WARPS * 32, smem, s>>>(in, ldi, (const uint4*)W, b, add, out, ldo, M, N, K, silu_out ? 1 : 0);
  SDXE_LAUNCH_CHECK();
  return 0;
}

template <bool BF16>
__global__ void cast_to_f32_kernel(const void* __restrict__ src, int src_dtype, float* __restrict__ dst, int64_t n, int r16) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = load_any(src, src_dtype, i);
    dst[i] = r16 ? round16<BF16>(v) : v;
  }
}

int cast_to_f32_launch(const void* src, int src_dtype, float* dst, int64_t n, bool r16, bool bf16, cudaStream_t s) {
  if (n == 0) return 0;
  const int blocks = (int)std::min<int64_t>((n + 255) / 256, (int64_t)num_sms() * 8);
  if (bf16) cast_to_f32_kernel<true><<<blocks, 256, 0, s>>>(src, src_dtype, dst, n, r16 ? 1 : 0);
  else cast_to_f32_kernel<false><<<blocks, 256, 0, s>>>(src, src_dtype, dst, n, r16 ? 1 : 0);
  SDXE_LAUNCH_CHECK();
  return 0;
}

// =============================================================================================================
// weight repack
// =============================================================================================================
template <bool BF16>
__global__ void pack_weight_kernel(const void* __restrict__ src, int src_dtype, typename T16<BF16>::type* __restrict__ dst,
                                   int mode, int rows, int cols, int ld, int tile) {
  // `cols` = logical K of the destination row (CONV3: 9 * Cin)
  const int64_t total = (int64_t)rows * cols;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(idx / cols), k = (int)(idx - (int64_t)r * cols);
    int64_t si;
    if (mode == PACK_CONV3) {
      const int cin = cols / 9;
      const int tap = k / cin, c = k - tap * cin;
      si = ((int64_t)r * cin + c) * 9 + tap;  // [Cout, Cin, 3, 3]
    } else if (mode == PACK_GEGLU) {
      const int half_rows = rows / 2, half_tile = tile / 2;
      const int t = r / tile, rr = r - t * tile;
      const int sr = rr < half_tile ? t * half_tile + rr : half_rows + t * half_tile + (rr - half_tile);
      si = (int64_t)sr * cols + k;
    } else {
      si = idx;
    }
    dst[(int64_t)r * ld + k] = T16<BF16>::from_f(load_any(src, src_dtype, si));
  }
}

int pack_weight_launch(const void* src, int src_dtype, void* dst, int mode, int rows, int cols, int ld, int tile,
                       bool bf16, cudaStream_t s) {
  const int64_t total = (int64_t)rows * cols;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)num_sms() * 16);
  if (bf16) pack_weight_kernel<true><<<blocks, 256, 0, s>>>(src, src_dtype, (__nv_bfloat16*)dst, mode, rows, cols, ld, tile);
  else pack_weight_kernel<false><<<blocks, 256, 0, s>>>(src, src_dtype, (__half*)dst, mode, rows, cols, ld, tile);
  SDXE_LAUNCH_CHECK();
  return 0;
}

template <bool BF16>
__global__ void pack_vector_kernel(const void* __restrict__ src, int src_dtype, float* __restrict__ dst, int n, int tile, int r16) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int si = i;
  if (tile > 0) {
    const int half_rows = n / 2, half_tile = tile / 2;
    const int t = i / tile, rr = i - t * tile;
    si = rr < half_tile ? t * half_tile + rr : half_rows + t * half_tile + (rr - half_tile);
  }
  float v = load_any(src, src_dtype, si);
  dst[i] = r16 ? round16<BF16>(v) : v;
}

int pack_vector_launch(const void* src, int src_dtype, float* dst, int n, int geglu_tile, bool r16, bool bf16, cudaStream_t s) {
  const int blocks = (n + 255) / 256;
  if (bf16) pack_vector_kernel<true><<<blocks, 256, 0, s>>>(src, src_dtype, dst, n, geglu_tile, r16 ? 1 : 0);
  else pack_vector_kernel<false><<<blocks, 256, 0, s>>>(src, src_dtype, dst, n, geglu_tile, r16 ? 1 : 0);
  SDXE_LAUNCH_CHECK();
  return 0;
}

// LayerNorm folded into the consuming GEMM (gemm.cuh): per output row n of a packed weight [rows, ld]
//   bias'[n] = bias[n] + sum_k beta[k] W[n, k];  W'[n, k] = round16(W[n, k] * gamma[k]) (in place);  c1[n] = sum_k W'[n, k]
// Row interleaving (GEGLU packing) is irrelevant: gamma / beta run along K, bias / c1 are indexed like the packed rows.
template <bool BF16>
__global__ void ln_fold_kernel(typename T16<BF16>::type* __restrict__ w, int rows, int K, int ld,
                               const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ bias,
                               float* __restrict__ c1) {
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (n >= rows) return;
  typename T16<BF16>::type* wr = w + (size_t)n * ld;
  float sb = 0.f, sc = 0.f;
  for (int k = lane; k < K; k += 32) {
    const float wv = T16<BF16>::to_f(wr[k]);
    sb = fmaf(beta[k], wv, sb);
    const typename T16<BF16>::type wf = T16<BF16>::from_f(wv * gamma[k]);
    wr[k] = wf;
    sc += T16<BF16>::to_f(wf);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sb += __shfl_xor_sync(0xffffffffu, sb, o);
    sc += __shfl_xor_sync(0xffffffffu, sc, o);
  }
  if (lane == 0) {
    bias[n] += sb;
    c1[n] = sc;
  }
}
int ln_fold_launch(void* w, int rows, int K, int ld, const float* gamma, const float* beta, float* bias, float* c1, bool bf16,
                   cudaStream_t s) {
  const int blocks = (rows * 32 + 255) / 256;
  if (bf16) ln_fold_kernel<true><<<blocks, 256, 0, s>>>((__nv_bfloat16*)w, rows, K, ld, gamma, beta, bias, c1);
  else ln_fold_kernel<false><<<blocks, 256, 0, s>>>((__half*)w, rows, K, ld, gamma, beta, bias, c1);
  SDXE_LAUNCH_CHECK();
  return 0;
}

// =============================================================================================================
// CLIP text encoder pieces (row N4: FrozenCLIPEmbedder / FrozenOpenCLIPEmbedder2 `transformer`,
// modules/sd_hijack_clip.py:351-360, modules/sd_hijack_open_clip.py:29-71). 77-token sequences: launch-latency-sized
// work, so plain CUDA-core kernels; the projections run on the wgmma GEMM with the LayerNorms folded in.
// =============================================================================================================
// x[m, :] = round16(tok[ids[m], :] + pos[m % T, :]); also the row's (sum, sum of squares) for the first folded LayerNorm.
template <bool BF16>
__global__ void clip_embed_kernel(const int32_t* __restrict__ ids, const typename T16<BF16>::type* __restrict__ tok,
                                  const typename T16<BF16>::type* __restrict__ pos, typename T16<BF16>::type* __restrict__ x,
                                  float2* __restrict__ stat, int M, int T, int C, int vocab) {
  const int m = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (m >= M) return;
  int id = ids[m];
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  const typename T16<BF16>::type* tr = tok + (size_t)id * C;
  const typename T16<BF16>::type* pr = pos + (size_t)(m % T) * C;
  float s = 0.f, q = 0.f;
  for (int c = lane; c < C; c += 32) {
    const typename T16<BF16>::type v = T16<BF16>::from_f(T16<BF16>::to_f(tr[c]) + T16<BF16>::to_f(pr[c]));
    x[(size_t)m * C + c] = v;
    const float f = T16<BF16>::to_f(v);
    s += f;
    q = fmaf(f, f, q);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if (lane == 0) stat[m] = make_float2(s, q);
}
int clip_embed_launch(const int32_t* ids, const void* tok, const void* pos, void* x, float2* stat, int M, int T, int C, int vocab,
                      bool bf16, cudaStream_t s) {
  const int blocks = (M * 32 + 255) / 256;
  if (bf16) clip_embed_kernel<true><<<blocks, 256, 0, s>>>(ids, (const __nv_bfloat16*)tok, (const __nv_bfloat16*)pos, (__nv_bfloat16*)x, stat, M, T, C, vocab);
  else clip_embed_kernel<false><<<blocks, 256, 0, s>>>(ids, (const __half*)tok, (const __half*)pos, (__half*)x, stat, M, T, C, vocab);
  SDXE_LAUNCH_CHECK();
  return 0;
}

// Textual-inversion "fixes" (modules/sd_hijack.py:340-366 EmbeddingsWithFixes): row rows[i] of the token embedding is replaced by
// the learned vector vec[i] before the position embedding is added: x[row, :] = round16(vec[i, :] + pos[row % T, :]), and
// the row's LayerNorm partial is recomputed. One warp per fix; a row named twice takes the LAST vector (fixes apply in order).
template <bool BF16>
__global__ void clip_fix_kernel(const int32_t* __restrict__ rows, const typename T16<BF16>::type* __restrict__ vec,
                                const typename T16<BF16>::type* __restrict__ pos, typename T16<BF16>::type* __restrict__ x,
                                float2* __restrict__ stat, int n_fix, int M, int T, int C) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= n_fix) return;
  const int m = rows[i];
  if (m < 0 || m >= M) return;
  for (int j = i + 1; j < n_fix; ++j)
    if (rows[j] == m) return;  // a later fix owns this row
  const typename T16<BF16>::type* vr = vec + (size_t)i * C;
  const typename T16<BF16>::type* pr = pos + (size_t)(m % T) * C;
  float s = 0.f, q = 0.f;
  for (int c = lane; c < C; c += 32) {
    const typename T16<BF16>::type v = T16<BF16>::from_f(T16<BF16>::to_f(vr[c]) + T16<BF16>::to_f(pr[c]));
    x[(size_t)m * C + c] = v;
    const float f = T16<BF16>::to_f(v);
    s += f;
    q = fmaf(f, f, q);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if (lane == 0) stat[m] = make_float2(s, q);
}
int clip_fix_launch(const int32_t* rows, const void* vec, const void* pos, void* x, float2* stat, int n_fix, int M, int T, int C,
                    bool bf16, cudaStream_t s) {
  if (n_fix <= 0) return 0;
  const int blocks = (n_fix * 32 + 255) / 256;
  if (bf16) clip_fix_kernel<true><<<blocks, 256, 0, s>>>(rows, (const __nv_bfloat16*)vec, (const __nv_bfloat16*)pos, (__nv_bfloat16*)x, stat, n_fix, M, T, C);
  else clip_fix_kernel<false><<<blocks, 256, 0, s>>>(rows, (const __half*)vec, (const __half*)pos, (__half*)x, stat, n_fix, M, T, C);
  SDXE_LAUNCH_CHECK();
  return 0;
}

// Causal self-attention over short sequences: qkv [B*T, 3C] (q | k | v, heads contiguous inside each), one CTA per
// (batch, head), K and V of the head in shared memory, one warp per query row (token t attends to tokens <= t), fp32 math.
template <bool BF16>
__global__ void __launch_bounds__(128) causal_attn_small_kernel(const typename T16<BF16>::type* __restrict__ qkv,
                                                                typename T16<BF16>::type* __restrict__ out, int T, int H, int d, float scale) {
  extern __shared__ float sm[];
  const int C = H * d, ld = 3 * C;
  const int b = blockIdx.x / H, h = blockIdx.x - b * H;
  float* sK = sm;                    // [T][d + 1]
  float* sV = sm + T * (d + 1);      // [T][d]
  float* sQ = sV + T * d;            // [4 warps][d]
  float* sP = sQ + 4 * d;            // [4 warps][T]
  const typename T16<BF16>::type* base = qkv + (size_t)b * T * ld + h * d;
  for (int i = threadIdx.x; i < T * d; i += blockDim.x) {
    const int t = i / d, c = i - t * d;
    sK[t * (d + 1) + c] = T16<BF16>::to_f(base[(size_t)t * ld + C + c]);
    sV[t * d + c] = T16<BF16>::to_f(base[(size_t)t * ld + 2 * C + c]);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* q = sQ + warp * d;
  float* p = sP + warp * T;
  for (int r = warp; r < T; r += 4) {
    for (int c = lane; c < d; c += 32) q[c] = T16<BF16>::to_f(base[(size_t)r * ld + c]) * scale;
    __syncwarp();
    float mx = -INFINITY;
    for (int j = lane; j <= r; j += 32) {
      float a = 0.f;
      for (int c = 0; c < d; ++c) a = fmaf(q[c], sK[j * (d + 1) + c], a);
      p[j] = a;
      mx = fmaxf(mx, a);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int j = lane; j <= r; j += 32) {
      const float e = __expf(p[j] - mx);
      p[j] = e;
      sum += e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    __syncwarp();
    const float inv = 1.f / sum;
    for (int c = lane; c < d; c += 32) {
      float a = 0.f;
      for (int j = 0; j <= r; ++j) a = fmaf(p[j], sV[j * d + c], a);
      out[((size_t)b * T + r) * C + h * d + c] = T16<BF16>::from_f(a * inv);
    }
    __syncwarp();
  }
}
int causal_attn_small_launch(const void* qkv, void* out, int B, int T, int H, int d, float scale, bool bf16, cudaStream_t s) {
  const size_t smem = sizeof(float) * ((size_t)T * (d + 1) + (size_t)T * d + 4 * d + 4 * T);
  if (smem > 96 * 1024) { set_last_error(__FILE__, __LINE__, "causal_attn_small: sequence too long"); return -1; }
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(causal_attn_small_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    cudaFuncSetAttribute(causal_attn_small_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    attr = true;
  }
  if (bf16) causal_attn_small_kernel<true><<<B * H, 128, smem, s>>>((const __nv_bfloat16*)qkv, (__nv_bfloat16*)out, T, H, d, scale);
  else causal_attn_small_kernel<false><<<B * H, 128, smem, s>>>((const __half*)qkv, (__half*)out, T, H, d, scale);
  SDXE_LAUNCH_CHECK();
  return 0;
}

// in place: mode 0 quick_gelu x * sigmoid(1.702 x) (CLIP-L), mode 1 erf GELU (OpenCLIP bigG)
template <bool BF16>
__global__ void act_inplace_kernel(typename T16<BF16>::type* __restrict__ x, int64_t n, int mode) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = T16<BF16>::to_f(x[i]);
    const float y = mode == 0 ? v / (1.f + __expf(-1.702f * v)) : gelu_erf_f(v);
    x[i] = T16<BF16>::from_f(y);
  }
}
int act_inplace_launch(void* x, int64_t n, int mode, bool bf16, cudaStream_t s) {
  const int blocks = (int)std::min<int64_t>((n + 255) / 256, (int64_t)num_sms() * 8);
  if (bf16) act_inplace_kernel<true><<<blocks, 256, 0, s>>>((__nv_bfloat16*)x, n, mode);
  else act_inplace_kernel<false><<<blocks, 256, 0, s>>>((__half*)x, n, mode);
  SDXE_LAUNCH_CHECK();
  return 0;
}

// =============================================================================================================
// sampler-step fusions (latents stay fp32, as in the reference: x comes from torch.randn fp32, modules/rng.py:19)
// =============================================================================================================
__global__ void denoiser_in_kernel(const float* __restrict__ x, const int32_t* __restrict__ src,
                                   const float* __restrict__ c_in, void* __restrict__ x_in, int rows, int64_t elems,
                                   int out_dtype) {
  const int64_t total = rows * elems;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(idx / elems);
    const int64_t e = idx - r * elems;
    store_any(x_in, out_dtype, idx, x[(int64_t)src[r] * elems + e] * c_in[r]);
  }
}

int denoiser_in_launch(const float* x, const int32_t* src, const float* c_in, void* x_in, int rows, int64_t elems,
                       int out_dtype, cudaStream_t s) {
  const int64_t total = rows * elems;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)num_sms() * 8);
  denoiser_in_kernel<<<blocks, 256, 0, s>>>(x, src, c_in, x_in, rows, elems, out_dtype);
  SDXE_LAUNCH_CHECK();
  return 0;
}

// rows [0,B): cond, [B,2B): uncond.  den_r = x_b + eps_r * (-sigma_b);  out_b = den_u + (den_c - den_u) * scale
__global__ void cfg_combine_kernel(const float* __restrict__ x, const void* __restrict__ eps,
                                   const float* __restrict__ sigma, float scale, float* __restrict__ out, int B,
                                   int64_t elems, int eps_dtype) {
  const int64_t total = B * elems;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(idx / elems);
    const float xv = x[idx], c_out = -sigma[b];
    const float dc = xv + load_any(eps, eps_dtype, idx) * c_out;
    const float du = xv + load_any(eps, eps_dtype, idx + total) * c_out;
    out[idx] = du + (dc - du) * scale;
  }
}

int cfg_combine_launch(const float* x, const void* eps, const float* sigma, float cond_scale, float* denoised, int B,
                       int64_t elems, int eps_dtype, cudaStream_t s) {
  const int64_t total = B * elems;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)num_sms() * 8);
  cfg_combine_kernel<<<blocks, 256, 0, s>>>(x, eps, sigma, cond_scale, denoised, B, elems, eps_dtype);
  SDXE_LAUNCH_CHECK();
  return 0;
}

// General CFG combine (sd_samplers_cfg_denoiser.py:74-82 with an arbitrary conds_list): image b owns the cond rows
// cond_rows[row_ptr[b] .. row_ptr[b+1]) of eps with weights cond_w[...] (already multiplied by cond_scale) and the uncond
// row uncond_row0 + b.  den_r = x_b + eps_r * (-sigma_b);  out_b = den_u + sum_k w_k (den_k - den_u).
__global__ void cfg_combine_multi_kernel(const float* __restrict__ x, const void* __restrict__ eps,
                                         const float* __restrict__ sigma, const int32_t* __restrict__ row_ptr,
                                         const int32_t* __restrict__ cond_rows, const float* __restrict__ cond_w,
                                         const int32_t* __restrict__ uncond_rows, float* __restrict__ out, int B,
                                         int64_t elems, int eps_dtype) {
  const int64_t total = B * elems;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(idx / elems);
    const int64_t e = idx - b * elems;
    const float xv = x[idx], c_out = -sigma[b];
    const float du = xv + load_any(eps, eps_dtype, (int64_t)uncond_rows[b] * elems + e) * c_out;
    float acc = du;
    for (int k = row_ptr[b]; k < row_ptr[b + 1]; ++k) {
      const float dc = xv + load_any(eps, eps_dtype, (int64_t)cond_rows[k] * elems + e) * c_out;
      acc += (dc - du) * cond_w[k];
    }
    out[idx] = acc;
  }
}

int cfg_combine_multi_launch(const float* x, const void* eps, const float* sigma, const int32_t* row_ptr,
                             const int32_t* cond_rows, const float* cond_w, const int32_t* uncond_rows, float* denoised,
                             int B, int64_t elems, int eps_dtype, cudaStream_t s) {
  const int64_t total = B * elems;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)num_sms() * 8);
  cfg_combine_multi_kernel<<<blocks, 256, 0, s>>>(x, eps, sigma, row_ptr, cond_rows, cond_w, uncond_rows, denoised, B, elems, eps_dtype);
  SDXE_LAUNCH_CHECK();
  return 0;
}

// CFG combine for denoisers whose per-row output is affine in (x_b, eps_r) with coefficients shared by all rows of image b
// (timestep denoisers: raw eps; LCM: c_out'(x - sigma eps) + c_skip' x). Then the guided output is also affine:
//   out_b = cx[b] x_b + ce[b] (e_u + sum_k w_k (e_k - e_u)).
// Optional side outputs, same pass: x0_out_b = x0_coef[2b] x_b + x0_coef[2b+1] e_{first cond row of b} (the timestep
// path's pred_x0, the sampler's last_latent) and uncond_out_b = e_u as fp32 (CFG++ steps along the uncond noise).
__global__ void cfg_combine_affine_kernel(const float* __restrict__ x, const void* __restrict__ eps,
                                          const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ cond_rows,
                                          const float* __restrict__ cond_w, const int32_t* __restrict__ uncond_rows,
                                          const float* __restrict__ cx, const float* __restrict__ ce, float* __restrict__ out,
                                          const float* __restrict__ x0_coef, float* __restrict__ x0_out,
                                          float* __restrict__ uncond_out, int B, int64_t elems, int eps_dtype) {
  const int64_t total = B * elems;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(idx / elems);
    const int64_t e = idx - b * elems;
    const float xv = x[idx];
    const float eu = load_any(eps, eps_dtype, (int64_t)uncond_rows[b] * elems + e);
    const int k0 = row_ptr[b], k1 = row_ptr[b + 1];
    float acc = eu;
    for (int k = k0; k < k1; ++k) acc += (load_any(eps, eps_dtype, (int64_t)cond_rows[k] * elems + e) - eu) * cond_w[k];
    out[idx] = cx[b] * xv + ce[b] * acc;
    if (x0_out) {
      const float e0 = load_any(eps, eps_dtype, (int64_t)cond_rows[k0] * elems + e);
      x0_out[idx] = x0_coef[2 * b] * xv + x0_coef[2 * b + 1] * e0;
    }
    if (uncond_out) uncond_out[idx] = eu;
  }
}

int cfg_combine_affine_launch(const float* x, const void* eps, const int32_t* row_ptr, const int32_t* cond_rows,
                              const float* cond_w, const int32_t* uncond_rows, const float* cx, const float* ce, float* out,
                              const float* x0_coef, float* x0_out, float* uncond_out, int B, int64_t elems, int eps_dtype,
                              cudaStream_t s) {
  const int64_t total = B * elems;
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)num_sms() * 8);
  cfg_combine_affine_kernel<<<blocks, 256, 0, s>>>(x, eps, row_ptr, cond_rows, cond_w, uncond_rows, cx, ce, out, x0_coef,
                                                   x0_out, uncond_out, B, elems, eps_dtype);
  SDXE_LAUNCH_CHECK();
  return 0;
}

// out = c0 p0 + c1 p1 + c2 p2 + c3 p3 (null pointers skipped; out may alias any input): the update of every k-diffusion
// sampler step is such a combination of x, denoised, a second denoised / derivative and noise, with host-side scalars.
__global__ void lincomb_kernel(float* __restrict__ out, const float* p0, float c0, const float* p1, float c1, const float* p2,
                               float c2, const float* p3, float c3, int64_t total) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float r = c0 * p0[i];
    if (p1) r = fmaf(c1, p1[i], r);
    if (p2) r = fmaf(c2, p2[i], r);
    if (p3) r = fmaf(c3, p3[i], r);
    out[i] = r;
  }
}
int lincomb_launch(float* out, const float* p0, float c0, const float* p1, float c1, const float* p2, float c2, const float* p3, float c3,
                   int64_t total, cudaStream_t s) {
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)num_sms() * 8);
  lincomb_kernel<<<blocks, 256, 0, s>>>(out, p0, c0, p1, c1, p2, c2, p3, c3, total);
  SDXE_LAUNCH_CHECK();
  return 0;
}

__global__ void euler_a_step_kernel(float* __restrict__ x, const float* __restrict__ den, const float* __restrict__ noise,
                                    float inv_sigma, float dt, float sigma_up, int64_t total) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const float xv = x[i];
    const float d = (xv - den[i]) * inv_sigma;
    float r = xv + d * dt;
    if (noise) r += noise[i] * sigma_up;
    x[i] = r;
  }
}

int euler_a_step_launch(float* x, const float* den, const float* noise, float sigma, float sigma_down, float sigma_up,
                        int64_t total, cudaStream_t s) {
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)num_sms() * 8);
  euler_a_step_kernel<<<blocks, 256, 0, s>>>(x, den, sigma_up > 0.f ? noise : nullptr, 1.f / sigma, sigma_down - sigma,
                                             sigma_up, total);
  SDXE_LAUNCH_CHECK();
  return 0;
}

__global__ void dpmpp_2m_step_kernel(float* __restrict__ x, const float* __restrict__ den, const float* __restrict__ old,
                                     float ratio, float neg_expm1, float c0, float c1, int64_t total) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float dd = c0 * den[i];
    if (old) dd += c1 * old[i];
    x[i] = ratio * x[i] + neg_expm1 * dd;
  }
}

int dpmpp_2m_step_launch(float* x, const float* den, const float* old, float ratio, float neg_expm1, float c0, float c1,
                         int64_t total, cudaStream_t s) {
  const int blocks = (int)std::min<int64_t>((total + 255) / 256, (int64_t)num_sms() * 8);
  dpmpp_2m_step_kernel<<<blocks, 256, 0, s>>>(x, den, c1 != 0.f ? old : nullptr, ratio, neg_expm1, c0, c1, total);
  SDXE_LAUNCH_CHECK();
  return 0;
}

}  // namespace sdxe
