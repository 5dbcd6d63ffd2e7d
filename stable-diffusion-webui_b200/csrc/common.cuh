// sm_90a device primitives shared by every kernel of the denoising engine:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma fences and shared-memory descriptors, and 16-bit pack helpers.
// Everything here is inline PTX; nothing is borrowed from a library at run time.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <cstdio>
#include <cstring>

namespace sdxe {

// ---------------------------------------------------------------------------------------------
// dtype tags (match include/sdxe.h)
// ---------------------------------------------------------------------------------------------
enum : int { DT_F16 = 0, DT_BF16 = 1, DT_F32 = 2 };

#define SDXE_DEVINL __device__ __forceinline__

SDXE_DEVINL uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
SDXE_DEVINL uint32_t lane_id() { return threadIdx.x & 31; }

SDXE_DEVINL bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
      "elect.sync rx|px, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, px;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---------------------------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------------------------
SDXE_DEVINL void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
SDXE_DEVINL void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
SDXE_DEVINL void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
SDXE_DEVINL void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
SDXE_DEVINL uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// Wait for the phase with the given parity to complete. A watchdog turns a protocol bug
// (wrong phase, missing arrive, bad TMA descriptor) into a trap instead of a hung GPU.
SDXE_DEVINL void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  uint64_t t0 = 0;
  for (uint32_t it = 0;; ++it) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}\n"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) return;
    if ((it & 0x3ff) == 0x3ff) {
      uint64_t now = global_timer_ns();
      if (t0 == 0) t0 = now;
      // 4 s. No printf: mbar_wait serves the wgmma kernels, and any function call in a kernel makes ptxas serialise all
      // of its wgmma (warning C7510, reported for every GEMM variant when the diagnostic printf was here)
      else if (now - t0 > 4000000000ull) __trap();
    }
  }
}

// Non-blocking probe of a phase (for a consumer that serves several producers in arrival order).
SDXE_DEVINL bool mbar_test(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}\n"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done != 0;
}

// generic-proxy smem writes -> visible to async proxy (TMA stores / wgmma operand reads)
SDXE_DEVINL void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// TMA loads (tile mode), completion on an mbarrier.
// ---------------------------------------------------------------------------------------------
SDXE_DEVINL void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
SDXE_DEVINL void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
SDXE_DEVINL void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
SDXE_DEVINL void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
SDXE_DEVINL void tma_load_5d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// TMA store smem -> global (bulk async-group completion). The issuing thread commits and later waits on its own groups.
SDXE_DEVINL void tma_store_2d(const CUtensorMap* m, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
SDXE_DEVINL void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
SDXE_DEVINL void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }  // smem reusable
SDXE_DEVINL void bulk_wait_read_1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }    // all but the newest group
SDXE_DEVINL void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }            // writes done

// ---------------------------------------------------------------------------------------------
// wgmma (sm_90a warpgroup MMA): fences and group completion. The MMA wrappers themselves are in wgmma.cuh.
// ---------------------------------------------------------------------------------------------
// orders this thread's register writes (accumulators, A fragments) before the next wgmma reads them
SDXE_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
SDXE_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> SDXE_DEVINL void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of an accumulator register across wgmma issue / wait
SDXE_DEVINL void reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// ---------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor (64 bit), 128B swizzle:
//   [0,14)  start address >> 4          [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset >> 4 [49,52) base offset = 0      [62,64) layout: 1 = 128B swizzle
//
// K-major (our A/B tiles: rows of 64 elements = 128 bytes, as TMA writes them): 8-row groups are 1024 B apart ->
// SBO = 1024; LBO unused (1). A K step of 16 elements (32 bytes, inside the swizzle atom) adds 2 to the address field.
// MN-major (V slabs: [kv rows][64 dv] with 128-byte rows, read transposed): 8-row groups along K are 1024 B apart ->
// SBO = 1024; LBO = distance between 64-element MN chunks (one slab here, so unused). 16 K rows add 128.
// ---------------------------------------------------------------------------------------------
SDXE_DEVINL uint64_t gmma_desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3fff);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32;
  d |= (uint64_t)1 << 62;  // SWIZZLE_128B
  return d;
}

// ---------------------------------------------------------------------------------------------
// 16-bit conversions, templated on the storage type
// ---------------------------------------------------------------------------------------------
template <bool BF16> struct T16;
template <> struct T16<false> {
  using type = __half;
  using type2 = __half2;
  static SDXE_DEVINL uint32_t pack(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  static SDXE_DEVINL float2 unpack(uint32_t u) { return __half22float2(*reinterpret_cast<__half2*>(&u)); }
  static SDXE_DEVINL float to_f(type v) { return __half2float(v); }
  static SDXE_DEVINL type from_f(float v) { return __float2half_rn(v); }
};
template <> struct T16<true> {
  using type = __nv_bfloat16;
  using type2 = __nv_bfloat162;
  static SDXE_DEVINL uint32_t pack(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  static SDXE_DEVINL float2 unpack(uint32_t u) { return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&u)); }
  static SDXE_DEVINL float to_f(type v) { return __bfloat162float(v); }
  static SDXE_DEVINL type from_f(float v) { return __float2bfloat16_rn(v); }
};

SDXE_DEVINL float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// 2^x on the FMA pipe (Cody-Waite: n = round(x) through the 1.5 * 2^23 magic add, r = x - n in [-0.5, 0.5], degree-3
// minimax polynomial for 2^r, 2^n through the exponent field). Max relative error 7.5e-5 — below half an ulp of fp16
// (2.4e-4) and far below bf16's (2e-3): used for a fraction of the softmax exponentials so that the MUFU pipe
// (16 ex2 / clk / SM) is not the only unit doing them (the FA-4 trick). x <= ~100; x -> -inf gives 2^-125 (~0).
SDXE_DEVINL float ex2_poly3(float x) {
  x = fmaxf(x, -125.f);
  const float magic = 12582912.f;
  const float t = x + magic;
  const float r = x - (t - magic);
  float p = fmaf(0.0551716685295105f, r, 0.2426111400127411f);
  p = fmaf(p, r, 0.6932609677314758f);
  p = fmaf(p, r, 0.9999280571937561f);
  return __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23));
}
SDXE_DEVINL float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
SDXE_DEVINL float silu_f(float x) { return x * rcp_approx(1.f + ex2_approx(-1.4426950408889634f * x)); }
SDXE_DEVINL float gelu_erf_f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
// erf-GELU with erf from Abramowitz-Stegun 7.1.26 (|abs err| < 1.5e-7, far below 16-bit output resolution):
// one MUFU.EX2, one MUFU.RCP and a handful of FMAs instead of libdevice erff's branchy ~30 instructions.
// With erf(|z|) = 1 - P(t) e^{-z^2}, t = 1 / (1 + p |z|), z = x / sqrt 2:
//   gelu(x) = x/2 (1 + erf z) = max(x, 0) - |x|/2 P(t) e^{-z^2}        (both signs of x)
// and with u = x sqrt(log2(e) / 2) (so that e^{-z^2} = 2^{-u^2}) the constants |z| / |u| and |x| / (2 |u|) fold into p and
// into P's coefficients: 11 FP32-pipe instructions + 2 MUFU per element (the textbook arrangement below took 15 + 2, and
// the GEGLU epilogue is instruction-bound).
#ifndef SDXE_GELU_V1
SDXE_DEVINL float gelu_fast_f(float x) {
  constexpr float C = 0.84932180028801904f;        // sqrt(log2(e) / 2)
  constexpr float S = 0.83255461115769776f;        // |z| / |u| = 1 / sqrt(log2(e))
  constexpr float H = 0.58870501125773735f;        // |x| / (2 |u|) = 1 / (2 C)
  const float u = x * C;
  const float a = fabsf(u);
  const float t = rcp_approx(fmaf(0.3275911f * S, a, 1.f));
  float p = fmaf(1.061405429f * H, t, -1.453152027f * H);
  p = fmaf(p, t, 1.421413741f * H);
  p = fmaf(p, t, -0.284496736f * H);
  p = fmaf(p, t, 0.254829592f * H);
  const float e = ex2_approx(-u * u);
  return fmaf(-(a * e), p * t, fmaxf(x, 0.f));
}
#else
SDXE_DEVINL float gelu_fast_f(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  const float t = rcp_approx(fmaf(0.3275911f, z, 1.f));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = ex2_approx(-z * z * 1.4426950408889634f);
  const float erf_abs = fmaf(-p * t, e, 1.f);          // erf(|x|/sqrt2)
  const float erfv = copysignf(erf_abs, x);
  return 0.5f * x * (1.f + erfv);
}
#endif

// ---------------------------------------------------------------------------------------------
// host: error handling + tensor-map encoding through the driver entry point (no -lcuda link)
// ---------------------------------------------------------------------------------------------
#define SDXE_CUDA_CHECK(expr)                                                         \
  do {                                                                                \
    cudaError_t _e = (expr);                                                          \
    if (_e != cudaSuccess) {                                                          \
      ::sdxe::set_last_error(__FILE__, __LINE__, cudaGetErrorString(_e));             \
      return -1;                                                                      \
    }                                                                                 \
  } while (0)

void set_last_error(const char* file, int line, const char* msg);
const char* last_error();

// 16-bit row-major 2D [rows, cols] with row pitch ld (elements): box = 64 cols x box_rows, 128B swizzle.
int make_tmap_2d(CUtensorMap* out, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows);
// per-head view of a row-major activation: element (j, tok, h, b) at base + b*batch_stride + tok*tok_stride + h*head_stride
// + j (strides in elements, multiples of 8). Inner extent d (NOT padded): a 64-wide box past d is zero-filled by TMA.
int make_tmap_heads(CUtensorMap* out, const void* base, int64_t d, int64_t tokens, int64_t heads, int64_t batch,
                    int64_t tok_stride, int64_t head_stride, int64_t batch_stride, int box_rows);
// 16-bit NHWC activations [N, H, W, C]: box = 64 ch x bw x bh x bn, 128B swizzle, OOB -> zero (= conv padding).
int make_tmap_nhwc(CUtensorMap* out, const void* base, int N, int H, int W, int C, int bw, int bh, int bn);
int make_tmap_nhwc_s2(CUtensorMap* out, const void* base, int N, int H, int W, int C, int bw, int bh, int bn);

int num_sms();

// Kernels launched by this library (sdxe_launch_count). Every launch site counts itself once, through SDXE_LAUNCH_CHECK;
// a replayed CUDA graph adds the count its capture recorded.
void count_launch(int n = 1);
int64_t launch_count();

#define SDXE_LAUNCH_CHECK()                 \
  do {                                      \
    ::sdxe::count_launch();                 \
    SDXE_CUDA_CHECK(cudaGetLastError());    \
  } while (0)

}  // namespace sdxe
