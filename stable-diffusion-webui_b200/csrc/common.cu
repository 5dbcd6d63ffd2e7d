// Host-side helpers: last-error string, launch counter, TMA tensor-map encoding via the driver entry point, device query.
#include "common.cuh"
#include <cstdio>
#include <cstring>
#include <atomic>
#include <mutex>

namespace sdxe {

static thread_local char g_err[1024] = "";
static std::atomic<int64_t> g_launches{0};

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int64_t launch_count() { return g_launches.load(std::memory_order_relaxed); }

void set_last_error(const char* file, int line, const char* msg) {
  snprintf(g_err, sizeof(g_err), "%s:%d: %s", file, line, msg);
}
const char* last_error() { return g_err; }

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

static int encode(CUtensorMap* out, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                  const cuuint32_t* box) {
  PFN_encodeTiled fn = get_encode();
  if (!fn) { set_last_error(__FILE__, __LINE__, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)"); return -1; }
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides, box,
                  estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed: %d (rank %d dims %llu %llu box %u %u base %p)", (int)r,
             rank, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1], base);
    set_last_error(__FILE__, __LINE__, buf);
    return -1;
  }
  return 0;
}

int make_tmap_2d(CUtensorMap* out, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  return encode(out, base, 2, dims, strides, box);
}

int make_tmap_heads(CUtensorMap* out, const void* base, int64_t d, int64_t tokens, int64_t heads, int64_t batch,
                    int64_t tok_stride, int64_t head_stride, int64_t batch_stride, int box_rows) {
  cuuint64_t dims[4] = {(cuuint64_t)d, (cuuint64_t)tokens, (cuuint64_t)heads, (cuuint64_t)batch};
  cuuint64_t strides[3] = {(cuuint64_t)tok_stride * 2, (cuuint64_t)head_stride * 2, (cuuint64_t)batch_stride * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)box_rows, 1, 1};
  return encode(out, base, 4, dims, strides, box);
}
int make_tmap_nhwc(CUtensorMap* out, const void* base, int N, int H, int W, int C, int bw, int bh, int bn) {
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {64, (cuuint32_t)bw, (cuuint32_t)bh, (cuuint32_t)bn};
  return encode(out, base, 4, dims, strides, box);
}

// Stride-2 view of an NHWC activation (H, W even): [N, H/2, 2, W/2, 2C] — a pixel pair is one 2C-wide "pixel", a row pair
// one extra dimension of size 2. Tap (dy, dx) of a 3x3 stride-2 conv reads input pixel (2 oh + ty, 2 ow + tx) with
// t = d - pad_lo: row pair oh + (ty >> 1), row parity ty & 1, pixel pair ow + (tx >> 1), channel offset (tx & 1) * C — a
// plain box per tap, out-of-range pairs zero-filled (the conv's padding). box = 64 channels x bw pairs x 1 x bh x bn.
int make_tmap_nhwc_s2(CUtensorMap* out, const void* base, int N, int H, int W, int C, int bw, int bh, int bn) {
  cuuint64_t dims[5] = {(cuuint64_t)2 * C, (cuuint64_t)W / 2, 2, (cuuint64_t)H / 2, (cuuint64_t)N};
  cuuint64_t strides[4] = {(cuuint64_t)C * 4, (cuuint64_t)W * C * 2, (cuuint64_t)W * C * 4, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[5] = {64, (cuuint32_t)bw, 1, (cuuint32_t)bh, (cuuint32_t)bn};
  return encode(out, base, 5, dims, strides, box);
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return 132;
    n = p.multiProcessorCount;
  }
  return n;
}

}  // namespace sdxe
