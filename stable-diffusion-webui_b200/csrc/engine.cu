// The denoising engine: weight ingestion / repack, static execution plans (one per input shape, replayed as a CUDA
// graph) for the UNet forward and the VAE decoder, and their C-ABI entry points (include/sdxe.h).
//
// Replaces, behind modules/sd_unet.py:75-77 (SdUnet.forward) and modules/sd_samplers_common.py:58
// (decode_first_stage), what the reference runs as ~10^3 PyTorch library launches per UNet call:
//   ldm UNetModel.forward (openaimodel.py; structure in SURVEY Appendix A) and ldm Decoder.forward (model.py).
// Activations are 16-bit NHWC ([n, h*w, c]) end to end; NCHW exists only at the caller boundary. The skip-concat is
// never materialised for GEMMs (two K segments) and is produced for free by the GroupNorm-apply pass for convs.
#include "../../include/sdxe.h"
#include "attention.cuh"
#include "gemm.cuh"
#include "kernels.cuh"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

using namespace sdxe;

namespace {

#define EFAIL(msg)                                  \
  do {                                              \
    set_last_error(__FILE__, __LINE__, (msg));      \
    return -1;                                      \
  } while (0)
#define ECHK(expr)            \
  do {                        \
    if ((expr) != 0) return -1; \
  } while (0)

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct RawWeight {
  void* dev = nullptr;
  int dtype = 0;
  std::vector<int64_t> shape;
  int64_t numel = 0;
};

// ---- packed weights ---------------------------------------------------------------------------------------------
struct LinW {  // 16-bit [N, ld] K-contiguous (+ fp32 bias)
  void* w = nullptr;
  float* b = nullptr;
  int N = 0, K = 0, ld = 0;
  int Nrows = 0;  // rows allocated (N rounded up to 16, zero filled) so a TMA box never exceeds the tensor
  int geglu_tile = 0;
  float* c1 = nullptr;  // LayerNorm folded in (gemm.cuh): row sums of the gamma-scaled weight; b then includes beta W^T
};
struct NormW {
  float* g = nullptr;
  float* b = nullptr;
  int C = 0;
};
struct ResW {
  NormW n1, n2;
  LinW c1, c2, skip;
  bool has_skip = false;
  int cin = 0, cout = 0;
  int emb_off = -1;  // UNet: column offset into the batched emb_layers output
};
// state-dict names of a ResBlock's layers, relative to the block
struct ResKeys {
  const char *n1, *c1, *n2, *c2, *skip;
};
const ResKeys UNET_RES = {".in_layers.0", ".in_layers.2", ".out_layers.0", ".out_layers.3", ".skip_connection"};
const ResKeys VAE_RES = {".norm1", ".conv1", ".norm2", ".conv2", ".nin_shortcut"};
struct TBlockW {
  NormW ln1, ln2, ln3;
  LinW qkv1, out1, q2, out2, ff1, ff2;
  int kv_off = -1;  // column offset of this block's cross-attention [k | v] in the batched context projection
};
struct STW {
  NormW gn;
  LinW proj_in, proj_out;
  std::vector<TBlockW> blocks;
  int C = 0, heads = 0, dh = 0;
};

// ---- UNet (ldm / sgm UNetModel) ---------------------------------------------------------------------------------
struct UNetBlockW {  // one TimestepEmbedSequential: ResBlock (+ SpatialTransformer) (+ Upsample, output blocks only)
  ResW res;
  bool has_st = false;
  STW st;
  bool has_up = false;
  LinW up;  // Upsample.conv
};
struct UNetLevelW {  // the input blocks of one level: its ResBlocks, then a Downsample except at the deepest level
  std::vector<UNetBlockW> blocks;
  bool has_down = false;
  LinW down;  // Downsample.op
};
struct UNetW {
  LinW te0, te2, le0, le2, emb_all;
  int emb_total = 0;
  // every transformer block's attn2.to_k / to_v stacked along N: the context is projected ONCE per UNet call
  LinW kv_all;
  int kv_total = 0;
  int n_attn1 = 0;  // self-attention layers (one Hypertile row each)
  LinW conv_in;
  std::vector<UNetLevelW> in_levels;
  ResW mid_r1, mid_r2;
  STW mid_st;
  std::vector<UNetBlockW> out_blocks;
  NormW out_norm;
  LinW out_conv;
  // Cross-attention K / V cache: a non-zero key is the caller's promise that the context passed under that key always has
  // the same contents (the conditioning of one job is step-invariant); a plan whose k|v buffer was last filled under the
  // same key skips the context cast + projection GEMM (modules/sd_samplers_cfg_denoiser.py re-sends the same cond_in
  // every sampler step).
  int64_t ctx_key = 0;
  // Hypertile rows (h', w', nh, nw, max_tiles) per attn1 layer for the next sdxe_unet_forward (sdxe_unet_set_hypertile)
  std::vector<int32_t> ht_rows;
};

// ---- VAE (ldm Encoder / Decoder of AutoencoderKL) ---------------------------------------------------------------
struct VaeMidW {  // mid: ResBlock -> AttnBlock (GN -> q|k|v -> single-head attention -> proj_out + x) -> ResBlock
  ResW r1, r2;
  NormW attn_norm;
  LinW qkv, proj;
};
struct VaeLevelW {  // down.{l} / up.{l}: ResBlocks, then the level's Downsample / Upsample conv if it has one
  std::vector<ResW> blocks;
  bool has_resample = false;
  LinW resample;
};
struct VaeW {
  LinW conv_in;
  std::vector<VaeLevelW> levels;  // level index as in the state dict
  VaeMidW mid;
  NormW norm_out;
  LinW conv_out;
  float* pq_w = nullptr;  // decoder: post_quant_conv [z, z] fp32, run on the caller's latent before conv_in
  float* pq_b = nullptr;
  LinW quant;             // encoder: quant_conv (1x1) after conv_out
};

// ---- CLIP text transformer (Hugging Face CLIPTextModel) ---------------------------------------------------------
struct ClipLayerW {  // CLIPEncoderLayer: LN1 -> q|k|v -> causal attention -> out_proj (+x) -> LN2 -> fc1 -> act -> fc2 (+x)
  LinW qkv, out, fc1, fc2;   // layer_norm1 / layer_norm2 are folded into qkv / fc1
};
struct ClipW {
  void* tok = nullptr;  // [vocab, C] 16-bit
  void* pos = nullptr;  // [positions, C] 16-bit
  std::vector<ClipLayerW> layers;
  NormW final_norm;
};

struct Buf {
  void* p = nullptr;
  size_t bytes = 0;
};
struct Act {  // NHWC 16-bit activation, row pitch == c
  void* p = nullptr;
  int n = 0, h = 0, w = 0, c = 0;
  Buf buf;
  int64_t rows() const { return (int64_t)n * h * w; }
};

struct Plan;
using KvKeys = std::vector<std::pair<std::string, int>>;  // (state-dict key, rows) of the batched cross-attention k|v

}  // namespace

struct sdxe_engine {
  sdxe_config cfg;
  bool bf16 = false;
  int dt = 0;
  std::unordered_map<std::string, RawWeight> raw;
  int64_t params = 0;
  bool finalized = false;
  std::string missing;

  // packed blob
  char* blob = nullptr;
  size_t blob_bytes = 0;
  size_t cursor = 0;
  bool sizing = true;

  // the model's packed weights: exactly the one of cfg.kind is set (sdxe_create)
  std::unique_ptr<UNetW> unet;
  std::unique_ptr<VaeW> vae;  // decoder or encoder
  std::unique_ptr<ClipW> clip;

  // activation pool
  std::multimap<size_t, void*> free_list;
  std::vector<void*> all_allocs;
  // Plan cache: one static plan (buffers + tensor maps + CUDA graph) per input shape, least-recently-used eviction.
  // A long-lived webui process sees many shapes (resolutions, batch sizes, 77 / 154 / 231-token prompts, B vs 2B
  // batches under s_min_uncond); every plan pins its own buffers (SDXL: > 100 MB of cross-attention k|v alone), so an
  // unbounded cache grows until cudaMalloc fails.
  std::map<std::string, std::unique_ptr<Plan>> plans;
  // Circular padding in every 3x3 convolution with padding 1 (sdxe_set_circular): sticky, part of the plan key
  bool circular = false;
  int max_plans = 8;                    // sdxe_set_plan_cache
  size_t pool_limit = (size_t)6 << 30;  // free (unowned) pool bytes kept after an eviction (sdxe_set_plan_cache)
  uint64_t tick = 0;
  std::vector<Buf>* track = nullptr;    // while a plan is being built: the buffers it currently holds
  std::vector<void*>* touched = nullptr;  // ... and every pool block it used at any point (scratch it released again)
  bool alloc_failed = false;
  cudaStream_t cap_stream = nullptr;
  bool profiling = false;
  double prof_ms[8] = {0}, prof_flops[8] = {0}, prof_bytes[8] = {0};
  int64_t prof_launches[8] = {0};

  ~sdxe_engine();
  // --- weights
  const RawWeight* find(const std::string& key, int64_t numel);
  void* alloc16(size_t elems);
  float* alloc32(size_t elems);
  int pack_linear(LinW& out, const std::vector<std::string>& wkeys, const std::vector<std::string>& bkeys, int n_each, int K,
                  int mode, int kpad = 0, int geglu_tile = 0);
  int pack_dense(LinW& out, const std::string& prefix, int N, int K);     // <prefix>.weight [N, K] / .bias
  int pack_conv3(LinW& out, const std::string& prefix, int N, int cin);  // <prefix>.weight [N, cin, 3, 3] / .bias
  int pack_norm(NormW& out, const std::string& prefix, int C);
  int fold_layer_norm(LinW& w, const NormW& ln);  // w consumes LayerNorm(ln) output: fold gamma / beta into w
  int pack_f32(float*& out, const std::string& key, int64_t n);
  int build_unet(UNetW& u);
  int build_vae_decoder(VaeW& v);
  int build_vae_encoder(VaeW& v);
  int build_clip(ClipW& c);
  int build_res(ResW& r, const std::string& p, int cin, int cout, const ResKeys& k);
  int build_st(UNetW& u, STW& s, const std::string& p, int C, int depth, KvKeys& kv);
  int build_vae_mid(VaeMidW& m, const std::string& p, int C);
  // --- activations
  Buf alloc(size_t bytes);
  void release(Buf& b);
};

namespace {

using OpFn = std::function<int(cudaStream_t)>;
enum : int { K_GEMM = 0, K_CONV = 1, K_ATTN = 2, K_GNORM = 3, K_LNORM = 4, K_OTHER = 5, K_NUM = 6 };
struct OpRec {
  OpFn fn;
  int kind = K_OTHER;
  double flops = 0, bytes = 0;  // algorithmic work of this launch
  std::string desc;
  OpRec() {}
  template <class F>
  OpRec(F f) : fn(std::move(f)) {}  // implicit: un-annotated ops are K_OTHER
  template <class F>
  OpRec(F f, int k, double fl, double by, std::string d = std::string()) : fn(std::move(f)), kind(k), flops(fl), bytes(by), desc(std::move(d)) {}
};

struct Plan {
  sdxe_engine* e = nullptr;
  std::vector<OpRec> pre, body, post;
  cudaGraphExec_t gexec = nullptr;
  cudaGraph_t graph = nullptr;
  std::vector<Buf> owned;   // buffers still held when the build finished: returned to the pool on eviction
  std::vector<void*> used;  // every pool block the plan's kernels touch (owned + scratch shared through the free list)
  uint64_t last_use = 0;
  int64_t kv_key = 0;       // context key the plan's cross-attention k|v buffer was computed under (0 = none)
  // per-call caller pointers, read by pre / post ops
  const void *x = nullptr, *t = nullptr, *ctx = nullptr, *y = nullptr;
  const int32_t* fix_rows = nullptr;  // CLIP: textual-inversion fixes of this call (device pointers), n_fix = 0: none
  const void* fix_vecs = nullptr;
  int n_fix = 0;
  void* out = nullptr;
  int io_dtype = 0;
  HtDraws ht_draws{};  // UNet with Hypertile: this call's tile draws, copied into the plan's device table by a pre op
  int launches_body = 0;
  ~Plan() {
    if (gexec) cudaGraphExecDestroy(gexec);
    if (graph) cudaGraphDestroy(graph);
  }
};

// Symbolic executor: every method allocates outputs from the engine pool, prepares kernel arguments (tensor maps)
// once, and appends a launch closure to the plan.
struct Builder {
  sdxe_engine* e;
  Plan* plan;
  bool bf16;
  std::vector<OpRec>* ops;
  // Hypertile: rows (h', w', nh, nw, max_tiles) of every attn1 layer in execution order (null: off), the plan's device
  // table of per-call draws, and the index of the next attn1 layer spatial_transformer emits
  const std::vector<int32_t>* ht = nullptr;
  const int* ht_table = nullptr;
  int ht_next = 0;
  // the plan's 3x3 convolutions with padding wrap around (torch padding_mode='circular') instead of reading zeros
  bool circular;
  // UNet: the batched timestep-embedding rows every ResBlock adds after its first conv (null: none)
  const float* emb = nullptr;
  int ld_emb = 0;

  Builder(sdxe_engine* e_, Plan* p) : e(e_), plan(p), bf16(e_->bf16), ops(&p->body), circular(e_->circular) {}

  Act new_act(int n, int h, int w, int c) {
    Act a;
    a.n = n; a.h = h; a.w = w; a.c = c;
    a.buf = e->alloc((size_t)n * h * w * c * 2);
    a.p = a.buf.p;
    return a;
  }
  void free_act(Act& a) {
    if (a.buf.p) e->release(a.buf);
    a.p = nullptr;
  }

  struct RowStats {  // per-row partial (sum, sum of squares) of an activation, [parts][M] float2
    Buf buf;
    const float2* p = nullptr;
    int parts = 0;
  };
  void free_stats(RowStats& st) {
    if (st.buf.p) e->release(st.buf);
    st.p = nullptr; st.parts = 0;
  }
  // out[M, N] = A (+A2) * W^T with the fused epilogues of gemm.cu
  struct GemmOpt : GemmEpi {
    const void* A2 = nullptr;
    int K1 = 0;            // columns taken from A (A2 supplies K - K1)
    // emit per-row partial statistics of the output for a following folded LayerNorm: filled in by gemm()
    RowStats* emit = nullptr;
  };
  static GemmW weight(const LinW& W) {
    GemmW w;
    w.w = W.w; w.rows = std::max(W.N, W.Nrows); w.ld = W.ld; w.N = W.N; w.K = W.K; w.bias = W.b; w.c1 = W.c1;
    return w;
  }
  int gemm(const void* A, int lda, int64_t M, const LinW& W, void* out, const GemmOpt& o) {
    GemmEpi epi = o;
    if (o.emit)
      epi.stat_out = [this, M, st = o.emit](int parts) {
        st->buf = e->alloc((size_t)parts * M * sizeof(float2));
        st->p = (const float2*)st->buf.p;
        st->parts = parts;
        return (float2*)st->buf.p;
      };
    GemmArgs a;
    ECHK(gemm_args(a, GemmA::matrix(A, M, lda, o.A2, o.K1), weight(W), out, epi, o.epi == EPI_GEGLU ? W.geglu_tile : 0));
    const bool b = bf16;
    const double nout = (o.epi == EPI_GEGLU) ? W.N / 2.0 : (double)W.N;
    const double by = 2.0 * ((double)M * W.K + (double)W.N * W.K + (double)M * nout + (o.residual ? (double)M * nout : 0.0));
    char d[160];
    snprintf(d, sizeof(d), "gemm M=%lld N=%d K=%d BN=%d st=%d epi=%d res=%d rv=%d dual=%d", (long long)M, W.N, W.K, a.BN, a.num_stages, o.epi,
             o.residual ? 1 : 0, o.rowvec ? 1 : 0, o.A2 ? 1 : 0);
    ops->push_back(OpRec([a, b](cudaStream_t s) { return gemm_launch(a, b, s); }, K_GEMM, 2.0 * (double)M * W.N * W.K, by, d));
    return 0;
  }

  // 3x3 conv of an NHWC activation, W packed [Cout, 9*Cin (ld)]: stride 1 pad 1, or stride 2 (ldm Downsample) with pad_lo
  // zero rows / columns before the image and output Ho x Wo. Implicit GEMM when the geometry allows it, else im2col.
  // With `circular`, a conv with pad_lo = 1 wraps around instead: im2col indexes modulo H and W, the implicit GEMM reads a
  // copy of x with its one-pixel circular halo written out (circular_pad_nhwc) with every tap in bounds. pad_lo = 0 (the
  // VAE encoder's Downsample, Conv2d(padding=0) after a constant pad) keeps its zeros, as padding_mode does not touch it.
  int conv3(const Act& x, const LinW& W, void* out, int ldo, const GemmOpt& o, int stride = 1, int pad_lo = 1, int Ho = 0,
            int Wo = 0) {
    static int s2_implicit = -1;
    if (s2_implicit < 0) { const char* ev = getenv("SDXE_CONV_S2_IMPLICIT"); s2_implicit = ev ? atoi(ev) : 1; }
    if (stride == 1) { Ho = x.h; Wo = x.w; }
    const bool circ = circular && pad_lo > 0;
    int bw, bh, bn;
    const bool implicit = x.c % 64 == 0 && W.ld == 9 * x.c && conv_tile_shape(Ho, Wo, &bw, &bh, &bn) &&
                          (stride == 1 || (s2_implicit && x.h % 2 == 0 && x.w % 2 == 0 && Ho == x.h / 2 && Wo == x.w / 2));
    if (!implicit) {  // generic geometry: explicit im2col (still CUDA; used for odd resolutions / narrow channel counts)
      const int kpad = W.ld;
      const int64_t M = (int64_t)x.n * Ho * Wo;
      Buf col = e->alloc((size_t)M * kpad * 2);
      const void* xp = x.p;
      void* cp = col.p;
      const int n = x.n, H = x.h, Wd = x.w, C = x.c;
      const bool b = bf16;
      auto fn = [=](cudaStream_t s) { return im2col3x3_launch(xp, cp, n, H, Wd, C, Ho, Wo, stride, pad_lo, kpad, circ, b, s); };
      if (circ) {
        char d[160];
        snprintf(d, sizeof(d), "im2col M=%lld K=%d Cin=%d HxW=%dx%d s=%d circ=1", (long long)M, kpad, C, H, Wd, stride);
        ops->push_back(OpRec(fn, K_OTHER, 0.0, 2.0 * (double)M * kpad * 2, d));
      } else {
        ops->push_back(fn);
      }
      LinW W2 = W;
      W2.K = kpad;  // zero-padded columns on both sides
      GemmOpt o2 = o;
      o2.ldo = ldo;
      ECHK(gemm(col.p, kpad, M, W2, out, o2));
      e->release(col);
      return 0;
    }
    GemmEpi epi = o;
    epi.ldo = ldo;
    GemmArgs a;
    const bool b = bf16;
    if (circ) {
      Buf pad = e->alloc((size_t)x.n * (x.h + 2) * (x.w + 2) * x.c * 2);
      const void* xp = x.p;
      void* pp = pad.p;
      const int n = x.n, H = x.h, Wd = x.w, C = x.c;
      char d[160];
      snprintf(d, sizeof(d), "circpad n=%d HxW=%dx%d C=%d", n, H, Wd, C);
      ops->push_back(OpRec([=](cudaStream_t s) { return circular_pad_nhwc_launch(xp, pp, n, H, Wd, C, s); }, K_OTHER, 0.0,
                           2.0 * n * C * ((double)H * Wd + (double)(H + 2) * (Wd + 2)), d));
      ECHK(gemm_args(a, GemmA::nhwc(pad.p, n, H + 2, Wd + 2, C, stride, 0, 1), weight(W), out, epi));
      e->release(pad);  // scratch: the next op that takes it runs after this conv on the same stream
    } else {
      ECHK(gemm_args(a, GemmA::nhwc(x.p, x.n, x.h, x.w, x.c, stride, pad_lo), weight(W), out, epi));
    }
    const double Md = (double)a.M;
    char d[160];
    double by;
    if (stride == 1) {
      by = 2.0 * (Md * x.c + (double)W.N * a.K + Md * W.N + (o.residual ? Md * W.N : 0.0));
      snprintf(d, sizeof(d), "conv3 M=%d N=%d Cin=%d HxW=%dx%d BN=%d st=%d res=%d rv=%d%s", a.M, W.N, x.c, x.h, x.w, a.BN, a.num_stages,
               o.residual ? 1 : 0, o.rowvec ? 1 : 0, circ ? " circ=1" : "");
    } else {
      by = 2.0 * (4.0 * Md * x.c + (double)W.N * a.K + Md * W.N);
      snprintf(d, sizeof(d), "conv3s2 M=%d N=%d Cin=%d HoxWo=%dx%d BN=%d st=%d%s", a.M, W.N, x.c, Ho, Wo, a.BN, a.num_stages,
               circ ? " circ=1" : "");
    }
    ops->push_back(OpRec([a, b](cudaStream_t s) { return gemm_launch(a, b, s); }, K_CONV, 2.0 * Md * W.N * a.K, by, d));
    return 0;
  }

  int group_norm(const Act& x1, const Act* x2, const NormW& nw, float eps, bool silu, Act& out) {
    const int c2 = x2 ? x2->c : 0;
    out = new_act(x1.n, x1.h, x1.w, x1.c + c2);
    Buf st = e->alloc(sizeof(float) * group_norm_scratch_floats(x1.n, 32));
    const void *p1 = x1.p, *p2 = x2 ? x2->p : nullptr;
    void* po = out.p;
    float* sp = (float*)st.p;
    const int c1 = x1.c, n = x1.n, hw = x1.h * x1.w;
    const float *g = nw.g, *bt = nw.b;
    const bool b = bf16;
    if (nw.C != c1 + c2) EFAIL("group_norm: channel mismatch");
    ops->push_back(OpRec([=](cudaStream_t s) { return group_norm_launch(p1, c1, p2, c2, g, bt, po, sp, n, hw, 32, eps, silu, b, s); },
                         K_GNORM, 0.0, 4.0 * (double)n * hw * (c1 + c2), "gn n=" + std::to_string(n) + " hw=" + std::to_string(hw) + " C=" + std::to_string(c1 + c2)));
    e->release(st);
    return 0;
  }
  // q: [B*Nq, ldq], k / v: [B*Nk, ldkv] row-major activations whose columns h*d .. h*d+d-1 belong to head h (the
  // projection GEMM's natural output), seen through per-head views: no padded per-head copy exists.
  // seg: Hypertile segmented self-attention over the tile-major rows of an seg_h x seg_w grid (AttnArgs::seg); its
  // FLOP estimate assumes the largest tile count, seg_mt.
  int attention(const void* q, const void* k, const void* v, int B, int H, int Nq, int Nk, int d, int ldq, int ldkv,
                float scale, void* out, int ldo, int dv_total, const int* seg = nullptr, int seg_h = 0, int seg_w = 0,
                int seg_mt = 0) {
    std::vector<AttnArgs> passes;
    const AttnView vq = {q, ldq, d, (int64_t)Nq * ldq}, vk = {k, ldkv, d, (int64_t)Nk * ldkv}, vv = {v, ldkv, d, (int64_t)Nk * ldkv};
    ECHK(attention_args(passes, vq, vk, vv, B, H, Nq, Nk, d, dv_total, scale, out, ldo, dv_total));
    const int dpad = (d + 63) / 64 * 64;
    for (AttnArgs a : passes) {  // value columns in passes (VAE d = 512, SD1.5 d = 160)
      const int dv = a.dv;
      const bool b = bf16;
      const double keys = seg ? (double)Nk / seg_mt : (double)Nk;
      const double fl = 2.0 * (double)B * H * Nq * keys * ((double)d + dv);
      const double by = 2.0 * (double)B * H * ((double)Nq * d + (double)Nk * (d + dv) + (double)Nq * dv);
      char dsc[160];
      if (seg) {
        a.seg = seg; a.seg_h = seg_h; a.seg_w = seg_w; a.seg_max_tiles = seg_mt;
        snprintf(dsc, sizeof(dsc), "attn B=%d H=%d Nq=%d Nk=%d d=%d dpad=%d dv=%d ht=%dx%d/%d", B, H, Nq, Nk, d, dpad, dv, seg_h, seg_w, seg_mt);
      } else {
        snprintf(dsc, sizeof(dsc), "attn B=%d H=%d Nq=%d Nk=%d d=%d dpad=%d dv=%d", B, H, Nq, Nk, d, dpad, dv);
      }
      ops->push_back(OpRec([a, b](cudaStream_t s) { return attention_launch(a, b, s); }, K_ATTN, fl, by, dsc));
    }
    return 0;
  }

  // 3x3 conv of the model's NCHW input: im2col3x3_nchw in `pre`, then the GEMM with K = ld. src: a plan buffer of the
  // engine's dtype, or null for the caller's x (in its io dtype, read at run time).
  int conv_in_nchw(const void* src, int n, int c, int h, int w, const LinW& W, Act& out) {
    const int kin = W.ld;
    Buf col = e->alloc((size_t)n * h * w * kin * 2);  // plan-owned
    {
      Plan* p = plan;
      void* cp = col.p;
      const int edt = e->dt;
      const bool b = bf16, circ = circular;
      plan->pre.push_back([=](cudaStream_t s) {
        return im2col3x3_nchw_launch(src ? src : p->x, src ? edt : p->io_dtype, cp, n, c, h, w, kin, circ, b, s);
      });
    }
    out = new_act(n, h, w, W.N);
    LinW Wk = W;
    Wk.K = kin;
    return gemm(col.p, kin, out.rows(), Wk, out.p, GemmOpt());
  }
  // ldm Upsample: nearest 2x, then 3x3 conv; replaces x
  int upsample_conv(Act& x, const LinW& W) {
    Act up = new_act(x.n, x.h * 2, x.w * 2, x.c);
    {
      const void* xp = x.p;
      void* upp = up.p;
      const int n = x.n, h = x.h, w = x.w, c = x.c;
      ops->push_back([=](cudaStream_t s) { return upsample2x_launch(xp, upp, n, h, w, c, s); });
    }
    free_act(x);
    x = new_act(up.n, up.h, up.w, up.c);
    ECHK(conv3(up, W, x.p, up.c, GemmOpt()));
    free_act(up);
    return 0;
  }
  // output head: GroupNorm + SiLU -> 3x3 conv -> the caller's NCHW output (in `post`); x is released
  int out_head(Act& x, const NormW& norm, float eps, const LinW& W) {
    Act g;
    ECHK(group_norm(x, nullptr, norm, eps, true, g));
    free_act(x);
    const int ldo = (int)align_up(W.N, 8);
    Buf outb = e->alloc((size_t)g.rows() * ldo * 2);  // plan-owned
    ECHK(conv3(g, W, outb.p, ldo, GemmOpt()));
    free_act(g);
    Plan* p = plan;
    void* ob = outb.p;
    const int n = g.n, oc = W.N, hw = g.h * g.w;
    const bool b = bf16;
    plan->post.push_back([=](cudaStream_t s) { return nhwc_to_nchw_launch(ob, ldo, p->out, p->io_dtype, n, oc, hw, b, s); });
    return 0;
  }

  // ---- UNet building blocks --------------------------------------------------------------------------------
  // ResBlock (ldm openaimodel.ResBlock, VAE ResnetBlock): GN32+SiLU -> conv3 (+emb) -> GN32+SiLU -> conv3 (+skip).
  // skip_src: the UNet decoder's skip-concat input.
  int res_block(const ResW& r, const Act& x, Act* skip_src, float eps, Act& out) {
    Act g1;
    ECHK(group_norm(x, skip_src, r.n1, eps, true, g1));
    Act h = new_act(x.n, x.h, x.w, r.cout);
    GemmOpt o1;
    if (emb) { o1.rowvec = emb + r.emb_off; o1.ldrv = ld_emb; o1.rows_per_sample = x.h * x.w; }
    ECHK(conv3(g1, r.c1, h.p, r.cout, o1));
    free_act(g1);
    Act g2;
    ECHK(group_norm(h, nullptr, r.n2, eps, true, g2));
    free_act(h);
    Act sk;
    const void* res_ptr;
    if (r.has_skip) {
      sk = new_act(x.n, x.h, x.w, r.cout);
      GemmOpt os;
      if (skip_src) { os.A2 = skip_src->p; os.K1 = x.c; }
      ECHK(gemm(x.p, x.c, x.rows(), r.skip, sk.p, os));
      res_ptr = sk.p;
    } else {
      if (skip_src) EFAIL("identity skip with concat input");
      res_ptr = x.p;
    }
    out = new_act(x.n, x.h, x.w, r.cout);
    GemmOpt o2;
    o2.residual = res_ptr; o2.ldr = r.cout;
    ECHK(conv3(g2, r.c2, out.p, r.cout, o2));
    free_act(g2);
    if (r.has_skip) free_act(sk);
    return 0;
  }
  // a ResBlock whose input is not needed afterwards: replaces x
  int res_replace(const ResW& r, Act& x, float eps, Act* skip_src = nullptr) {
    Act out;
    ECHK(res_block(r, x, skip_src, eps, out));
    free_act(x);
    x = out;
    return 0;
  }

  // SpatialTransformer (modules/sd_hijack_unet.py:83-102) with BasicTransformerBlocks; replaces x
  // kv_all: [B * ctx_len, ld_kv] = every block's cross-attention k | v projection of the context (one GEMM per call)
  int spatial_transformer(const STW& st, Act& x, const void* kv_all, int ld_kv, int ctx_len) {
    const int C = st.C, H = st.heads, dh = st.dh;
    const int64_t M = x.rows();
    const int tokens = x.h * x.w, B = x.n;
    const float scale = 1.0f / sqrtf((float)dh);
    Act xn;
    ECHK(group_norm(x, nullptr, st.gn, 1e-6f, false, xn));
    Act h = new_act(x.n, x.h, x.w, C);
    // The three LayerNorms of a block are folded into the GEMMs that consume them: the GEMM that PRODUCES the token
    // stream h also emits each row's (sum, sum of squares), the consumer's epilogue normalises with them.
    RowStats hs;
    {
      GemmOpt oi;
      oi.emit = &hs;
      ECHK(gemm(xn.p, C, M, st.proj_in, h.p, oi));
    }
    free_act(xn);
    for (size_t bi = 0; bi < st.blocks.size(); ++bi) {
      const TBlockW& tb = st.blocks[bi];
      const bool last = bi + 1 == st.blocks.size();
      // --- self attention: q | k | v = LN1(h) W^T
      Act qkv = new_act(x.n, x.h, x.w, 3 * C);
      GemmOpt oq;
      oq.ln_part = hs.p; oq.ln_parts = hs.parts;
      ECHK(gemm(h.p, C, M, tb.qkv1, qkv.p, oq));  // columns: [q | k | v], heads contiguous inside each
      free_stats(hs);
      Act att = new_act(x.n, x.h, x.w, C);
      const int li = ht_next++;
      if (ht && (*ht)[5 * li + 4] > 0) {
        // Hypertile: q|k|v rows regrouped tile-major, attention inside each tile, outputs stored at their natural rows
        const int hp = (*ht)[5 * li], wp = (*ht)[5 * li + 1], mt = (*ht)[5 * li + 4];
        if ((int64_t)hp * wp != tokens) EFAIL("sdxe_unet_set_hypertile: h' * w' differs from the layer's token count");
        Act qkvt = new_act(x.n, x.h, x.w, 3 * C);
        {
          const void* src = qkv.p;
          void* dst = qkvt.p;
          const int* seg = ht_table + 2 * li;
          char d[96];
          snprintf(d, sizeof(d), "ht_gather M=%lld C=%d grid=%dx%d", (long long)M, 3 * C, hp, wp);
          ops->push_back(OpRec([=](cudaStream_t s) { return hypertile_gather_launch(src, dst, B, hp, wp, 3 * C, seg, s); }, K_OTHER,
                               0.0, 4.0 * (double)M * 3 * C, d));
        }
        free_act(qkv);
        const uint16_t* t16 = (const uint16_t*)qkvt.p;
        ECHK(attention(t16, t16 + C, t16 + 2 * C, B, H, tokens, tokens, dh, 3 * C, 3 * C, scale, att.p, C, dh, ht_table + 2 * li, hp,
                       wp, mt));
        free_act(qkvt);
      } else {
        const uint16_t* qkv16 = (const uint16_t*)qkv.p;
        ECHK(attention(qkv16, qkv16 + C, qkv16 + 2 * C, B, H, tokens, tokens, dh, 3 * C, 3 * C, scale, att.p, C, dh));
        free_act(qkv);
      }
      Act h2 = new_act(x.n, x.h, x.w, C);
      GemmOpt oo;
      oo.residual = h.p; oo.ldr = C; oo.emit = &hs;
      ECHK(gemm(att.p, C, M, tb.out1, h2.p, oo));
      free_act(h);
      h = h2;
      // --- cross attention: q = LN2(h) W^T
      Act q2 = new_act(x.n, x.h, x.w, C);
      GemmOpt oq2;
      oq2.ln_part = hs.p; oq2.ln_parts = hs.parts;
      ECHK(gemm(h.p, C, M, tb.q2, q2.p, oq2));
      free_stats(hs);
      const uint16_t* kv = (const uint16_t*)kv_all + tb.kv_off;  // columns: [k | v] of this block
      ECHK(attention(q2.p, kv, kv + C, B, H, tokens, ctx_len, dh, C, ld_kv, scale, att.p, C, dh));
      free_act(q2);
      Act h3 = new_act(x.n, x.h, x.w, C);
      GemmOpt oo2;
      oo2.residual = h.p; oo2.ldr = C; oo2.emit = &hs;
      ECHK(gemm(att.p, C, M, tb.out2, h3.p, oo2));
      free_act(att);
      free_act(h);
      h = h3;
      // --- feed forward: GEGLU(LN3(h)) fused into the first GEMM's epilogue
      Act ff = new_act(x.n, x.h, x.w, 4 * C);
      GemmOpt og;
      og.epi = EPI_GEGLU;
      og.ln_part = hs.p; og.ln_parts = hs.parts;
      ECHK(gemm(h.p, C, M, tb.ff1, ff.p, og));
      free_stats(hs);
      Act h4 = new_act(x.n, x.h, x.w, C);
      GemmOpt of;
      of.residual = h.p; of.ldr = C;
      if (!last) of.emit = &hs;  // the next block's LN1
      ECHK(gemm(ff.p, 4 * C, M, tb.ff2, h4.p, of));
      free_act(ff);
      free_act(h);
      h = h4;
    }
    Act out = new_act(x.n, x.h, x.w, C);
    GemmOpt op;
    op.residual = x.p; op.ldr = C;
    ECHK(gemm(h.p, C, M, st.proj_out, out.p, op));
    free_act(h);
    free_act(x);
    x = out;
    return 0;
  }

  // ---- VAE building blocks ---------------------------------------------------------------------------------
  // mid block: ResBlock -> AttnBlock (sd_hijack_optimizations.py:637-655) -> ResBlock; replaces cur
  int vae_mid(const VaeMidW& m, Act& cur) {
    ECHK(res_replace(m.r1, cur, 1e-6f));
    const int C = cur.c, tokens = cur.h * cur.w, n = cur.n;
    const int64_t M = cur.rows();
    Act xn;
    ECHK(group_norm(cur, nullptr, m.attn_norm, 1e-6f, false, xn));
    Buf qkv = e->alloc((size_t)M * 3 * C * 2);
    ECHK(gemm(xn.p, C, M, m.qkv, qkv.p, GemmOpt()));
    free_act(xn);
    if (C % 64 != 0 || C > 512) EFAIL("vae attention: channel count must be a multiple of 64 and <= 512");
    Act att = new_act(n, cur.h, cur.w, C);
    const uint16_t* qp = (const uint16_t*)qkv.p;
    ECHK(attention(qp, qp + C, qp + 2 * C, n, 1, tokens, tokens, C, 3 * C, 3 * C, 1.0f / sqrtf((float)C), att.p, C, C));
    e->release(qkv);
    Act o = new_act(n, cur.h, cur.w, C);
    GemmOpt op;
    op.residual = cur.p; op.ldr = C;
    ECHK(gemm(att.p, C, M, m.proj, o.p, op));
    free_act(att);
    free_act(cur);
    cur = o;
    return res_replace(m.r2, cur, 1e-6f);
  }
};

}  // namespace

// =================================================================================================================
// engine: weights
// =================================================================================================================
sdxe_engine::~sdxe_engine() {
  plans.clear();
  for (auto& kv : raw) if (kv.second.dev) cudaFree(kv.second.dev);
  for (void* p : all_allocs) cudaFree(p);
  if (blob) cudaFree(blob);
  if (cap_stream) cudaStreamDestroy(cap_stream);
}

const RawWeight* sdxe_engine::find(const std::string& key, int64_t numel) {
  auto it = raw.find(key);
  if (it == raw.end()) {
    if (missing.size() < 600) missing += (missing.empty() ? "" : ", ") + key;
    return nullptr;
  }
  if (it->second.numel != numel) {
    if (missing.size() < 600) missing += (missing.empty() ? "" : ", ") + key + "(shape)";
    return nullptr;
  }
  return &it->second;
}
void* sdxe_engine::alloc16(size_t elems) {
  cursor = align_up(cursor, 256);
  void* p = sizing ? nullptr : blob + cursor;
  cursor += elems * 2;
  return p;
}
float* sdxe_engine::alloc32(size_t elems) {
  cursor = align_up(cursor, 256);
  float* p = sizing ? nullptr : reinterpret_cast<float*>(blob + cursor);
  cursor += elems * 4;
  return p;
}

// mode: PACK_PLAIN ([n_each, K] per key, keys stacked along N), PACK_CONV3 (single key [N, K/9, 3, 3]), PACK_GEGLU
int sdxe_engine::pack_linear(LinW& out, const std::vector<std::string>& wkeys, const std::vector<std::string>& bkeys,
                             int n_each, int K, int mode, int kpad, int geglu_tile) {
  const int N = n_each * (int)wkeys.size();
  const int ld = kpad ? kpad : K;
  out.N = N; out.K = K; out.ld = ld; out.geglu_tile = geglu_tile;
  out.Nrows = (int)align_up((size_t)N, 16);
  out.w = alloc16((size_t)out.Nrows * ld);
  out.b = bkeys.empty() ? nullptr : alloc32(align_up((size_t)N, 8));
  for (size_t i = 0; i < wkeys.size(); ++i) {
    const RawWeight* w = find(wkeys[i], (int64_t)n_each * K);
    if (!sizing && w) {
      if (ld != K) SDXE_CUDA_CHECK(cudaMemsetAsync((char*)out.w + (size_t)i * n_each * ld * 2, 0, (size_t)n_each * ld * 2, 0));
      ECHK(pack_weight_launch(w->dev, w->dtype, (char*)out.w + (size_t)i * n_each * ld * 2, mode, n_each, K, ld, geglu_tile, bf16, 0));
    }
  }
  for (size_t i = 0; i < bkeys.size(); ++i) {
    const RawWeight* b = find(bkeys[i], n_each);
    if (!sizing && b) {
      if (i == 0) SDXE_CUDA_CHECK(cudaMemsetAsync(out.b, 0, align_up((size_t)N, 8) * 4, 0));
      ECHK(pack_vector_launch(b->dev, b->dtype, out.b + i * n_each, n_each, mode == PACK_GEGLU ? geglu_tile : 0, true, bf16, 0));
    }
  }
  return 0;
}
int sdxe_engine::pack_norm(NormW& out, const std::string& prefix, int C) {
  out.C = C;
  out.g = alloc32(C);
  out.b = alloc32(C);
  const RawWeight* g = find(prefix + ".weight", C);
  const RawWeight* b = find(prefix + ".bias", C);
  if (!sizing && g && b) {
    ECHK(pack_vector_launch(g->dev, g->dtype, out.g, C, 0, true, bf16, 0));
    ECHK(pack_vector_launch(b->dev, b->dtype, out.b, C, 0, true, bf16, 0));
  }
  return 0;
}
int sdxe_engine::fold_layer_norm(LinW& w, const NormW& ln) {
  if (ln.C != w.K) EFAIL("fold_layer_norm: width mismatch");
  const size_t nb = align_up((size_t)w.N, 8);
  const bool had_bias = w.b != nullptr;
  if (!had_bias) w.b = alloc32(nb);
  w.c1 = alloc32(nb);
  if (!sizing) {
    if (!had_bias) SDXE_CUDA_CHECK(cudaMemsetAsync(w.b, 0, nb * 4, 0));
    SDXE_CUDA_CHECK(cudaMemsetAsync(w.c1, 0, nb * 4, 0));
    ECHK(ln_fold_launch(w.w, w.N, w.K, w.ld, ln.g, ln.b, w.b, w.c1, bf16, 0));
  }
  return 0;
}
int sdxe_engine::pack_f32(float*& out, const std::string& key, int64_t n) {
  out = alloc32(n);
  const RawWeight* w = find(key, n);
  if (!sizing && w) ECHK(pack_vector_launch(w->dev, w->dtype, out, (int)n, 0, true, bf16, 0));
  return 0;
}

static int conv_kpad(int cin) {
  // 3x3 conv weights are stored [Cout, 9*Cin]; narrow inputs (latents) are padded to one 64-wide K block
  const int k = 9 * cin;
  return (cin % 64 == 0) ? k : (int)align_up(k, 64);
}
int sdxe_engine::pack_dense(LinW& out, const std::string& prefix, int N, int K) {
  return pack_linear(out, {prefix + ".weight"}, {prefix + ".bias"}, N, K, PACK_PLAIN);
}
int sdxe_engine::pack_conv3(LinW& out, const std::string& prefix, int N, int cin) {
  return pack_linear(out, {prefix + ".weight"}, {prefix + ".bias"}, N, 9 * cin, PACK_CONV3, conv_kpad(cin));
}

int sdxe_engine::build_res(ResW& r, const std::string& p, int cin, int cout, const ResKeys& k) {
  r.cin = cin; r.cout = cout;
  ECHK(pack_norm(r.n1, p + k.n1, cin));
  ECHK(pack_conv3(r.c1, p + k.c1, cout, cin));
  ECHK(pack_norm(r.n2, p + k.n2, cout));
  ECHK(pack_conv3(r.c2, p + k.c2, cout, cout));
  r.has_skip = cin != cout;
  if (r.has_skip) ECHK(pack_dense(r.skip, p + k.skip, cout, cin));
  return 0;
}

// =================================================================================================================
// UNet weights
// =================================================================================================================
// kv: the blocks' cross-attention k / v keys, packed as one matrix after every block is known (build_unet)
int sdxe_engine::build_st(UNetW& u, STW& s, const std::string& p, int C, int depth, KvKeys& kv) {
  s.C = C;
  if (cfg.num_head_channels > 0) { s.dh = cfg.num_head_channels; s.heads = C / s.dh; }
  else { s.heads = cfg.num_heads; s.dh = C / s.heads; }
  if (s.dh % 8) EFAIL("head dim must be a multiple of 8");
  ECHK(pack_norm(s.gn, p + ".norm", C));
  ECHK(pack_dense(s.proj_in, p + ".proj_in", C, C));
  ECHK(pack_dense(s.proj_out, p + ".proj_out", C, C));
  s.blocks.resize(depth);
  u.n_attn1 += depth;
  for (int j = 0; j < depth; ++j) {
    TBlockW& t = s.blocks[j];
    const std::string b = p + ".transformer_blocks." + std::to_string(j);
    ECHK(pack_norm(t.ln1, b + ".norm1", C));
    ECHK(pack_norm(t.ln2, b + ".norm2", C));
    ECHK(pack_norm(t.ln3, b + ".norm3", C));
    ECHK(pack_linear(t.qkv1, {b + ".attn1.to_q.weight", b + ".attn1.to_k.weight", b + ".attn1.to_v.weight"}, {}, C, C, PACK_PLAIN));
    ECHK(pack_dense(t.out1, b + ".attn1.to_out.0", C, C));
    ECHK(pack_linear(t.q2, {b + ".attn2.to_q.weight"}, {}, C, C, PACK_PLAIN));
    t.kv_off = u.kv_total;
    kv.push_back({b + ".attn2.to_k.weight", C});
    kv.push_back({b + ".attn2.to_v.weight", C});
    u.kv_total += 2 * C;
    ECHK(pack_dense(t.out2, b + ".attn2.to_out.0", C, C));
    const int n1 = 8 * C;
    const int tile = n1 % 256 == 0 ? 256 : (n1 % 128 == 0 ? 128 : 64);
    ECHK(pack_linear(t.ff1, {b + ".ff.net.0.proj.weight"}, {b + ".ff.net.0.proj.bias"}, n1, C, PACK_GEGLU, 0, tile));
    ECHK(pack_dense(t.ff2, b + ".ff.net.2", C, 4 * C));
    // norm1 / norm2 / norm3 are folded into the GEMMs that consume them (no LayerNorm kernel runs)
    ECHK(fold_layer_norm(t.qkv1, t.ln1));
    ECHK(fold_layer_norm(t.q2, t.ln2));
    ECHK(fold_layer_norm(t.ff1, t.ln3));
  }
  return 0;
}

int sdxe_engine::build_unet(UNetW& u) {
  const int mc = cfg.model_channels, ted = 4 * mc, nl = cfg.num_levels, nrb = cfg.num_res_blocks;
  ECHK(pack_dense(u.te0, "time_embed.0", ted, mc));
  ECHK(pack_dense(u.te2, "time_embed.2", ted, ted));
  if (cfg.adm_in_channels > 0) {
    ECHK(pack_dense(u.le0, "label_emb.0.0", ted, cfg.adm_in_channels));
    ECHK(pack_dense(u.le2, "label_emb.0.2", ted, ted));
  }
  u.in_levels.assign(nl, {});
  u.out_blocks.clear();
  u.kv_total = u.n_attn1 = 0;
  KvKeys kv;
  std::vector<std::string> emb_w, emb_b;  // batched emb_layers (every ResBlock's Linear(SiLU(emb)) in one skinny GEMM)
  std::vector<int> emb_n;
  int emb_cursor = 0;
  auto add_res = [&](ResW& r, const std::string& p, int cin, int cout) {
    ECHK(build_res(r, p, cin, cout, UNET_RES));
    r.emb_off = emb_cursor;
    emb_cursor += r.cout;
    emb_w.push_back(p + ".emb_layers.1.weight");
    emb_b.push_back(p + ".emb_layers.1.bias");
    emb_n.push_back(r.cout);
    return 0;
  };
  ECHK(pack_conv3(u.conv_in, "input_blocks.0.0", mc, cfg.in_channels));
  std::vector<int> chans = {mc};
  int ch = mc, idx = 1;
  for (int level = 0; level < nl; ++level) {
    const int mult = cfg.channel_mult[level];
    UNetLevelW& lv = u.in_levels[level];
    lv.blocks.resize(nrb);
    for (UNetBlockW& b : lv.blocks) {
      const std::string p = "input_blocks." + std::to_string(idx++);
      ECHK(add_res(b.res, p + ".0", ch, mult * mc));
      ch = mult * mc;
      b.has_st = cfg.transformer_depth[level] > 0;
      if (b.has_st) ECHK(build_st(u, b.st, p + ".1", ch, cfg.transformer_depth[level], kv));
      chans.push_back(ch);
    }
    lv.has_down = level != nl - 1;
    if (lv.has_down) {
      ECHK(pack_conv3(lv.down, "input_blocks." + std::to_string(idx++) + ".0.op", ch, ch));
      chans.push_back(ch);
    }
  }
  ECHK(add_res(u.mid_r1, "middle_block.0", ch, ch));
  ECHK(build_st(u, u.mid_st, "middle_block.1", ch, std::max(1, cfg.transformer_depth_middle), kv));
  ECHK(add_res(u.mid_r2, "middle_block.2", ch, ch));
  idx = 0;
  for (int level = nl - 1; level >= 0; --level) {
    const int mult = cfg.channel_mult[level];
    for (int i = 0; i <= nrb; ++i) {
      const int ich = chans.back();
      chans.pop_back();
      UNetBlockW b;
      const std::string p = "output_blocks." + std::to_string(idx++);
      ECHK(add_res(b.res, p + ".0", ch + ich, mc * mult));
      ch = mc * mult;
      b.has_st = cfg.transformer_depth[level] > 0;
      if (b.has_st) ECHK(build_st(u, b.st, p + ".1", ch, cfg.transformer_depth[level], kv));
      b.has_up = level && i == nrb;
      if (b.has_up) ECHK(pack_conv3(b.up, p + "." + std::to_string(b.has_st ? 2 : 1) + ".conv", ch, ch));
      u.out_blocks.push_back(b);
    }
  }
  ECHK(pack_norm(u.out_norm, "out.0", ch));
  ECHK(pack_conv3(u.out_conv, "out.2", cfg.out_channels, ch));
  // batched emb_layers: rows of different widths -> pack key by key
  u.emb_total = emb_cursor;
  LinW& ea = u.emb_all;
  ea.N = u.emb_total; ea.K = ted; ea.ld = ted;
  ea.w = alloc16((size_t)u.emb_total * ted);
  ea.b = alloc32(align_up((size_t)u.emb_total, 8));
  int off = 0;
  for (size_t i = 0; i < emb_w.size(); ++i) {
    const RawWeight* w = find(emb_w[i], (int64_t)emb_n[i] * ted);
    const RawWeight* b = find(emb_b[i], emb_n[i]);
    if (!sizing && w && b) {
      ECHK(pack_weight_launch(w->dev, w->dtype, (char*)ea.w + (size_t)off * ted * 2, PACK_PLAIN, emb_n[i], ted, ted, 0, bf16, 0));
      ECHK(pack_vector_launch(b->dev, b->dtype, ea.b + off, emb_n[i], 0, true, bf16, 0));
    }
    off += emb_n[i];
  }
  // batched cross-attention K/V projection weights [kv_total, context_dim]
  const int ctx = cfg.context_dim;
  LinW& kva = u.kv_all;
  kva.N = u.kv_total; kva.K = ctx; kva.ld = ctx; kva.b = nullptr;
  kva.Nrows = (int)align_up((size_t)u.kv_total, 16);
  kva.w = alloc16((size_t)kva.Nrows * ctx);
  int row = 0;
  for (const auto& k : kv) {
    const RawWeight* w = find(k.first, (int64_t)k.second * ctx);
    if (!sizing && w)
      ECHK(pack_weight_launch(w->dev, w->dtype, (char*)kva.w + (size_t)row * ctx * 2, PACK_PLAIN, k.second, ctx, ctx, 0, bf16, 0));
    row += k.second;
  }
  return 0;
}

// =================================================================================================================
// VAE weights
// =================================================================================================================
int sdxe_engine::build_vae_mid(VaeMidW& m, const std::string& p, int C) {
  const std::string a = p + ".attn_1.";
  ECHK(build_res(m.r1, p + ".block_1", C, C, VAE_RES));
  ECHK(pack_norm(m.attn_norm, a + "norm", C));
  ECHK(pack_linear(m.qkv, {a + "q.weight", a + "k.weight", a + "v.weight"}, {a + "q.bias", a + "k.bias", a + "v.bias"}, C, C, PACK_PLAIN));
  ECHK(pack_dense(m.proj, a + "proj_out", C, C));
  return build_res(m.r2, p + ".block_2", C, C, VAE_RES);
}

int sdxe_engine::build_vae_decoder(VaeW& v) {
  const int z = cfg.vae_z_channels, nl = cfg.num_levels, nrb = cfg.num_res_blocks;
  ECHK(pack_f32(v.pq_w, "post_quant_conv.weight", (int64_t)z * z));
  ECHK(pack_f32(v.pq_b, "post_quant_conv.bias", z));
  int bi = cfg.vae_ch * cfg.channel_mult[nl - 1];
  ECHK(pack_conv3(v.conv_in, "decoder.conv_in", bi, z));
  ECHK(build_vae_mid(v.mid, "decoder.mid", bi));
  v.levels.assign(nl, {});
  for (int level = nl - 1; level >= 0; --level) {
    VaeLevelW& lv = v.levels[level];
    const std::string p = "decoder.up." + std::to_string(level);
    const int bo = cfg.vae_ch * cfg.channel_mult[level];
    lv.blocks.resize(nrb + 1);
    for (int j = 0; j <= nrb; ++j, bi = bo) ECHK(build_res(lv.blocks[j], p + ".block." + std::to_string(j), bi, bo, VAE_RES));
    lv.has_resample = level != 0;
    if (lv.has_resample) ECHK(pack_conv3(lv.resample, p + ".upsample.conv", bi, bi));
  }
  ECHK(pack_norm(v.norm_out, "decoder.norm_out", bi));
  return pack_conv3(v.conv_out, "decoder.conv_out", cfg.vae_out_ch, bi);
}

int sdxe_engine::build_vae_encoder(VaeW& v) {
  const int z = cfg.vae_z_channels, nl = cfg.num_levels, nrb = cfg.num_res_blocks, ch = cfg.vae_ch;
  ECHK(pack_conv3(v.conv_in, "encoder.conv_in", ch, cfg.vae_out_ch));
  v.levels.assign(nl, {});
  int bi = ch;
  for (int level = 0; level < nl; ++level) {
    VaeLevelW& lv = v.levels[level];
    const std::string p = "encoder.down." + std::to_string(level);
    const int bo = ch * cfg.channel_mult[level];
    lv.blocks.resize(nrb);
    for (int j = 0; j < nrb; ++j, bi = bo) ECHK(build_res(lv.blocks[j], p + ".block." + std::to_string(j), bi, bo, VAE_RES));
    lv.has_resample = level != nl - 1;
    if (lv.has_resample) ECHK(pack_conv3(lv.resample, p + ".downsample.conv", bi, bi));
  }
  ECHK(build_vae_mid(v.mid, "encoder.mid", bi));
  ECHK(pack_norm(v.norm_out, "encoder.norm_out", bi));
  ECHK(pack_conv3(v.conv_out, "encoder.conv_out", 2 * z, bi));
  return pack_dense(v.quant, "quant_conv", 2 * z, 2 * z);
}

// =================================================================================================================
// CLIP text transformer weights (Hugging Face CLIPTextModel names; open_clip towers are renamed on the host)
// =================================================================================================================
int sdxe_engine::build_clip(ClipW& c) {
  const int C = cfg.clip_hidden, I = cfg.clip_intermediate, L = cfg.clip_layers;
  const std::string tm = "text_model.";
  c.tok = alloc16((size_t)cfg.clip_vocab * C);
  c.pos = alloc16((size_t)cfg.clip_positions * C);
  const RawWeight* wt = find(tm + "embeddings.token_embedding.weight", (int64_t)cfg.clip_vocab * C);
  const RawWeight* wp = find(tm + "embeddings.position_embedding.weight", (int64_t)cfg.clip_positions * C);
  if (!sizing && wt) ECHK(pack_weight_launch(wt->dev, wt->dtype, c.tok, PACK_PLAIN, cfg.clip_vocab, C, C, 0, bf16, 0));
  if (!sizing && wp) ECHK(pack_weight_launch(wp->dev, wp->dtype, c.pos, PACK_PLAIN, cfg.clip_positions, C, C, 0, bf16, 0));
  c.layers.resize(L);
  for (int l = 0; l < L; ++l) {
    ClipLayerW& w = c.layers[l];
    const std::string p = tm + "encoder.layers." + std::to_string(l) + ".";
    NormW ln1, ln2;
    ECHK(pack_norm(ln1, p + "layer_norm1", C));
    ECHK(pack_norm(ln2, p + "layer_norm2", C));
    ECHK(pack_linear(w.qkv, {p + "self_attn.q_proj.weight", p + "self_attn.k_proj.weight", p + "self_attn.v_proj.weight"},
                     {p + "self_attn.q_proj.bias", p + "self_attn.k_proj.bias", p + "self_attn.v_proj.bias"}, C, C, PACK_PLAIN));
    ECHK(pack_dense(w.out, p + "self_attn.out_proj", C, C));
    ECHK(pack_dense(w.fc1, p + "mlp.fc1", I, C));
    ECHK(pack_dense(w.fc2, p + "mlp.fc2", C, I));
    ECHK(fold_layer_norm(w.qkv, ln1));
    ECHK(fold_layer_norm(w.fc1, ln2));
  }
  return pack_norm(c.final_norm, tm + "final_layer_norm", C);
}

// =================================================================================================================
// engine: activation pool
// =================================================================================================================
Buf sdxe_engine::alloc(size_t bytes) {
  bytes = align_up(std::max<size_t>(bytes, 256), 1024);
  Buf b;
  auto it = free_list.lower_bound(bytes);
  if (it != free_list.end() && it->first <= bytes + bytes / 2 + (1 << 20)) {
    b = Buf{it->second, it->first};
    free_list.erase(it);
  } else {
    void* p = nullptr;
    if (cudaMalloc(&p, bytes) != cudaSuccess) {
      cudaGetLastError();  // clear the sticky error; the plan build is abandoned by its caller (alloc_failed)
      set_last_error(__FILE__, __LINE__, "cudaMalloc failed (activation pool)");
      alloc_failed = true;
      return Buf();
    }
    all_allocs.push_back(p);
    b = Buf{p, bytes};
  }
  if (track) track->push_back(b);
  if (touched) touched->push_back(b.p);
  return b;
}
void sdxe_engine::release(Buf& b) {
  if (b.p) {
    free_list.insert({b.bytes, b.p});
    if (track) {
      for (size_t i = track->size(); i-- > 0;)
        if ((*track)[i].p == b.p) { track->erase(track->begin() + i); break; }
    }
  }
  b.p = nullptr;
}
// =================================================================================================================
// plans
// =================================================================================================================
namespace {

int run_ops(std::vector<OpRec>& ops, cudaStream_t s) {
  for (auto& r : ops) ECHK(r.fn(s));
  return 0;
}

// Profiling pass: every body op bracketed by CUDA events on the launching stream (eager, no graph).
int run_ops_profiled(sdxe_engine* e, std::vector<OpRec>& ops, cudaStream_t s);

int run_plan(sdxe_engine* e, Plan* p, cudaStream_t stream) {
  ECHK(run_ops(p->pre, stream));
  if (e->profiling) {
    ECHK(run_ops_profiled(e, p->body, stream));
  } else {
    if (!p->gexec) {
      // capture the body once on a private stream, then replay on the caller's stream
      if (!e->cap_stream) SDXE_CUDA_CHECK(cudaStreamCreateWithFlags(&e->cap_stream, cudaStreamNonBlocking));
      SDXE_CUDA_CHECK(cudaStreamBeginCapture(e->cap_stream, cudaStreamCaptureModeThreadLocal));
      const int64_t l0 = launch_count();
      int rc = run_ops(p->body, e->cap_stream);
      p->launches_body = (int)(launch_count() - l0);
      cudaGraph_t g = nullptr;
      cudaError_t ce = cudaStreamEndCapture(e->cap_stream, &g);
      if (rc != 0) { if (g) cudaGraphDestroy(g); return -1; }
      SDXE_CUDA_CHECK(ce);
      p->graph = g;
      SDXE_CUDA_CHECK(cudaGraphInstantiate(&p->gexec, g, 0));
    } else {
      count_launch(p->launches_body);
    }
    SDXE_CUDA_CHECK(cudaGraphLaunch(p->gexec, stream));
  }
  ECHK(run_ops(p->post, stream));
  return 0;
}

int run_ops_profiled(sdxe_engine* e, std::vector<OpRec>& ops, cudaStream_t s) {
  const size_t n = ops.size();
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& x : ev) SDXE_CUDA_CHECK(cudaEventCreate(&x));
  int rc = 0;
  SDXE_CUDA_CHECK(cudaEventRecord(ev[0], s));
  for (size_t i = 0; i < n && rc == 0; ++i) {
    rc = ops[i].fn(s);
    cudaEventRecord(ev[i + 1], s);
  }
  cudaStreamSynchronize(s);
  if (rc == 0) {
    const char* dump = getenv("SDXE_PROFILE_DUMP");
    FILE* df = dump ? fopen(dump, "a") : nullptr;
    for (size_t i = 0; i < n; ++i) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, ev[i], ev[i + 1]);
      if (df) fprintf(df, "%zu,%d,%s,%.4f,%.0f,%.0f\n", i, ops[i].kind, ops[i].desc.c_str(), ms * 1000.0, ops[i].flops, ops[i].bytes);
      const int k = ops[i].kind;
      e->prof_ms[k] += ms;
      e->prof_flops[k] += ops[i].flops;
      e->prof_bytes[k] += ops[i].bytes;
      e->prof_launches[k] += 1;
    }
    if (df) fclose(df);
  }
  for (auto& x : ev) cudaEventDestroy(x);
  return rc;
}

// ---- UNet plan -----------------------------------------------------------------------------------------------
int build_unet_plan(sdxe_engine* e, Plan* p, int n, int h, int w, int ctx_len, const std::vector<int32_t>* ht) {
  const sdxe_config& cfg = e->cfg;
  const UNetW& u = *e->unet;
  Builder B(e, p);
  const bool bf16 = e->bf16;
  const int mc = cfg.model_channels, ted = 4 * mc;
  if (ht) {  // Hypertile: the draws are data, written per call into a plan-owned table that the tiled layers read
    Buf table = e->alloc(sizeof(int) * ht->size() / 5 * 2);
    int* tp = (int*)table.p;
    p->pre.push_back([=](cudaStream_t s) { return hypertile_table_launch(p->ht_draws, tp, s); });
    B.ht = ht;
    B.ht_table = tp;
  }

  // ---- pre: caller tensors -> plan-owned buffers (outside the graph: caller pointers change per call)
  Buf ctx16 = e->alloc((size_t)n * ctx_len * cfg.context_dim * 2);
  Buf temb = e->alloc(sizeof(float) * n * mc);
  Buf y32 = e->alloc(sizeof(float) * std::max(1, n * cfg.adm_in_channels));
  {
    float* te = (float*)temb.p; float* yy = (float*)y32.p;
    const int adm = cfg.adm_in_channels;
    p->pre.push_back([=](cudaStream_t s) { return timestep_embedding_launch(p->t, p->io_dtype, te, n, mc, bf16, s); });
    if (adm > 0)
      p->pre.push_back([=](cudaStream_t s) {
        if (!p->y) { set_last_error(__FILE__, __LINE__, "unet_forward: y (vector conditioning) required"); return -1; }
        return cast_to_f32_launch(p->y, p->io_dtype, yy, (int64_t)n * adm, true, bf16, s);
      });
  }
  // ---- embeddings (fp32 vectors rounded through the 16-bit type where the reference's autocast rounds)
  Buf e1 = e->alloc(sizeof(float) * n * ted), emb = e->alloc(sizeof(float) * n * ted), l1 = e->alloc(sizeof(float) * n * ted);
  Buf emb_all = e->alloc(sizeof(float) * n * u.emb_total);
  {
    const LinW te0 = u.te0, te2 = u.te2, le0 = u.le0, le2 = u.le2, ea = u.emb_all;
    float *pt = (float*)temb.p, *p1 = (float*)e1.p, *pe = (float*)emb.p, *pl = (float*)l1.p, *pa = (float*)emb_all.p, *py = (float*)y32.p;
    const int adm = cfg.adm_in_channels, etot = u.emb_total;
    // time_embed = Linear -> SiLU -> Linear; every consumer of `emb` (the ResBlocks' emb_layers) applies SiLU first,
    // so the SiLU'd vector is what gets stored (rounded through the 16-bit type at each step like the reference).
    B.ops->push_back([=](cudaStream_t s) { return skinny_linear_launch(pt, mc, te0.w, te0.b, nullptr, p1, ted, n, ted, mc, true, bf16, s); });
    if (adm > 0) {
      // emb = time_embed(t_emb) + label_emb(y): label branch first, the sum happens inside the last time_embed GEMM
      B.ops->push_back([=](cudaStream_t s) { return skinny_linear_launch(py, adm, le0.w, le0.b, nullptr, pl, ted, n, ted, adm, true, bf16, s); });
      B.ops->push_back([=](cudaStream_t s) { return skinny_linear_launch(pl, ted, le2.w, le2.b, nullptr, pe, ted, n, ted, ted, false, bf16, s); });
      B.ops->push_back([=](cudaStream_t s) { return skinny_linear_launch(p1, ted, te2.w, te2.b, pe, pe, ted, n, ted, ted, true, bf16, s); });
    } else {
      B.ops->push_back([=](cudaStream_t s) { return skinny_linear_launch(p1, ted, te2.w, te2.b, nullptr, pe, ted, n, ted, ted, true, bf16, s); });
    }
    B.ops->push_back([=](cudaStream_t s) { return skinny_linear_launch(pe, ted, ea.w, ea.b, nullptr, pa, etot, n, etot, ted, false, bf16, s); });
  }
  B.emb = (const float*)emb_all.p;
  B.ld_emb = u.emb_total;
  // ---- cross-attention keys / values of ALL transformer blocks: one GEMM over the context (plan-owned buffer)
  Buf kvbuf = e->alloc((size_t)n * ctx_len * std::max(8, u.kv_total) * 2);
  {
    // runs before the graph, and only when the context changed (ctx_key): cast the caller's context, project it once
    auto kv_ops = std::make_shared<std::vector<OpRec>>();
    if (u.kv_total > 0) {
      B.ops = kv_ops.get();
      const int rc = B.gemm(ctx16.p, cfg.context_dim, (int64_t)n * ctx_len, u.kv_all, kvbuf.p, Builder::GemmOpt());
      B.ops = &p->body;
      ECHK(rc);
    }
    void* cx = ctx16.p;
    const int cdim = cfg.context_dim;
    const UNetW* up = &u;
    p->pre.push_back([=](cudaStream_t s) {
      if (up->ctx_key != 0 && p->kv_key == up->ctx_key && !e->profiling) return 0;
      ECHK(cast_rows_launch(p->ctx, p->io_dtype, cx, (int64_t)n * ctx_len, cdim, cdim, bf16, s));
      if (e->profiling) ECHK(run_ops_profiled(e, *kv_ops, s));
      else ECHK(run_ops(*kv_ops, s));
      p->kv_key = up->ctx_key;
      return 0;
    });
  }
  auto transformer = [&](const UNetBlockW& b, Act& x) { return b.has_st ? B.spatial_transformer(b.st, x, kvbuf.p, u.kv_total, ctx_len) : 0; };

  // ---- input blocks; every output stays alive on the skip stack
  std::vector<Act> hs;
  Act cur;
  ECHK(B.conv_in_nchw(nullptr, n, cfg.in_channels, h, w, u.conv_in, cur));
  hs.push_back(cur);
  for (const UNetLevelW& lv : u.in_levels) {
    for (const UNetBlockW& b : lv.blocks) {
      Act r;
      ECHK(B.res_block(b.res, cur, nullptr, 1e-5f, r));
      ECHK(transformer(b, r));
      cur = r;
      hs.push_back(cur);
    }
    if (lv.has_down) {
      const int Ho = (cur.h + 2 - 3) / 2 + 1, Wo = (cur.w + 2 - 3) / 2 + 1;
      Act d = B.new_act(n, Ho, Wo, lv.down.N);
      ECHK(B.conv3(cur, lv.down, d.p, lv.down.N, Builder::GemmOpt(), 2, 1, Ho, Wo));
      cur = d;
      hs.push_back(cur);
    }
  }
  // ---- middle (its input, the last input block's output, stays on the skip stack)
  Act r;
  ECHK(B.res_block(u.mid_r1, cur, nullptr, 1e-5f, r));
  ECHK(B.spatial_transformer(u.mid_st, r, kvbuf.p, u.kv_total, ctx_len));
  ECHK(B.res_replace(u.mid_r2, r, 1e-5f));
  cur = r;
  // ---- output blocks
  for (const UNetBlockW& b : u.out_blocks) {
    Act skip = hs.back();
    hs.pop_back();
    if (skip.h != cur.h || skip.w != cur.w) EFAIL("unet: skip / hidden size mismatch (latent size must be divisible by 2^(levels-1))");
    ECHK(B.res_replace(b.res, cur, 1e-5f, &skip));
    B.free_act(skip);
    ECHK(transformer(b, cur));
    if (b.has_up) ECHK(B.upsample_conv(cur, b.up));
  }
  // ---- out: GN + SiLU + conv3 -> [M, 8] (4 valid channels)
  ECHK(B.out_head(cur, u.out_norm, 1e-5f, u.out_conv));
  // plan-owned buffers (conv_in's im2col, ctx16, temb, y32, e1, emb, l1, emb_all, kvbuf, out_head's output) stay reserved for this plan
  return 0;
}

// post_quant_conv on the caller's NCHW latent (z channels, tiny): fp32 weights, output rounded to 16-bit, NCHW
template <bool BF16>
__global__ void post_quant_kernel(const void* __restrict__ z, int io_dtype, const float* __restrict__ w,
                                  const float* __restrict__ b, typename T16<BF16>::type* __restrict__ out, int n, int C, int hw) {
  const int64_t total = (int64_t)n * C * hw;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int p = (int)(idx % hw);
    const int co = (int)((idx / hw) % C);
    const int img = (int)(idx / ((int64_t)hw * C));
    float acc = b[co];
    for (int ci = 0; ci < C; ++ci) {
      const int64_t si = ((int64_t)img * C + ci) * hw + p;
      float v;
      if (io_dtype == DT_F16) v = __half2float(reinterpret_cast<const __half*>(z)[si]);
      else if (io_dtype == DT_BF16) v = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(z)[si]);
      else v = reinterpret_cast<const float*>(z)[si];
      // the reference feeds the VAE in dtype_vae (sd_samplers_common.py:58): round the latent first
      v = T16<BF16>::to_f(T16<BF16>::from_f(v));
      acc = fmaf(w[co * C + ci], v, acc);
    }
    out[idx] = T16<BF16>::from_f(acc);
  }
}

// AutoencoderKL.encode up to the moments: x [n, 3, H, W] -> [n, 2z, H/8, W/8]
int build_vae_encode_plan(sdxe_engine* e, Plan* p, int n, int H, int W) {
  const sdxe_config& cfg = e->cfg;
  const VaeW& v = *e->vae;
  Builder B(e, p);
  const bool bf16 = e->bf16;
  const int z2 = 2 * cfg.vae_z_channels;
  Act cur;
  ECHK(B.conv_in_nchw(nullptr, n, cfg.vae_out_ch, H, W, v.conv_in, cur));
  for (const VaeLevelW& lv : v.levels) {
    for (const ResW& r : lv.blocks) ECHK(B.res_replace(r, cur, 1e-6f));
    if (lv.has_resample) {
      // ldm Downsample (with_conv): pad (0,1,0,1) then conv3x3 stride 2, padding 0 -> taps start at the pixel itself
      const int Ho = cur.h / 2, Wo = cur.w / 2;
      Act d = B.new_act(n, Ho, Wo, cur.c);
      ECHK(B.conv3(cur, lv.resample, d.p, cur.c, Builder::GemmOpt(), 2, 0, Ho, Wo));
      B.free_act(cur);
      cur = d;
    }
  }
  ECHK(B.vae_mid(v.mid, cur));
  Act g;
  ECHK(B.group_norm(cur, nullptr, v.norm_out, 1e-6f, true, g));
  const int Ho = cur.h, Wo = cur.w;
  B.free_act(cur);
  const int ld8 = (int)align_up(z2, 8);
  Act mo = B.new_act(n, Ho, Wo, ld8);
  ECHK(B.conv3(g, v.conv_out, mo.p, ld8, Builder::GemmOpt()));
  B.free_act(g);
  Buf outb = e->alloc((size_t)n * Ho * Wo * ld8 * 2);
  ECHK(B.gemm(mo.p, ld8, (int64_t)n * Ho * Wo, v.quant, outb.p, Builder::GemmOpt()));  // quant_conv (1x1)
  B.free_act(mo);
  {
    void* ob = outb.p;
    const int hw = Ho * Wo;
    p->post.push_back([=](cudaStream_t s) { return nhwc_to_nchw_launch(ob, ld8, p->out, p->io_dtype, n, z2, hw, bf16, s); });
  }
  return 0;
}

int build_vae_plan(sdxe_engine* e, Plan* p, int n, int h, int w) {
  const VaeW& v = *e->vae;
  Builder B(e, p);
  const bool bf16 = e->bf16;
  const int z = e->cfg.vae_z_channels;
  Buf zq = e->alloc((size_t)n * h * w * z * 2);
  {
    void* zp = zq.p;
    const float *pw = v.pq_w, *pb = v.pq_b;
    const int hw = h * w;
    p->pre.push_back([=](cudaStream_t s) {
      const int64_t total = (int64_t)n * z * hw;
      const int blocks = (int)std::min<int64_t>((total + 255) / 256, 4096);
      if (bf16) post_quant_kernel<true><<<blocks, 256, 0, s>>>(p->x, p->io_dtype, pw, pb, (__nv_bfloat16*)zp, n, z, hw);
      else post_quant_kernel<false><<<blocks, 256, 0, s>>>(p->x, p->io_dtype, pw, pb, (__half*)zp, n, z, hw);
      SDXE_LAUNCH_CHECK();
      return 0;
    });
  }
  Act cur;
  ECHK(B.conv_in_nchw(zq.p, n, z, h, w, v.conv_in, cur));
  ECHK(B.vae_mid(v.mid, cur));
  for (auto lv = v.levels.rbegin(); lv != v.levels.rend(); ++lv) {
    for (const ResW& r : lv->blocks) ECHK(B.res_replace(r, cur, 1e-6f));
    if (lv->has_resample) ECHK(B.upsample_conv(cur, lv->resample));
  }
  return B.out_head(cur, v.norm_out, 1e-6f, v.conv_out);
}

// hidden_states[layer] (optionally + final_layer_norm) of the text transformer for n sequences of T tokens
int build_clip_plan(sdxe_engine* e, Plan* plan, int n, int T, int layer, int final_norm) {
  const sdxe_config& cfg = e->cfg;
  const ClipW& c = *e->clip;
  const int C = cfg.clip_hidden, I = cfg.clip_intermediate, H = cfg.clip_heads, d = C / H;
  const int64_t M = (int64_t)n * T;
  const bool b = e->bf16;
  Builder B(e, plan);
  Buf x = e->alloc((size_t)M * C * 2);
  Builder::RowStats st;
  st.buf = e->alloc((size_t)M * sizeof(float2));
  st.p = (const float2*)st.buf.p;
  st.parts = 1;
  {
    void* xp = x.p;
    float2* sp = (float2*)st.buf.p;
    const void *tok = c.tok, *pos = c.pos;
    const int vocab = cfg.clip_vocab;
    plan->pre.push_back([=](cudaStream_t s) {
      ECHK(clip_embed_launch((const int32_t*)plan->x, tok, pos, xp, sp, (int)M, T, C, vocab, b, s));
      return clip_fix_launch(plan->fix_rows, plan->fix_vecs, pos, xp, sp, plan->n_fix, (int)M, T, C, b, s);
    });
  }
  const float scale = 1.0f / sqrtf((float)d);
  for (int l = 0; l < layer; ++l) {
    const ClipLayerW& w = c.layers[l];
    Buf qkv = e->alloc((size_t)M * 3 * C * 2);
    Builder::GemmOpt oq;
    oq.ln_part = st.p; oq.ln_parts = st.parts;
    ECHK(B.gemm(x.p, C, M, w.qkv, qkv.p, oq));
    B.free_stats(st);
    Buf att = e->alloc((size_t)M * C * 2);
    {
      const void* qp = qkv.p;
      void* ap = att.p;
      B.ops->push_back(OpRec([=](cudaStream_t s) { return causal_attn_small_launch(qp, ap, n, T, H, d, scale, b, s); }, K_ATTN,
                             2.0 * n * H * (double)T * T * d, 2.0 * (double)M * 4 * C, "causal attn"));
    }
    e->release(qkv);
    Buf x2 = e->alloc((size_t)M * C * 2);
    Builder::GemmOpt oo;
    oo.residual = x.p; oo.ldr = C; oo.emit = &st;
    ECHK(B.gemm(att.p, C, M, w.out, x2.p, oo));
    e->release(att);
    e->release(x);
    x = x2;
    Buf hmid = e->alloc((size_t)M * I * 2);
    Builder::GemmOpt o1;
    o1.ln_part = st.p; o1.ln_parts = st.parts;
    ECHK(B.gemm(x.p, C, M, w.fc1, hmid.p, o1));
    B.free_stats(st);
    {
      void* hp = hmid.p;
      const int mode = cfg.clip_act;
      B.ops->push_back(OpRec([=](cudaStream_t s) { return act_inplace_launch(hp, M * (int64_t)I, mode, b, s); }, K_OTHER, 0.0,
                             4.0 * (double)M * I, "clip act"));
    }
    Buf x3 = e->alloc((size_t)M * C * 2);
    Builder::GemmOpt o2;
    o2.residual = x.p; o2.ldr = C;
    if (l + 1 < layer) o2.emit = &st;
    ECHK(B.gemm(hmid.p, I, M, w.fc2, x3.p, o2));
    e->release(hmid);
    e->release(x);
    x = x3;
  }
  if (layer == 0) B.free_stats(st);
  Buf y = x;
  if (final_norm) {
    y = e->alloc((size_t)M * C * 2);
    const void* xp = x.p;
    void* yp = y.p;
    const float *g = c.final_norm.g, *bt = c.final_norm.b;
    B.ops->push_back(OpRec([=](cudaStream_t s) { return layer_norm_launch(xp, g, bt, yp, (int)M, C, 1e-5f, b, s); }, K_LNORM, 0.0,
                           4.0 * (double)M * C, "final_layer_norm"));
  }
  {
    const void* yp = y.p;
    const int dt = e->dt;
    plan->post.push_back([=](cudaStream_t s) {
      if (plan->io_dtype == SDXE_F32) return cast_to_f32_launch(yp, dt, (float*)plan->out, M * (int64_t)C, false, b, s);
      SDXE_CUDA_CHECK(cudaMemcpyAsync(plan->out, yp, (size_t)M * C * 2, cudaMemcpyDeviceToDevice, s));
      return 0;
    });
  }
  return 0;
}

// =================================================================================================================
// plan cache
// =================================================================================================================
// Drop the least recently used plan: its graph is destroyed and the buffers it pinned go back to the pool; pool memory
// beyond pool_limit is returned to the driver (largest blocks first).
void evict_lru(sdxe_engine* e) {
  auto victim = e->plans.end();
  for (auto it = e->plans.begin(); it != e->plans.end(); ++it)
    if (victim == e->plans.end() || it->second->last_use < victim->second->last_use) victim = it;
  if (victim == e->plans.end()) return;
  cudaDeviceSynchronize();  // the plan's last replay may still be running
  for (auto& b : victim->second->owned)
    if (b.p) e->free_list.insert({b.bytes, b.p});
  e->plans.erase(victim);
  // free-list blocks double as scratch of the plans that are still cached: only blocks no live plan touches may go
  size_t free_bytes = 0;
  for (auto& kv : e->free_list) free_bytes += kv.first;
  if (free_bytes <= e->pool_limit) return;
  std::vector<void*> live;
  for (auto& kv : e->plans) live.insert(live.end(), kv.second->used.begin(), kv.second->used.end());
  std::sort(live.begin(), live.end());
  for (auto it = e->free_list.end(); it != e->free_list.begin() && free_bytes > e->pool_limit;) {
    --it;
    if (std::binary_search(live.begin(), live.end(), it->second)) continue;
    free_bytes -= it->first;
    cudaFree(it->second);
    e->all_allocs.erase(std::remove(e->all_allocs.begin(), e->all_allocs.end(), it->second), e->all_allocs.end());
    it = e->free_list.erase(it);
  }
}

template <class BuildFn>
Plan* get_plan(sdxe_engine* e, const std::string& key, BuildFn build) {
  auto it = e->plans.find(key);
  if (it != e->plans.end()) {
    it->second->last_use = ++e->tick;
    return it->second.get();
  }
  while ((int)e->plans.size() >= e->max_plans) evict_lru(e);
  for (int attempt = 0; attempt < 2; ++attempt) {
    std::unique_ptr<Plan> p(new Plan());
    p->e = e;
    std::vector<Buf> held;
    std::vector<void*> used;
    e->track = &held;
    e->touched = &used;
    e->alloc_failed = false;
    const int rc = build(p.get());
    e->track = nullptr;
    e->touched = nullptr;
    if (rc == 0 && !e->alloc_failed) {
      std::sort(used.begin(), used.end());
      used.erase(std::unique(used.begin(), used.end()), used.end());
      p->used = std::move(used);
      p->owned = std::move(held);
      p->last_use = ++e->tick;
      return e->plans.emplace(key, std::move(p)).first->second.get();
    }
    for (auto& b : held)  // a failed build leaks nothing: whatever it still held goes back to the pool
      if (b.p) e->free_list.insert({b.bytes, b.p});
    if (!e->alloc_failed || attempt == 1) break;
    // out of device memory: drop every cached plan and the whole free pool, then try once more
    while (!e->plans.empty()) evict_lru(e);
    cudaDeviceSynchronize();
    for (auto& kv : e->free_list) {
      cudaFree(kv.second);
      e->all_allocs.erase(std::remove(e->all_allocs.begin(), e->all_allocs.end(), kv.second), e->all_allocs.end());
    }
    e->free_list.clear();
  }
  if (e->alloc_failed) set_last_error(__FILE__, __LINE__, "out of device memory while building the execution plan");
  return nullptr;
}

// One model forward: `e` must be a finalized engine of `kind` and io_dtype a type it reads and writes; `args` checks the
// remaining arguments and may extend the plan key; the plan for the key is fetched or built, gets this call's pointers
// (x, out, io_dtype, then `bind`) and runs on `stream`. `entry` / `model` name the call and the model in error messages.
int run_forward(sdxe_engine* e, int kind, const char* entry, const char* model, int io_dtype, std::string key,
                const std::function<int(std::string& key)>& args, const std::function<int(Plan*)>& build, const void* x,
                void* out, void* stream, const std::function<void(Plan*)>& bind = nullptr) {
  if (!e || !e->finalized || e->cfg.kind != kind) EFAIL((std::string(entry) + ": engine is not a finalized " + model).c_str());
  if (kind == SDXE_MODEL_CLIP_TEXT ? io_dtype != e->dt && io_dtype != SDXE_F32
                                   : io_dtype != SDXE_F16 && io_dtype != SDXE_BF16 && io_dtype != SDXE_F32)
    EFAIL((std::string(entry) + (kind == SDXE_MODEL_CLIP_TEXT ? ": out must be the engine's 16-bit type or fp32" : ": io dtype")).c_str());
  ECHK(args(key));
  if (e->circular) key += ":circ";  // only UNet and VAE engines take Tiling (sdxe_set_circular)
  Plan* p = get_plan(e, key, build);
  if (!p) return -1;
  p->x = x; p->out = out; p->io_dtype = io_dtype;
  if (bind) bind(p);
  return run_plan(e, p, (cudaStream_t)stream);
}

std::string dims_key(char tag, std::initializer_list<int> dims) {
  std::string key(1, tag);
  for (int d : dims) key += ":" + std::to_string(d);
  return key;
}

}  // namespace

// =================================================================================================================
// C-ABI
// =================================================================================================================
extern "C" {

int sdxe_create(const sdxe_config* cfg, sdxe_engine** out) {
  if (!cfg || !out) EFAIL("sdxe_create: null argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) EFAIL("sdxe_create: no CUDA device (this engine has no CPU path)");
  if (cfg->dtype != SDXE_F16 && cfg->dtype != SDXE_BF16) EFAIL("sdxe_create: dtype must be F16 or BF16");
  if (cfg->kind != SDXE_MODEL_CLIP_TEXT && (cfg->num_levels < 1 || cfg->num_levels > SDXE_MAX_LEVELS)) EFAIL("sdxe_create: num_levels");
  if (cfg->kind == SDXE_MODEL_UNET) {
    if (cfg->model_channels % 32) EFAIL("sdxe_create: model_channels must be a multiple of 32");
    if (cfg->context_dim % 8) EFAIL("sdxe_create: context_dim % 8");
  } else if (cfg->kind == SDXE_MODEL_VAE_DECODER || cfg->kind == SDXE_MODEL_VAE_ENCODER) {
    if (cfg->vae_ch % 32) EFAIL("sdxe_create: vae_ch must be a multiple of 32");
  } else if (cfg->kind == SDXE_MODEL_CLIP_TEXT) {
    if (cfg->clip_hidden % 64 || cfg->clip_heads < 1 || cfg->clip_hidden % cfg->clip_heads || (cfg->clip_hidden / cfg->clip_heads) % 8 ||
        cfg->clip_intermediate % 64 || cfg->clip_layers < 1 || cfg->clip_vocab < 2 || cfg->clip_positions < 1 || cfg->clip_positions > 128)
      EFAIL("sdxe_create: CLIP text config");
  } else {
    EFAIL("sdxe_create: unknown model kind");
  }
  sdxe_engine* e = new sdxe_engine();
  e->cfg = *cfg;
  e->bf16 = cfg->dtype == SDXE_BF16;
  e->dt = cfg->dtype;
  switch (cfg->kind) {
    case SDXE_MODEL_UNET: e->unet.reset(new UNetW()); break;
    case SDXE_MODEL_CLIP_TEXT: e->clip.reset(new ClipW()); break;
    default: e->vae.reset(new VaeW()); break;
  }
  if (gemm_init() != 0 || attention_init() != 0 || kernels_init() != 0) { delete e; return -1; }
  *out = e;
  return 0;
}

void sdxe_destroy(sdxe_engine* e) {
  if (!e) return;
  cudaDeviceSynchronize();
  delete e;
}

int sdxe_set_weight(sdxe_engine* e, const char* key, const void* data, int dtype, int ndim, const int64_t* shape) {
  if (!e || !key || !data) EFAIL("sdxe_set_weight: null argument");
  if (e->finalized) EFAIL("sdxe_set_weight: engine already finalized");
  if (dtype != SDXE_F16 && dtype != SDXE_BF16 && dtype != SDXE_F32) EFAIL("sdxe_set_weight: dtype");
  RawWeight w;
  w.dtype = dtype;
  w.numel = 1;
  for (int i = 0; i < ndim; ++i) { w.shape.push_back(shape[i]); w.numel *= shape[i]; }
  const size_t bytes = (size_t)w.numel * (dtype == SDXE_F32 ? 4 : 2);
  SDXE_CUDA_CHECK(cudaMalloc(&w.dev, std::max<size_t>(bytes, 16)));
  SDXE_CUDA_CHECK(cudaMemcpy(w.dev, data, bytes, cudaMemcpyDefault));
  auto it = e->raw.find(key);
  if (it != e->raw.end()) {
    e->params -= it->second.numel;
    cudaFree(it->second.dev);
  }
  e->raw[key] = w;
  e->params += w.numel;
  return 0;
}

int64_t sdxe_param_count(const sdxe_engine* e) { return e ? e->params : -1; }

int sdxe_finalize(sdxe_engine* e) {
  if (!e) EFAIL("sdxe_finalize: null");
  if (e->finalized) return 0;
  for (int pass = 0; pass < 2; ++pass) {
    e->sizing = pass == 0;
    e->cursor = 0;
    e->missing.clear();
    int rc;
    switch (e->cfg.kind) {
      case SDXE_MODEL_UNET: rc = e->build_unet(*e->unet); break;
      case SDXE_MODEL_VAE_ENCODER: rc = e->build_vae_encoder(*e->vae); break;
      case SDXE_MODEL_CLIP_TEXT: rc = e->build_clip(*e->clip); break;
      default: rc = e->build_vae_decoder(*e->vae); break;
    }
    if (rc != 0) return -1;
    if (!e->missing.empty()) {
      std::string m = "sdxe_finalize: missing / mis-shaped weights: " + e->missing;
      set_last_error(__FILE__, __LINE__, m.c_str());
      return -3;
    }
    if (pass == 0) {
      e->blob_bytes = align_up(e->cursor, 256);
      SDXE_CUDA_CHECK(cudaMalloc((void**)&e->blob, e->blob_bytes));
      SDXE_CUDA_CHECK(cudaMemset(e->blob, 0, e->blob_bytes));
    }
  }
  SDXE_CUDA_CHECK(cudaDeviceSynchronize());
  for (auto& kv : e->raw) {
    if (kv.second.dev) cudaFree(kv.second.dev);
    kv.second.dev = nullptr;
  }
  e->finalized = true;
  return 0;
}

int sdxe_weight_blob(sdxe_engine* e, void** device_ptr, int64_t* bytes) {
  if (!e || !e->finalized) EFAIL("sdxe_weight_blob: engine not finalized");
  *device_ptr = e->blob;
  *bytes = (int64_t)e->blob_bytes;
  return 0;
}

int sdxe_unet_forward(sdxe_engine* e, const void* x, const void* t, const void* ctx, const void* y, void* out, int n,
                      int h, int w, int ctx_len, int io_dtype, void* stream) {
  std::vector<int32_t> ht;
  HtDraws draws;
  auto args = [&](std::string& key) {
    if (!x || !t || !ctx || !out || n <= 0 || h <= 0 || w <= 0 || ctx_len <= 0) EFAIL("sdxe_unet_forward: bad argument");
    ht.swap(e->unet->ht_rows);  // a Hypertile table applies to one call
    if (ht.empty()) return 0;
    // the plan is keyed on the structural part (h', w', max_tiles per layer); the draws (nh, nw) are data
    draws.n = (int)ht.size() / 5;
    if (draws.n != e->unet->n_attn1) EFAIL("sdxe_unet_forward: the Hypertile table needs one row per attn1 layer");
    key += ":ht";
    for (int i = 0; i < draws.n; ++i) {
      const int32_t* r = &ht[5 * i];
      const int hp = r[0], wp = r[1], nh = r[2], nw = r[3], mt = r[4];
      if (mt > 0 ? (hp < 1 || wp < 1 || nh < 1 || nw < 1 || hp % nh || wp % nw || nh * nw > mt) : (nh != 1 || nw != 1))
        EFAIL("sdxe_unet_forward: bad Hypertile row (nh | h', nw | w', nh * nw <= max_tiles; untiled rows draw (1, 1))");
      draws.v[2 * i] = nh;
      draws.v[2 * i + 1] = nw;
      key += mt > 0 ? "," + std::to_string(hp) + "x" + std::to_string(wp) + "/" + std::to_string(mt) : ",-";
    }
    return 0;
  };
  return run_forward(e, SDXE_MODEL_UNET, "sdxe_unet_forward", "UNet", io_dtype, dims_key('u', {n, h, w, ctx_len}), args,
                     [&](Plan* pl) { return build_unet_plan(e, pl, n, h, w, ctx_len, ht.empty() ? nullptr : &ht); }, x, out, stream,
                     [&](Plan* p) {
                       if (!ht.empty()) p->ht_draws = draws;
                       p->t = t; p->ctx = ctx; p->y = y;
                     });
}

int sdxe_clip_forward(sdxe_engine* e, const int32_t* tokens, void* out, int n, int T, int layer, int final_norm, int io_dtype,
                      void* stream) {
  return sdxe_clip_forward_fixes(e, tokens, out, n, T, layer, final_norm, io_dtype, nullptr, nullptr, 0, stream);
}

int sdxe_clip_forward_fixes(sdxe_engine* e, const int32_t* tokens, void* out, int n, int T, int layer, int final_norm, int io_dtype,
                            const int32_t* fix_rows, const void* fix_vecs, int n_fix, void* stream) {
  const int fnorm = final_norm ? 1 : 0;
  auto args = [&](std::string&) {
    if (!tokens || !out || n <= 0 || T <= 0 || T > e->cfg.clip_positions || layer < 0 || layer > e->cfg.clip_layers) EFAIL("sdxe_clip_forward: bad argument");
    if (n_fix < 0 || (n_fix > 0 && (!fix_rows || !fix_vecs))) EFAIL("sdxe_clip_forward_fixes: bad fix arguments");
    return 0;
  };
  return run_forward(e, SDXE_MODEL_CLIP_TEXT, "sdxe_clip_forward", "CLIP text model", io_dtype, dims_key('c', {n, T, layer, fnorm}),
                     args, [&](Plan* pl) { return build_clip_plan(e, pl, n, T, layer, fnorm); }, tokens, out, stream,
                     [&](Plan* p) { p->fix_rows = fix_rows; p->fix_vecs = fix_vecs; p->n_fix = n_fix; });
}

int sdxe_unet_set_context_key(sdxe_engine* e, int64_t key) {
  if (!e || e->cfg.kind != SDXE_MODEL_UNET) EFAIL("sdxe_unet_set_context_key: not a UNet engine");
  e->unet->ctx_key = key;
  return 0;
}

int sdxe_unet_set_hypertile(sdxe_engine* e, const int32_t* layers, int n_layers) {
  if (!e || e->cfg.kind != SDXE_MODEL_UNET) EFAIL("sdxe_unet_set_hypertile: not a UNet engine");
  if (n_layers < 0 || n_layers > HT_MAX_LAYERS || (n_layers > 0 && !layers)) EFAIL("sdxe_unet_set_hypertile: bad argument");
  e->unet->ht_rows.assign(layers, layers + 5 * n_layers);
  return 0;
}

int sdxe_set_circular(sdxe_engine* e, int enable) {
  if (!e || (e->cfg.kind != SDXE_MODEL_UNET && e->cfg.kind != SDXE_MODEL_VAE_DECODER && e->cfg.kind != SDXE_MODEL_VAE_ENCODER))
    EFAIL("sdxe_set_circular: not a UNet or VAE engine");
  e->circular = enable != 0;
  return 0;
}

int sdxe_set_plan_cache(sdxe_engine* e, int max_plans, int64_t pool_limit_mb) {
  if (!e || max_plans < 1) EFAIL("sdxe_set_plan_cache: bad argument");
  e->max_plans = max_plans;
  if (pool_limit_mb >= 0) e->pool_limit = (size_t)pool_limit_mb << 20;
  while ((int)e->plans.size() > e->max_plans) evict_lru(e);
  return 0;
}

int64_t sdxe_pool_bytes(sdxe_engine* e, int64_t* n_plans) {
  if (!e) return -1;
  if (n_plans) *n_plans = (int64_t)e->plans.size();
  int64_t total = 0;
  for (auto& kv : e->free_list) total += (int64_t)kv.first;
  for (auto& kv : e->plans)
    for (auto& b : kv.second->owned) total += (int64_t)b.bytes;
  return total;
}

int sdxe_profile(sdxe_engine* e, int enable) {
  if (!e) EFAIL("sdxe_profile: null");
  e->profiling = enable != 0;
  if (enable) {
    for (int k = 0; k < 8; ++k) { e->prof_ms[k] = e->prof_flops[k] = e->prof_bytes[k] = 0; e->prof_launches[k] = 0; }
  }
  return 0;
}

int sdxe_profile_read(sdxe_engine* e, int kind, double* ms, double* flops, double* bytes, int64_t* launches) {
  if (!e || kind < 0 || kind >= K_NUM) EFAIL("sdxe_profile_read: bad argument");
  *ms = e->prof_ms[kind]; *flops = e->prof_flops[kind]; *bytes = e->prof_bytes[kind]; *launches = e->prof_launches[kind];
  return 0;
}

int sdxe_vae_decode(sdxe_engine* e, const void* z, void* out, int n, int h, int w, int io_dtype, void* stream) {
  auto args = [&](std::string&) {
    if (!z || !out || n <= 0 || h <= 0 || w <= 0) EFAIL("sdxe_vae_decode: bad argument");
    return 0;
  };
  return run_forward(e, SDXE_MODEL_VAE_DECODER, "sdxe_vae_decode", "VAE decoder", io_dtype, dims_key('v', {n, h, w}), args,
                     [&](Plan* pl) { return build_vae_plan(e, pl, n, h, w); }, z, out, stream);
}

int sdxe_vae_encode(sdxe_engine* e, const void* x, void* out, int n, int h, int w, int io_dtype, void* stream) {
  auto args = [&](std::string&) {
    const int f = 1 << (e->cfg.num_levels - 1);  // spatial reduction of the encoder (8 for the SD VAE)
    if (!x || !out || n <= 0 || h <= 0 || w <= 0 || (h % f) || (w % f)) EFAIL("sdxe_vae_encode: bad argument (H, W must be multiples of the encoder's downsampling factor)");
    return 0;
  };
  return run_forward(e, SDXE_MODEL_VAE_ENCODER, "sdxe_vae_encode", "VAE encoder", io_dtype, dims_key('e', {n, h, w}), args,
                     [&](Plan* pl) { return build_vae_encode_plan(e, pl, n, h, w); }, x, out, stream);
}

}  // extern "C"
