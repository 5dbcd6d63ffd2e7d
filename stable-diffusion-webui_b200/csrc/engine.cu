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
  bool used = false;
};

// ---- packed weights ------------------------------------------------------------------------------------------
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
struct BlockW {  // one TimestepEmbedSequential
  int kind = 0;  // 0 conv_in, 1 res(+st)(+up), 2 downsample
  ResW res;
  bool has_st = false;
  STW st;
  bool has_up = false;
  LinW up;    // Upsample.conv
  LinW down;  // Downsample.op
  LinW conv_in;
  int ch_out = 0;
};

struct ClipLayerW {  // CLIPEncoderLayer: LN1 -> q|k|v -> causal attention -> out_proj (+x) -> LN2 -> fc1 -> act -> fc2 (+x)
  LinW qkv, out, fc1, fc2;   // layer_norm1 / layer_norm2 are folded into qkv / fc1
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

  // UNet
  LinW te0, te2, le0, le2, emb_all;
  int emb_total = 0;
  // every transformer block's attn2.to_k / to_v stacked along N: the context is projected ONCE per UNet call
  LinW kv_all;
  int kv_total = 0;
  std::vector<std::string> kv_keys;
  std::vector<int> kv_rows;
  std::vector<BlockW> in_blocks, out_blocks;
  ResW mid_r1, mid_r2;
  STW mid_st;
  NormW out_norm;
  LinW out_conv;
  // VAE decoder
  float* pq_w = nullptr;  // post_quant_conv [z, z] fp32
  float* pq_b = nullptr;
  LinW v_conv_in, v_conv_out, v_qkv, v_proj;
  ResW v_mid1, v_mid2;
  NormW v_attn_norm, v_norm_out;
  std::vector<std::vector<ResW>> v_up_blocks;  // [level][block], level index as in the state dict
  // VAE encoder (ldm Encoder: conv_in, down.{l}.block.{j} (+ downsample), mid, norm_out, conv_out; then quant_conv)
  LinW e_conv_in, e_conv_out, e_qkv, e_proj, e_quant;
  ResW e_mid1, e_mid2;
  NormW e_attn_norm, e_norm_out;
  std::vector<std::vector<ResW>> e_down_blocks;
  std::vector<LinW> e_down_conv;
  std::vector<LinW> v_up_conv;                    // per level (level 0 unused)
  // CLIP text transformer
  void* c_tok = nullptr;   // [vocab, C] 16-bit
  void* c_pos = nullptr;   // [positions, C] 16-bit
  std::vector<ClipLayerW> c_layers;
  NormW c_final;

  // activation pool
  std::multimap<size_t, void*> free_list;
  std::vector<void*> all_allocs;
  // Plan cache: one static plan (buffers + tensor maps + CUDA graph) per input shape, least-recently-used eviction.
  // A long-lived webui process sees many shapes (resolutions, batch sizes, 77 / 154 / 231-token prompts, B vs 2B
  // batches under s_min_uncond); every plan pins its own buffers (SDXL: > 100 MB of cross-attention k|v alone), so an
  // unbounded cache grows until cudaMalloc fails.
  std::map<std::string, std::unique_ptr<Plan>> plans;
  // Cross-attention K / V cache: a non-zero key is the caller's promise that the context passed under that key always has
  // the same contents (the conditioning of one job is step-invariant); a plan whose k|v buffer was last filled under the
  // same key skips the context cast + projection GEMM (modules/sd_samplers_cfg_denoiser.py re-sends the same cond_in
  // every sampler step).
  int64_t ctx_key = 0;
  // Hypertile rows (h', w', nh, nw, max_tiles) per attn1 layer for the next sdxe_unet_forward (sdxe_unet_set_hypertile)
  std::vector<int32_t> ht_rows;
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
  int pack_norm(NormW& out, const std::string& prefix, int C);
  int fold_layer_norm(LinW& w, const NormW& ln);  // w consumes LayerNorm(ln) output: fold gamma / beta into w
  int pack_f32(float*& out, const std::string& key, int64_t n);
  int build_unet();
  int build_vae();
  int build_vae_encoder();
  int build_clip();
  int build_res(ResW& r, const std::string& p, int cin, int cout, const ResKeys& k);
  int build_st(STW& s, const std::string& p, int C, int depth);
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

  Builder(sdxe_engine* e_, Plan* p) : e(e_), plan(p), bf16(e_->bf16), ops(&p->body) {}

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
  int conv3(const Act& x, const LinW& W, void* out, int ldo, const GemmOpt& o, int stride = 1, int pad_lo = 1, int Ho = 0,
            int Wo = 0) {
    static int s2_implicit = -1;
    if (s2_implicit < 0) { const char* ev = getenv("SDXE_CONV_S2_IMPLICIT"); s2_implicit = ev ? atoi(ev) : 1; }
    if (stride == 1) { Ho = x.h; Wo = x.w; }
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
      ops->push_back([=](cudaStream_t s) { return im2col3x3_launch(xp, cp, n, H, Wd, C, Ho, Wo, stride, pad_lo, kpad, b, s); });
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
    ECHK(gemm_args(a, GemmA::nhwc(x.p, x.n, x.h, x.w, x.c, stride, pad_lo), weight(W), out, epi));
    const bool b = bf16;
    const double Md = (double)a.M;
    char d[160];
    double by;
    if (stride == 1) {
      by = 2.0 * (Md * x.c + (double)W.N * a.K + Md * W.N + (o.residual ? Md * W.N : 0.0));
      snprintf(d, sizeof(d), "conv3 M=%d N=%d Cin=%d HxW=%dx%d BN=%d st=%d res=%d rv=%d", a.M, W.N, x.c, x.h, x.w, a.BN, a.num_stages,
               o.residual ? 1 : 0, o.rowvec ? 1 : 0);
    } else {
      by = 2.0 * (4.0 * Md * x.c + (double)W.N * a.K + Md * W.N);
      snprintf(d, sizeof(d), "conv3s2 M=%d N=%d Cin=%d HoxWo=%dx%d BN=%d st=%d", a.M, W.N, x.c, Ho, Wo, a.BN, a.num_stages);
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
      const bool b = bf16;
      plan->pre.push_back([=](cudaStream_t s) {
        return im2col3x3_nchw_launch(src ? src : p->x, src ? edt : p->io_dtype, cp, n, c, h, w, kin, b, s);
      });
    }
    out = new_act(n, h, w, W.N);
    LinW Wk = W;
    Wk.K = kin;
    return gemm(col.p, kin, out.rows(), Wk, out.p, GemmOpt());
  }
  // ldm Upsample: nearest 2x, then 3x3 conv; x is released
  int upsample_conv(Act& x, const LinW& W, Act& out) {
    Act up = new_act(x.n, x.h * 2, x.w * 2, x.c);
    {
      const void* xp = x.p;
      void* upp = up.p;
      const int n = x.n, h = x.h, w = x.w, c = x.c;
      ops->push_back([=](cudaStream_t s) { return upsample2x_launch(xp, upp, n, h, w, c, s); });
    }
    free_act(x);
    out = new_act(up.n, up.h, up.w, up.c);
    ECHK(conv3(up, W, out.p, up.c, GemmOpt()));
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
  // emb_all: the UNet's batched timestep-embedding rows (null: none); skip_src: the UNet decoder's skip-concat input.
  int res_block(const ResW& r, Act& x, Act* skip_src, const float* emb_all, int ld_emb, float eps, Act& out) {
    Act g1;
    ECHK(group_norm(x, skip_src, r.n1, eps, true, g1));
    Act h = new_act(x.n, x.h, x.w, r.cout);
    GemmOpt o1;
    if (emb_all) { o1.rowvec = emb_all + r.emb_off; o1.ldrv = ld_emb; o1.rows_per_sample = x.h * x.w; }
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

  // SpatialTransformer (modules/sd_hijack_unet.py:83-102) with BasicTransformerBlocks
  // kv_all: [B * ctx_len, ld_kv] = every block's cross-attention k | v projection of the context (one GEMM per call)
  int spatial_transformer(const STW& st, Act& x, const void* kv_all, int ld_kv, int ctx_len, Act& out) {
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
    out = new_act(x.n, x.h, x.w, C);
    GemmOpt op;
    op.residual = x.p; op.ldr = C;
    ECHK(gemm(h.p, C, M, st.proj_out, out.p, op));
    free_act(h);
    return 0;
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
  it->second.used = true;
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

int sdxe_engine::build_res(ResW& r, const std::string& p, int cin, int cout, const ResKeys& k) {
  r.cin = cin; r.cout = cout;
  const std::string c1 = p + k.c1, c2 = p + k.c2, sk = p + k.skip;
  ECHK(pack_norm(r.n1, p + k.n1, cin));
  ECHK(pack_linear(r.c1, {c1 + ".weight"}, {c1 + ".bias"}, cout, 9 * cin, PACK_CONV3, conv_kpad(cin)));
  ECHK(pack_norm(r.n2, p + k.n2, cout));
  ECHK(pack_linear(r.c2, {c2 + ".weight"}, {c2 + ".bias"}, cout, 9 * cout, PACK_CONV3, conv_kpad(cout)));
  r.has_skip = cin != cout;
  if (r.has_skip) ECHK(pack_linear(r.skip, {sk + ".weight"}, {sk + ".bias"}, cout, cin, PACK_PLAIN));
  return 0;
}

int sdxe_engine::build_st(STW& s, const std::string& p, int C, int depth) {
  s.C = C;
  if (cfg.num_head_channels > 0) { s.dh = cfg.num_head_channels; s.heads = C / s.dh; }
  else { s.heads = cfg.num_heads; s.dh = C / s.heads; }
  if (s.dh % 8) EFAIL("head dim must be a multiple of 8");
  const int ctx = cfg.context_dim;
  ECHK(pack_norm(s.gn, p + ".norm", C));
  ECHK(pack_linear(s.proj_in, {p + ".proj_in.weight"}, {p + ".proj_in.bias"}, C, C, PACK_PLAIN));
  ECHK(pack_linear(s.proj_out, {p + ".proj_out.weight"}, {p + ".proj_out.bias"}, C, C, PACK_PLAIN));
  s.blocks.resize(depth);
  for (int j = 0; j < depth; ++j) {
    TBlockW& t = s.blocks[j];
    const std::string b = p + ".transformer_blocks." + std::to_string(j);
    ECHK(pack_norm(t.ln1, b + ".norm1", C));
    ECHK(pack_norm(t.ln2, b + ".norm2", C));
    ECHK(pack_norm(t.ln3, b + ".norm3", C));
    ECHK(pack_linear(t.qkv1, {b + ".attn1.to_q.weight", b + ".attn1.to_k.weight", b + ".attn1.to_v.weight"}, {}, C, C, PACK_PLAIN));
    ECHK(pack_linear(t.out1, {b + ".attn1.to_out.0.weight"}, {b + ".attn1.to_out.0.bias"}, C, C, PACK_PLAIN));
    ECHK(pack_linear(t.q2, {b + ".attn2.to_q.weight"}, {}, C, C, PACK_PLAIN));
    t.kv_off = kv_total;  // packed after all blocks are known (build_unet)
    kv_keys.push_back(b + ".attn2.to_k.weight"); kv_rows.push_back(C);
    kv_keys.push_back(b + ".attn2.to_v.weight"); kv_rows.push_back(C);
    kv_total += 2 * C;
    ECHK(pack_linear(t.out2, {b + ".attn2.to_out.0.weight"}, {b + ".attn2.to_out.0.bias"}, C, C, PACK_PLAIN));
    const int n1 = 8 * C;
    const int tile = n1 % 256 == 0 ? 256 : (n1 % 128 == 0 ? 128 : 64);
    ECHK(pack_linear(t.ff1, {b + ".ff.net.0.proj.weight"}, {b + ".ff.net.0.proj.bias"}, n1, C, PACK_GEGLU, 0, tile));
    ECHK(pack_linear(t.ff2, {b + ".ff.net.2.weight"}, {b + ".ff.net.2.bias"}, C, 4 * C, PACK_PLAIN));
    // norm1 / norm2 / norm3 are folded into the GEMMs that consume them (no LayerNorm kernel runs)
    ECHK(fold_layer_norm(t.qkv1, t.ln1));
    ECHK(fold_layer_norm(t.q2, t.ln2));
    ECHK(fold_layer_norm(t.ff1, t.ln3));
  }
  return 0;
}

int sdxe_engine::build_unet() {
  const int mc = cfg.model_channels, ted = 4 * mc, nl = cfg.num_levels, nrb = cfg.num_res_blocks;
  ECHK(pack_linear(te0, {"time_embed.0.weight"}, {"time_embed.0.bias"}, ted, mc, PACK_PLAIN));
  ECHK(pack_linear(te2, {"time_embed.2.weight"}, {"time_embed.2.bias"}, ted, ted, PACK_PLAIN));
  if (cfg.adm_in_channels > 0) {
    ECHK(pack_linear(le0, {"label_emb.0.0.weight"}, {"label_emb.0.0.bias"}, ted, cfg.adm_in_channels, PACK_PLAIN));
    ECHK(pack_linear(le2, {"label_emb.0.2.weight"}, {"label_emb.0.2.bias"}, ted, ted, PACK_PLAIN));
  }
  in_blocks.clear(); out_blocks.clear();
  kv_keys.clear(); kv_rows.clear(); kv_total = 0;
  std::vector<std::string> emb_w, emb_b;  // batched emb_layers (every ResBlock's Linear(SiLU(emb)) in one skinny GEMM)
  std::vector<int> emb_n;
  int emb_cursor = 0;
  auto add_emb = [&](ResW& r, const std::string& p) {
    r.emb_off = emb_cursor;
    emb_cursor += r.cout;
    emb_w.push_back(p + ".emb_layers.1.weight");
    emb_b.push_back(p + ".emb_layers.1.bias");
    emb_n.push_back(r.cout);
  };
  {
    BlockW b0;
    b0.kind = 0;
    ECHK(pack_linear(b0.conv_in, {"input_blocks.0.0.weight"}, {"input_blocks.0.0.bias"}, mc, 9 * cfg.in_channels, PACK_CONV3,
                     conv_kpad(cfg.in_channels)));
    b0.ch_out = mc;
    in_blocks.push_back(b0);
  }
  std::vector<int> chans = {mc};
  int ch = mc, idx = 1;
  for (int level = 0; level < nl; ++level) {
    const int mult = cfg.channel_mult[level];
    for (int r = 0; r < nrb; ++r) {
      BlockW b;
      b.kind = 1;
      const std::string p = "input_blocks." + std::to_string(idx);
      ECHK(build_res(b.res, p + ".0", ch, mult * mc, UNET_RES));
      add_emb(b.res, p + ".0");
      ch = mult * mc;
      if (cfg.transformer_depth[level] > 0) {
        b.has_st = true;
        ECHK(build_st(b.st, p + ".1", ch, cfg.transformer_depth[level]));
      }
      b.ch_out = ch;
      in_blocks.push_back(b);
      chans.push_back(ch);
      ++idx;
    }
    if (level != nl - 1) {
      BlockW b;
      b.kind = 2;
      const std::string p = "input_blocks." + std::to_string(idx) + ".0.op";
      ECHK(pack_linear(b.down, {p + ".weight"}, {p + ".bias"}, ch, 9 * ch, PACK_CONV3, conv_kpad(ch)));
      b.ch_out = ch;
      in_blocks.push_back(b);
      chans.push_back(ch);
      ++idx;
    }
  }
  ECHK(build_res(mid_r1, "middle_block.0", ch, ch, UNET_RES));
  add_emb(mid_r1, "middle_block.0");
  ECHK(build_st(mid_st, "middle_block.1", ch, std::max(1, cfg.transformer_depth_middle)));
  ECHK(build_res(mid_r2, "middle_block.2", ch, ch, UNET_RES));
  add_emb(mid_r2, "middle_block.2");
  idx = 0;
  for (int level = nl - 1; level >= 0; --level) {
    const int mult = cfg.channel_mult[level];
    for (int i = 0; i <= nrb; ++i) {
      const int ich = chans.back();
      chans.pop_back();
      BlockW b;
      b.kind = 1;
      const std::string p = "output_blocks." + std::to_string(idx);
      ECHK(build_res(b.res, p + ".0", ch + ich, mc * mult, UNET_RES));
      add_emb(b.res, p + ".0");
      ch = mc * mult;
      int sub = 1;
      if (cfg.transformer_depth[level] > 0) {
        b.has_st = true;
        ECHK(build_st(b.st, p + ".1", ch, cfg.transformer_depth[level]));
        sub = 2;
      }
      if (level && i == nrb) {
        b.has_up = true;
        const std::string u = p + "." + std::to_string(sub) + ".conv";
        ECHK(pack_linear(b.up, {u + ".weight"}, {u + ".bias"}, ch, 9 * ch, PACK_CONV3, conv_kpad(ch)));
      }
      b.ch_out = ch;
      out_blocks.push_back(b);
      ++idx;
    }
  }
  ECHK(pack_norm(out_norm, "out.0", ch));
  ECHK(pack_linear(out_conv, {"out.2.weight"}, {"out.2.bias"}, cfg.out_channels, 9 * ch, PACK_CONV3, conv_kpad(ch)));
  // batched emb_layers: rows of different widths -> pack key by key
  emb_total = emb_cursor;
  emb_all.N = emb_total; emb_all.K = ted; emb_all.ld = ted;
  emb_all.w = alloc16((size_t)emb_total * ted);
  emb_all.b = alloc32(align_up((size_t)emb_total, 8));
  int off = 0;
  for (size_t i = 0; i < emb_w.size(); ++i) {
    const RawWeight* w = find(emb_w[i], (int64_t)emb_n[i] * ted);
    const RawWeight* b = find(emb_b[i], emb_n[i]);
    if (!sizing && w && b) {
      ECHK(pack_weight_launch(w->dev, w->dtype, (char*)emb_all.w + (size_t)off * ted * 2, PACK_PLAIN, emb_n[i], ted, ted, 0, bf16, 0));
      ECHK(pack_vector_launch(b->dev, b->dtype, emb_all.b + off, emb_n[i], 0, true, bf16, 0));
    }
    off += emb_n[i];
  }
  // batched cross-attention K/V projection weights [kv_total, context_dim]
  {
    const int ctx = cfg.context_dim;
    kv_all.N = kv_total; kv_all.K = ctx; kv_all.ld = ctx; kv_all.b = nullptr;
    kv_all.Nrows = (int)align_up((size_t)kv_total, 16);
    kv_all.w = alloc16((size_t)kv_all.Nrows * ctx);
    int row = 0;
    for (size_t i = 0; i < kv_keys.size(); ++i) {
      const RawWeight* w = find(kv_keys[i], (int64_t)kv_rows[i] * ctx);
      if (!sizing && w)
        ECHK(pack_weight_launch(w->dev, w->dtype, (char*)kv_all.w + (size_t)row * ctx * 2, PACK_PLAIN, kv_rows[i], ctx, ctx, 0, bf16, 0));
      row += kv_rows[i];
    }
  }
  return 0;
}

int sdxe_engine::build_vae() {
  const int z = cfg.vae_z_channels, nl = cfg.num_levels, nrb = cfg.num_res_blocks;
  ECHK(pack_f32(pq_w, "post_quant_conv.weight", (int64_t)z * z));
  ECHK(pack_f32(pq_b, "post_quant_conv.bias", z));
  int bi = cfg.vae_ch * cfg.channel_mult[nl - 1];
  ECHK(pack_linear(v_conv_in, {"decoder.conv_in.weight"}, {"decoder.conv_in.bias"}, bi, 9 * z, PACK_CONV3, conv_kpad(z)));
  ECHK(build_res(v_mid1, "decoder.mid.block_1", bi, bi, VAE_RES));
  ECHK(pack_norm(v_attn_norm, "decoder.mid.attn_1.norm", bi));
  ECHK(pack_linear(v_qkv, {"decoder.mid.attn_1.q.weight", "decoder.mid.attn_1.k.weight", "decoder.mid.attn_1.v.weight"},
                   {"decoder.mid.attn_1.q.bias", "decoder.mid.attn_1.k.bias", "decoder.mid.attn_1.v.bias"}, bi, bi, PACK_PLAIN));
  ECHK(pack_linear(v_proj, {"decoder.mid.attn_1.proj_out.weight"}, {"decoder.mid.attn_1.proj_out.bias"}, bi, bi, PACK_PLAIN));
  ECHK(build_res(v_mid2, "decoder.mid.block_2", bi, bi, VAE_RES));
  v_up_blocks.assign(nl, {});
  v_up_conv.assign(nl, LinW());
  for (int level = nl - 1; level >= 0; --level) {
    const int bo = cfg.vae_ch * cfg.channel_mult[level];
    for (int j = 0; j <= nrb; ++j) {
      ResW r;
      ECHK(build_res(r, "decoder.up." + std::to_string(level) + ".block." + std::to_string(j), bi, bo, VAE_RES));
      v_up_blocks[level].push_back(r);
      bi = bo;
    }
    if (level != 0) {
      const std::string u = "decoder.up." + std::to_string(level) + ".upsample.conv";
      ECHK(pack_linear(v_up_conv[level], {u + ".weight"}, {u + ".bias"}, bi, 9 * bi, PACK_CONV3, conv_kpad(bi)));
    }
  }
  ECHK(pack_norm(v_norm_out, "decoder.norm_out", bi));
  ECHK(pack_linear(v_conv_out, {"decoder.conv_out.weight"}, {"decoder.conv_out.bias"}, cfg.vae_out_ch, 9 * bi, PACK_CONV3, conv_kpad(bi)));
  return 0;
}

int sdxe_engine::build_vae_encoder() {
  const int z = cfg.vae_z_channels, nl = cfg.num_levels, nrb = cfg.num_res_blocks, ch = cfg.vae_ch, cin = cfg.vae_out_ch;
  ECHK(pack_linear(e_conv_in, {"encoder.conv_in.weight"}, {"encoder.conv_in.bias"}, ch, 9 * cin, PACK_CONV3, conv_kpad(cin)));
  e_down_blocks.assign(nl, {});
  e_down_conv.assign(nl, LinW());
  int bi = ch;
  for (int level = 0; level < nl; ++level) {
    const int bo = ch * cfg.channel_mult[level];
    for (int j = 0; j < nrb; ++j) {
      ResW r;
      ECHK(build_res(r, "encoder.down." + std::to_string(level) + ".block." + std::to_string(j), bi, bo, VAE_RES));
      e_down_blocks[level].push_back(r);
      bi = bo;
    }
    if (level != nl - 1) {
      const std::string d = "encoder.down." + std::to_string(level) + ".downsample.conv";
      ECHK(pack_linear(e_down_conv[level], {d + ".weight"}, {d + ".bias"}, bi, 9 * bi, PACK_CONV3, conv_kpad(bi)));
    }
  }
  ECHK(build_res(e_mid1, "encoder.mid.block_1", bi, bi, VAE_RES));
  ECHK(pack_norm(e_attn_norm, "encoder.mid.attn_1.norm", bi));
  ECHK(pack_linear(e_qkv, {"encoder.mid.attn_1.q.weight", "encoder.mid.attn_1.k.weight", "encoder.mid.attn_1.v.weight"},
                   {"encoder.mid.attn_1.q.bias", "encoder.mid.attn_1.k.bias", "encoder.mid.attn_1.v.bias"}, bi, bi, PACK_PLAIN));
  ECHK(pack_linear(e_proj, {"encoder.mid.attn_1.proj_out.weight"}, {"encoder.mid.attn_1.proj_out.bias"}, bi, bi, PACK_PLAIN));
  ECHK(build_res(e_mid2, "encoder.mid.block_2", bi, bi, VAE_RES));
  ECHK(pack_norm(e_norm_out, "encoder.norm_out", bi));
  ECHK(pack_linear(e_conv_out, {"encoder.conv_out.weight"}, {"encoder.conv_out.bias"}, 2 * z, 9 * bi, PACK_CONV3, conv_kpad(bi)));
  ECHK(pack_linear(e_quant, {"quant_conv.weight"}, {"quant_conv.bias"}, 2 * z, 2 * z, PACK_PLAIN));
  return 0;
}

// =================================================================================================================
// CLIP text transformer weights (Hugging Face CLIPTextModel names; open_clip towers are renamed on the host)
// =================================================================================================================
int sdxe_engine::build_clip() {
  const int C = cfg.clip_hidden, I = cfg.clip_intermediate, L = cfg.clip_layers;
  const std::string tm = "text_model.";
  c_tok = alloc16((size_t)cfg.clip_vocab * C);
  c_pos = alloc16((size_t)cfg.clip_positions * C);
  const RawWeight* wt = find(tm + "embeddings.token_embedding.weight", (int64_t)cfg.clip_vocab * C);
  const RawWeight* wp = find(tm + "embeddings.position_embedding.weight", (int64_t)cfg.clip_positions * C);
  if (!sizing && wt) ECHK(pack_weight_launch(wt->dev, wt->dtype, c_tok, PACK_PLAIN, cfg.clip_vocab, C, C, 0, bf16, 0));
  if (!sizing && wp) ECHK(pack_weight_launch(wp->dev, wp->dtype, c_pos, PACK_PLAIN, cfg.clip_positions, C, C, 0, bf16, 0));
  c_layers.resize(L);
  for (int l = 0; l < L; ++l) {
    ClipLayerW& w = c_layers[l];
    const std::string p = tm + "encoder.layers." + std::to_string(l) + ".";
    NormW ln1, ln2;
    ECHK(pack_norm(ln1, p + "layer_norm1", C));
    ECHK(pack_norm(ln2, p + "layer_norm2", C));
    ECHK(pack_linear(w.qkv, {p + "self_attn.q_proj.weight", p + "self_attn.k_proj.weight", p + "self_attn.v_proj.weight"},
                     {p + "self_attn.q_proj.bias", p + "self_attn.k_proj.bias", p + "self_attn.v_proj.bias"}, C, C, PACK_PLAIN));
    ECHK(pack_linear(w.out, {p + "self_attn.out_proj.weight"}, {p + "self_attn.out_proj.bias"}, C, C, PACK_PLAIN));
    ECHK(pack_linear(w.fc1, {p + "mlp.fc1.weight"}, {p + "mlp.fc1.bias"}, I, C, PACK_PLAIN));
    ECHK(pack_linear(w.fc2, {p + "mlp.fc2.weight"}, {p + "mlp.fc2.bias"}, C, I, PACK_PLAIN));
    ECHK(fold_layer_norm(w.qkv, ln1));
    ECHK(fold_layer_norm(w.fc1, ln2));
  }
  ECHK(pack_norm(c_final, tm + "final_layer_norm", C));
  return 0;
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
  Buf emb_all = e->alloc(sizeof(float) * n * e->emb_total);
  {
    const LinW te0 = e->te0, te2 = e->te2, le0 = e->le0, le2 = e->le2, ea = e->emb_all;
    float *pt = (float*)temb.p, *p1 = (float*)e1.p, *pe = (float*)emb.p, *pl = (float*)l1.p, *pa = (float*)emb_all.p, *py = (float*)y32.p;
    const int adm = cfg.adm_in_channels, etot = e->emb_total;
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
  const float* emb_ptr = (const float*)emb_all.p;
  const int ld_emb = e->emb_total;
  // ---- cross-attention keys / values of ALL transformer blocks: one GEMM over the context (plan-owned buffer)
  Buf kvbuf = e->alloc((size_t)n * ctx_len * std::max(8, e->kv_total) * 2);
  {
    // runs before the graph, and only when the context changed (ctx_key): cast the caller's context, project it once
    auto kv_ops = std::make_shared<std::vector<OpRec>>();
    if (e->kv_total > 0) {
      B.ops = kv_ops.get();
      const int rc = B.gemm(ctx16.p, cfg.context_dim, (int64_t)n * ctx_len, e->kv_all, kvbuf.p, Builder::GemmOpt());
      B.ops = &p->body;
      ECHK(rc);
    }
    void* cx = ctx16.p;
    const int cdim = cfg.context_dim;
    p->pre.push_back([=](cudaStream_t s) {
      if (e->ctx_key != 0 && p->kv_key == e->ctx_key && !e->profiling) return 0;
      ECHK(cast_rows_launch(p->ctx, p->io_dtype, cx, (int64_t)n * ctx_len, cdim, cdim, bf16, s));
      if (e->profiling) ECHK(run_ops_profiled(e, *kv_ops, s));
      else ECHK(run_ops(*kv_ops, s));
      p->kv_key = e->ctx_key;
      return 0;
    });
  }

  // ---- input blocks
  std::vector<Act> hs;
  Act cur;
  for (size_t bi = 0; bi < e->in_blocks.size(); ++bi) {
    const BlockW& b = e->in_blocks[bi];
    if (b.kind == 0) {
      ECHK(B.conv_in_nchw(nullptr, n, cfg.in_channels, h, w, b.conv_in, cur));
    } else if (b.kind == 1) {
      Act r;
      ECHK(B.res_block(b.res, cur, nullptr, emb_ptr, ld_emb, 1e-5f, r));
      // `cur` stays alive: it is on the skip stack
      if (b.has_st) {
        Act t;
        ECHK(B.spatial_transformer(b.st, r, kvbuf.p, e->kv_total, ctx_len, t));
        B.free_act(r);
        r = t;
      }
      cur = r;
    } else {
      const int Ho = (cur.h + 2 - 3) / 2 + 1, Wo = (cur.w + 2 - 3) / 2 + 1;
      Act d = B.new_act(n, Ho, Wo, b.ch_out);
      ECHK(B.conv3(cur, b.down, d.p, b.ch_out, Builder::GemmOpt(), 2, 1, Ho, Wo));
      cur = d;
    }
    hs.push_back(cur);
  }
  // ---- middle
  {
    Act r1, t, r2;
    ECHK(B.res_block(e->mid_r1, cur, nullptr, emb_ptr, ld_emb, 1e-5f, r1));
    ECHK(B.spatial_transformer(e->mid_st, r1, kvbuf.p, e->kv_total, ctx_len, t));
    B.free_act(r1);
    ECHK(B.res_block(e->mid_r2, t, nullptr, emb_ptr, ld_emb, 1e-5f, r2));
    B.free_act(t);
    cur = r2;  // note: hs.back() (same tensor as the old cur) is still owned by the skip stack
  }
  // ---- output blocks
  bool cur_owned = true;
  for (size_t bi = 0; bi < e->out_blocks.size(); ++bi) {
    const BlockW& b = e->out_blocks[bi];
    Act skip = hs.back();
    hs.pop_back();
    if (skip.h != cur.h || skip.w != cur.w) EFAIL("unet: skip / hidden size mismatch (latent size must be divisible by 2^(levels-1))");
    Act r;
    ECHK(B.res_block(b.res, cur, &skip, emb_ptr, ld_emb, 1e-5f, r));
    if (cur_owned) B.free_act(cur);
    B.free_act(skip);
    if (b.has_st) {
      Act t;
      ECHK(B.spatial_transformer(b.st, r, kvbuf.p, e->kv_total, ctx_len, t));
      B.free_act(r);
      r = t;
    }
    if (b.has_up) {
      Act c;
      ECHK(B.upsample_conv(r, b.up, c));
      r = c;
    }
    cur = r;
    cur_owned = true;
  }
  // ---- out: GN + SiLU + conv3 -> [M, 8] (4 valid channels)
  ECHK(B.out_head(cur, e->out_norm, 1e-5f, e->out_conv));
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

// AttnBlock (sd_hijack_optimizations.py:637-655): GN -> fused q|k|v 1x1 conv -> single-head attention -> proj + x
int vae_attn_block(sdxe_engine* e, Builder& B, Act& cur, const NormW& norm, const LinW& qkv_w, const LinW& proj_w) {
  const int C = cur.c, tokens = cur.h * cur.w, n = cur.n;
  const int64_t M = cur.rows();
  Act xn;
  ECHK(B.group_norm(cur, nullptr, norm, 1e-6f, false, xn));
  Buf qkv = e->alloc((size_t)M * 3 * C * 2);
  ECHK(B.gemm(xn.p, C, M, qkv_w, qkv.p, Builder::GemmOpt()));
  B.free_act(xn);
  if (C % 64 != 0 || C > 512) EFAIL("vae attention: channel count must be a multiple of 64 and <= 512");
  Act att = B.new_act(n, cur.h, cur.w, C);
  const uint16_t* qp = (const uint16_t*)qkv.p;
  ECHK(B.attention(qp, qp + C, qp + 2 * C, n, 1, tokens, tokens, C, 3 * C, 3 * C, 1.0f / sqrtf((float)C), att.p, C, C));
  e->release(qkv);
  Act o = B.new_act(n, cur.h, cur.w, C);
  Builder::GemmOpt op;
  op.residual = cur.p; op.ldr = C;
  ECHK(B.gemm(att.p, C, M, proj_w, o.p, op));
  B.free_act(att);
  B.free_act(cur);
  cur = o;
  return 0;
}

// AutoencoderKL.encode up to the moments: x [n, 3, H, W] -> [n, 2z, H/8, W/8]
int build_vae_encode_plan(sdxe_engine* e, Plan* p, int n, int H, int W) {
  const sdxe_config& cfg = e->cfg;
  Builder B(e, p);
  const bool bf16 = e->bf16;
  const int nl = cfg.num_levels, cin = cfg.vae_out_ch, z2 = 2 * cfg.vae_z_channels;
  Act cur;
  ECHK(B.conv_in_nchw(nullptr, n, cin, H, W, e->e_conv_in, cur));
  Act t;
  for (int level = 0; level < nl; ++level) {
    for (const ResW& r : e->e_down_blocks[level]) {
      ECHK(B.res_block(r, cur, nullptr, nullptr, 0, 1e-6f, t));
      B.free_act(cur);
      cur = t;
    }
    if (level != nl - 1) {
      // ldm Downsample (with_conv): pad (0,1,0,1) then conv3x3 stride 2, padding 0 -> taps start at the pixel itself
      const int Ho = cur.h / 2, Wo = cur.w / 2;
      Act d = B.new_act(n, Ho, Wo, cur.c);
      ECHK(B.conv3(cur, e->e_down_conv[level], d.p, cur.c, Builder::GemmOpt(), 2, 0, Ho, Wo));
      B.free_act(cur);
      cur = d;
    }
  }
  ECHK(B.res_block(e->e_mid1, cur, nullptr, nullptr, 0, 1e-6f, t));
  B.free_act(cur);
  cur = t;
  ECHK(vae_attn_block(e, B, cur, e->e_attn_norm, e->e_qkv, e->e_proj));
  ECHK(B.res_block(e->e_mid2, cur, nullptr, nullptr, 0, 1e-6f, t));
  B.free_act(cur);
  cur = t;
  Act g;
  ECHK(B.group_norm(cur, nullptr, e->e_norm_out, 1e-6f, true, g));
  const int Ho = cur.h, Wo = cur.w;
  B.free_act(cur);
  const int ld8 = (int)align_up(z2, 8);
  Act mo = B.new_act(n, Ho, Wo, ld8);
  ECHK(B.conv3(g, e->e_conv_out, mo.p, ld8, Builder::GemmOpt()));
  B.free_act(g);
  Buf outb = e->alloc((size_t)n * Ho * Wo * ld8 * 2);
  ECHK(B.gemm(mo.p, ld8, (int64_t)n * Ho * Wo, e->e_quant, outb.p, Builder::GemmOpt()));  // quant_conv (1x1)
  B.free_act(mo);
  {
    void* ob = outb.p;
    const int hw = Ho * Wo;
    p->post.push_back([=](cudaStream_t s) { return nhwc_to_nchw_launch(ob, ld8, p->out, p->io_dtype, n, z2, hw, bf16, s); });
  }
  return 0;
}

int build_vae_plan(sdxe_engine* e, Plan* p, int n, int h, int w) {
  const sdxe_config& cfg = e->cfg;
  Builder B(e, p);
  const bool bf16 = e->bf16;
  const int z = cfg.vae_z_channels, nl = cfg.num_levels;
  Buf zq = e->alloc((size_t)n * h * w * z * 2);
  {
    void* zp = zq.p;
    const float *pw = e->pq_w, *pb = e->pq_b;
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
  ECHK(B.conv_in_nchw(zq.p, n, z, h, w, e->v_conv_in, cur));
  Act t;
  ECHK(B.res_block(e->v_mid1, cur, nullptr, nullptr, 0, 1e-6f, t));
  B.free_act(cur);
  cur = t;
  ECHK(vae_attn_block(e, B, cur, e->v_attn_norm, e->v_qkv, e->v_proj));
  ECHK(B.res_block(e->v_mid2, cur, nullptr, nullptr, 0, 1e-6f, t));
  B.free_act(cur);
  cur = t;
  for (int level = nl - 1; level >= 0; --level) {
    for (const ResW& r : e->v_up_blocks[level]) {
      ECHK(B.res_block(r, cur, nullptr, nullptr, 0, 1e-6f, t));
      B.free_act(cur);
      cur = t;
    }
    if (level != 0) {
      ECHK(B.upsample_conv(cur, e->v_up_conv[level], t));
      cur = t;
    }
  }
  return B.out_head(cur, e->v_norm_out, 1e-6f, e->v_conv_out);
}

}  // namespace

// =================================================================================================================
// C-ABI
// =================================================================================================================
namespace {

// hidden_states[layer] (optionally + final_layer_norm) of the text transformer for n sequences of T tokens
int build_clip_plan(sdxe_engine* e, Plan* plan, int n, int T, int layer, int final_norm) {
  const sdxe_config& cfg = e->cfg;
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
    const void *tok = e->c_tok, *pos = e->c_pos;
    const int vocab = cfg.clip_vocab;
    plan->pre.push_back([=](cudaStream_t s) {
      ECHK(clip_embed_launch((const int32_t*)plan->x, tok, pos, xp, sp, (int)M, T, C, vocab, b, s));
      return clip_fix_launch(plan->fix_rows, plan->fix_vecs, pos, xp, sp, plan->n_fix, (int)M, T, C, b, s);
    });
  }
  const float scale = 1.0f / sqrtf((float)d);
  for (int l = 0; l < layer; ++l) {
    const ClipLayerW& w = e->c_layers[l];
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
    const float *g = e->c_final.g, *bt = e->c_final.b;
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

}  // namespace

namespace {

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

}  // namespace

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
    int rc = e->cfg.kind == SDXE_MODEL_UNET ? e->build_unet()
             : (e->cfg.kind == SDXE_MODEL_VAE_ENCODER ? e->build_vae_encoder() : (e->cfg.kind == SDXE_MODEL_CLIP_TEXT ? e->build_clip() : e->build_vae()));
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
  if (!e || !e->finalized || e->cfg.kind != SDXE_MODEL_UNET) EFAIL("sdxe_unet_forward: engine is not a finalized UNet");
  if (!x || !t || !ctx || !out || n <= 0 || h <= 0 || w <= 0 || ctx_len <= 0) EFAIL("sdxe_unet_forward: bad argument");
  if (io_dtype != SDXE_F16 && io_dtype != SDXE_BF16 && io_dtype != SDXE_F32) EFAIL("sdxe_unet_forward: io dtype");
  std::string key = "u:" + std::to_string(n) + ":" + std::to_string(h) + ":" + std::to_string(w) + ":" + std::to_string(ctx_len);
  std::vector<int32_t> ht;
  ht.swap(e->ht_rows);  // a Hypertile table applies to one call
  HtDraws draws;
  if (!ht.empty()) {
    // the plan is keyed on the structural part (h', w', max_tiles per layer); the draws (nh, nw) are data
    int n_attn1 = (int)e->mid_st.blocks.size();
    for (const auto* blocks : {&e->in_blocks, &e->out_blocks})
      for (const BlockW& b : *blocks)
        if (b.has_st) n_attn1 += (int)b.st.blocks.size();
    draws.n = (int)ht.size() / 5;
    if (draws.n != n_attn1) EFAIL("sdxe_unet_forward: the Hypertile table needs one row per attn1 layer");
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
  }
  Plan* p = get_plan(e, key, [&](Plan* pl) { return build_unet_plan(e, pl, n, h, w, ctx_len, ht.empty() ? nullptr : &ht); });
  if (!p) return -1;
  if (!ht.empty()) p->ht_draws = draws;
  p->x = x; p->t = t; p->ctx = ctx; p->y = y; p->out = out; p->io_dtype = io_dtype;
  return run_plan(e, p, (cudaStream_t)stream);
}

int sdxe_clip_forward(sdxe_engine* e, const int32_t* tokens, void* out, int n, int T, int layer, int final_norm, int io_dtype,
                      void* stream) {
  return sdxe_clip_forward_fixes(e, tokens, out, n, T, layer, final_norm, io_dtype, nullptr, nullptr, 0, stream);
}

int sdxe_clip_forward_fixes(sdxe_engine* e, const int32_t* tokens, void* out, int n, int T, int layer, int final_norm, int io_dtype,
                            const int32_t* fix_rows, const void* fix_vecs, int n_fix, void* stream) {
  if (!e || !e->finalized || e->cfg.kind != SDXE_MODEL_CLIP_TEXT) EFAIL("sdxe_clip_forward: engine is not a finalized CLIP text model");
  if (!tokens || !out || n <= 0 || T <= 0 || T > e->cfg.clip_positions || layer < 0 || layer > e->cfg.clip_layers) EFAIL("sdxe_clip_forward: bad argument");
  if (io_dtype != e->dt && io_dtype != SDXE_F32) EFAIL("sdxe_clip_forward: out must be the engine's 16-bit type or fp32");
  const std::string key = "c:" + std::to_string(n) + ":" + std::to_string(T) + ":" + std::to_string(layer) + ":" + std::to_string(final_norm ? 1 : 0);
  Plan* p = get_plan(e, key, [&](Plan* pl) { return build_clip_plan(e, pl, n, T, layer, final_norm ? 1 : 0); });
  if (!p) return -1;
  if (n_fix < 0 || (n_fix > 0 && (!fix_rows || !fix_vecs))) EFAIL("sdxe_clip_forward_fixes: bad fix arguments");
  p->x = tokens; p->out = out; p->io_dtype = io_dtype;
  p->fix_rows = fix_rows; p->fix_vecs = fix_vecs; p->n_fix = n_fix;
  return run_plan(e, p, (cudaStream_t)stream);
}

int sdxe_unet_set_context_key(sdxe_engine* e, int64_t key) {
  if (!e || e->cfg.kind != SDXE_MODEL_UNET) EFAIL("sdxe_unet_set_context_key: not a UNet engine");
  e->ctx_key = key;
  return 0;
}

int sdxe_unet_set_hypertile(sdxe_engine* e, const int32_t* layers, int n_layers) {
  if (!e || e->cfg.kind != SDXE_MODEL_UNET) EFAIL("sdxe_unet_set_hypertile: not a UNet engine");
  if (n_layers < 0 || n_layers > HT_MAX_LAYERS || (n_layers > 0 && !layers)) EFAIL("sdxe_unet_set_hypertile: bad argument");
  e->ht_rows.assign(layers, layers + 5 * n_layers);
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
  if (!e || !e->finalized || e->cfg.kind != SDXE_MODEL_VAE_DECODER) EFAIL("sdxe_vae_decode: engine is not a finalized VAE decoder");
  if (!z || !out || n <= 0 || h <= 0 || w <= 0) EFAIL("sdxe_vae_decode: bad argument");
  if (io_dtype != SDXE_F16 && io_dtype != SDXE_BF16 && io_dtype != SDXE_F32) EFAIL("sdxe_vae_decode: io dtype");
  const std::string key = "v:" + std::to_string(n) + ":" + std::to_string(h) + ":" + std::to_string(w);
  Plan* p = get_plan(e, key, [&](Plan* pl) { return build_vae_plan(e, pl, n, h, w); });
  if (!p) return -1;
  p->x = z; p->out = out; p->io_dtype = io_dtype;
  return run_plan(e, p, (cudaStream_t)stream);
}

int sdxe_vae_encode(sdxe_engine* e, const void* x, void* out, int n, int h, int w, int io_dtype, void* stream) {
  if (!e || !e->finalized || e->cfg.kind != SDXE_MODEL_VAE_ENCODER) EFAIL("sdxe_vae_encode: engine is not a finalized VAE encoder");
  const int f = 1 << (e->cfg.num_levels - 1);  // spatial reduction of the encoder (8 for the SD VAE)
  if (!x || !out || n <= 0 || h <= 0 || w <= 0 || (h % f) || (w % f)) EFAIL("sdxe_vae_encode: bad argument (H, W must be multiples of the encoder's downsampling factor)");
  if (io_dtype != SDXE_F16 && io_dtype != SDXE_BF16 && io_dtype != SDXE_F32) EFAIL("sdxe_vae_encode: io dtype");
  const std::string key = "e:" + std::to_string(n) + ":" + std::to_string(h) + ":" + std::to_string(w);
  Plan* p = get_plan(e, key, [&](Plan* pl) { return build_vae_encode_plan(e, pl, n, h, w); });
  if (!p) return -1;
  p->x = x; p->out = out; p->io_dtype = io_dtype;
  return run_plan(e, p, (cudaStream_t)stream);
}

}  // extern "C"
