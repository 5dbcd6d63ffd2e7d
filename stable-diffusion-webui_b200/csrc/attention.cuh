// Argument block of the wgmma flash-attention kernel (attention.cu).
#pragma once
#include "common.cuh"
#include <vector>

namespace sdxe {

struct alignas(64) AttnArgs {
  // 4D per-head views (common.cuh make_tmap_heads): {d (true head dim: boxes reaching past it are zero-filled), token,
  // head, batch}, 128B swizzle. Box 64 x 128 for Q, 64 x 64 for K and V.
  CUtensorMap tmQ;
  CUtensorMap tmK;
  CUtensorMap tmV;
  int B, H, Nq, Nk;
  int dqk_slabs;    // dqk_pad / 64  (1..8)
  int dv_slabs;     // value columns of this pass / 64, rounded up (1..2); wider heads run in several passes
  int dv;           // valid value columns of this pass that are stored (multiple of 8)
  int dqk;          // valid q/k columns (<= dqk_slabs * 64); columns beyond are zero padding
  int num_slots;    // set by the launcher
  float scale_log2; // softmax scale * log2(e)
  void* out;        // [B*Nq, ldo] 16-bit; head h writes columns out_col0 + h*out_hstride ...
  int ldo;
  int out_col0;
  int out_hstride;
  // Hypertile (segmented) attention, seg != null: the Nq = Nk tokens of a batch are the tile-major rows of an
  // seg_h x seg_w grid cut into nh x nw tiles, (nh, nw) = seg[0], seg[1] read from device memory at run time. Each query
  // attends to the T = (seg_h / nh) (seg_w / nw) keys of its own tile and its output row goes back to its natural
  // (row-major grid) position. The grid is sized for seg_max_tiles tiles.
  const int* seg;
  int seg_h, seg_w, seg_max_tiles;
};

static constexpr int ATTN_Q_BOX_ROWS = 128;
static constexpr int ATTN_KV_BOX_ROWS = 64;
static constexpr int ATTN_MAX_DV = 128;  // value columns per pass

// One operand of attention as a per-head view: element j of token t, head h, batch b at
// p + b * batch_stride + t * tok_stride + h * head_stride + j (strides in elements, multiples of 8).
struct AttnView {
  const void* p;
  int64_t tok_stride, head_stride, batch_stride;
};
// softmax(q k^T * scale) v with q / k of head dim dqk and dv value columns per head, written to out[b * Nq + t, h * out_hstride
// + j] (row pitch ldo). Value columns run in passes of at most ATTN_MAX_DV: one AttnArgs per pass. Returns 0 / -1.
int attention_args(std::vector<AttnArgs>& passes, const AttnView& q, const AttnView& k, const AttnView& v, int B, int H,
                   int Nq, int Nk, int dqk, int dv, float scale, void* out, int ldo, int out_hstride);
int attention_launch(const AttnArgs& a, bool bf16, cudaStream_t stream);
int attention_init();

// Hypertile (extensions-builtin/hypertile/hypertile.py:269-313): the per-call tile draws (nh, nw) of n layers, passed
// by value (kernel parameters are captured at launch) and written to table[2 * layer + {0, 1}].
static constexpr int HT_MAX_LAYERS = 128;
struct HtDraws {
  int n;
  int v[2 * HT_MAX_LAYERS];
};
int hypertile_table_launch(const HtDraws& d, int* table, cudaStream_t stream);
// dst[b, tile-major row] = src[b, natural row] for the B x (seg_h * seg_w) rows of `row_elems` 16-bit elements (a
// multiple of 8): the regrouping b (nh h nw w) c -> (b nh nw) (h w) c with (nh, nw) = seg[0], seg[1].
int hypertile_gather_launch(const void* src, void* dst, int B, int seg_h, int seg_w, int row_elems, const int* seg,
                            cudaStream_t stream);

}  // namespace sdxe
