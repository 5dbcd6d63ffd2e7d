// FlashAttention-style softmax(Q K^T * scale) V for sm_90a on wgmma + TMA + mbarrier.
//
// Replaces every CrossAttention.forward / AttnBlock.forward variant of the reference
// (modules/sd_hijack_optimizations.py:180-655: split, Doggettx, InvokeAI, sub-quadratic, xformers, sdp):
// one kernel for UNet self-attention (Nk = Nq in {4096,1024,256,64}), cross-attention (Nk = 77*k) and the
// VAE AttnBlock (single head, d = 512, run as passes over 128-wide slices of V).
//
// Inputs are the projection GEMMs' row-major outputs ([B*tokens, 3C] = q|k|v, heads contiguous inside each) seen
// through 4D tensor maps (d, token, head, batch): a 64-wide slab reaching past the head dim d is zero-filled by TMA,
// so no padded / transposed per-head copy exists. Output is merged-head [B*Nq, H*d] for the out-projection.
//
// CTA = one 128-row query tile of one (batch, head):
//   warp 8     : TMA producer. Q slabs once (resident), then per 64-key block its K slabs and V slabs (64 x 64
//                elements, 8 KB, 128B swizzle) through one in-order ring, in exactly the order they are consumed.
//   warps 0-7  : two warpgroups of 64 query rows each. S = Q K^T with wgmma from shared memory into registers, online
//                softmax on the accumulator fragment, P converted in registers into the A operand of O += P V
//                (V read MN-major straight from its natural [kv, dv] layout), final 1/l scaling and store. Each
//                warpgroup runs the softmax of a block under its O += P V of the previous block.
#include "attention.cuh"
#include "wgmma.cuh"
#include <algorithm>
#include <cstring>
#include <type_traits>

namespace sdxe {

static constexpr int SLAB_BYTES = 64 * 64 * 2;    // one K or V slab: 64 keys x 64 columns
static constexpr int Q_SLAB_BYTES = 128 * 64 * 2;  // one Q slab: 128 query rows x 64 columns
static constexpr int ATT_THREADS = 288;            // warpgroups 0-1: MMA + softmax, warp 8: TMA producer
static constexpr int CONSUMER_WARPS = 8;
static constexpr int KV_BLOCK = 64;
static constexpr int SMEM_BUDGET = 227 * 1024;

// One K slab's share of S = Q K^T, committed as one group: the first STEPS k16 steps of the 64-wide slab (acc = 0
// starts S).
template <int STEPS, bool BF16> SDXE_DEVINL void qk_slab(float* s, uint64_t qd, uint64_t kd, int acc) {
  wgmma_fence();
  wgmma_ss<64, BF16>(s, qd, kd, acc);
#pragma unroll
  for (int k = 1; k < STEPS; ++k) wgmma_ss<64, BF16>(s, qd + 2 * k, kd + 2 * k, 1);
  wgmma_commit();
}
// One V slab's O += P V over the 64 keys of a block at width N, committed as one group. V is read MN-major; +16 key
// rows = +2048 B.
template <int N, bool BF16> SDXE_DEVINL void pv_slab(float* o, const uint32_t (&pa)[4][4], uint64_t vd) {
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) wgmma_rs_tb<N, BF16>(o, pa[kk], vd + 128 * kk, 1);
  wgmma_commit();
}

// SEG: Hypertile segmented attention (AttnArgs::seg). A CTA takes query block blockIdx.x % qblocks of tile
// blockIdx.x / qblocks; CTAs past the drawn tile count exit. Only addressing differs from the plain kernel: a draw of
// (1, 1) computes bit-identical results.
template <bool BF16, int NVS, bool SEG, int HD>
__global__ void __launch_bounds__(ATT_THREADS, 1) attention_kernel(const __grid_constant__ AttnArgs a) {
  using T = T16<BF16>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;

  const int NS = a.num_slots;
  const uint32_t sQ = sbase;
  const uint32_t sRing = sQ + a.dqk_slabs * Q_SLAB_BYTES;
  const uint32_t bar_base = sRing + NS * SLAB_BYTES;
  auto slot_full = [&](int s) { return bar_base + 8u * s; };
  auto slot_empty = [&](int s) { return bar_base + 8u * (NS + s); };
  const uint32_t q_full = bar_base + 8u * (2 * NS);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int q0 = blockIdx.x * 128;  // SEG: relative to the tile's first row
  int Nk = a.Nk;              // SEG: the tile's token count T
  int row0 = 0;               // SEG: first (tile-major) row of the tile
  int tile = 0, th = 0, tw = 0, nw = 1;
  if constexpr (SEG) {
    const int nh = a.seg[0];
    nw = a.seg[1];
    th = a.seg_h / nh;
    tw = a.seg_w / nw;
    Nk = th * tw;
    const int qblocks = (Nk + 127) / 128;
    tile = blockIdx.x / qblocks;
    if (tile >= nh * nw) return;  // the grid covers seg_max_tiles tiles
    row0 = tile * Nk;
    q0 = (blockIdx.x - tile * qblocks) * 128;
  }
  const int bh = blockIdx.y;
  const int hb_b = bh / a.H, hb_h = bh - hb_b * a.H;  // (batch, head) coordinates of the 4D per-head tensor maps
  const int nblk = (Nk + KV_BLOCK - 1) / KV_BLOCK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < NS; ++s) { mbar_init(slot_full(s), 1); mbar_init(slot_empty(s), CONSUMER_WARPS); }
    mbar_init(q_full, 1);
    fence_mbar_init();
    tma_prefetch_desc(&a.tmQ);
    tma_prefetch_desc(&a.tmK);
    tma_prefetch_desc(&a.tmV);
  }
  __syncthreads();

  if (warp == CONSUMER_WARPS) {
    // ---------------------------------------------------------------- producer (converged warp, elected issue)
    if (elect_one()) {
      mbar_expect_tx(q_full, a.dqk_slabs * Q_SLAB_BYTES);
      for (int c = 0; c < a.dqk_slabs; ++c) tma_load_4d(sQ + c * Q_SLAB_BYTES, &a.tmQ, q_full, c * 64, row0 + q0, hb_h, hb_b);
    }
    __syncwarp();
    int slot = 0;
    uint32_t phase = 0;
    auto push = [&](const CUtensorMap* tm, int c0, int r0) {
      mbar_wait(slot_empty(slot), phase ^ 1u);
      if (elect_one()) {
        mbar_expect_tx(slot_full(slot), SLAB_BYTES);
        tma_load_4d(sRing + slot * SLAB_BYTES, tm, slot_full(slot), c0, r0, hb_h, hb_b);
      }
      __syncwarp();
      if (++slot == NS) { slot = 0; phase ^= 1u; }
    };
    // K_0, then K_j before V_{j-1}: the order in which the software-pipelined consumers take them
    for (int j = 0; j <= nblk; ++j) {
      if (j < nblk)
        for (int c = 0; c < a.dqk_slabs; ++c) push(&a.tmK, c * 64, row0 + j * KV_BLOCK);
      if (j > 0)
        for (int vs = 0; vs < NVS; ++vs) push(&a.tmV, vs * 64, row0 + (j - 1) * KV_BLOCK);
    }
    return;
  }

  // ------------------------------------------------------------------ MMA + softmax warpgroups
  // Accumulator fragment of wgmma m64n64 (per warp 16 rows): x[4 i + 2 h + e] is row (lane / 4 + 8 h) of the warp's
  // band, column 8 i + 2 (lane % 4) + e.
  const int wg = warp >> 2;
  const int band = (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const float sl2 = a.scale_log2;
  const uint64_t qdesc0 = gmma_desc_sw128(sQ + (uint32_t)wg * (64 * 128), 16, 1024);
  // k16 steps of QK^T in the last K slab and width of O += P V in the last V slab of the pass, for the head dims the
  // UNets run (d = 40; 80; 160 in passes of 128 and 32 value columns). Steps and columns past the head dim would only
  // multiply zero padding; any other head dim runs whole 64-wide slabs.
  constexpr int QK_LAST = HD == 40 ? 3 : HD == 80 ? 1 : HD == 160 ? 2 : 4;
  constexpr int PV_LAST = HD == 40 ? 40 : HD == 80 ? 16 : (HD == 160 && NVS == 1) ? 32 : 64;
  float o[NVS][32];
#pragma unroll
  for (int vs = 0; vs < NVS; ++vs)
#pragma unroll
    for (int i = 0; i < 32; ++i) o[vs][i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  int slot = 0;
  uint32_t phase = 0;
  auto advance = [&]() { if (++slot == NS) { slot = 0; phase ^= 1u; } };
  auto release_from = [&](int first, int count) {  // slots first .. first + count - 1 (ring order) may be refilled
    if (lane == 0)
      for (int t = 0, s = first; t < count; ++t, s = (s + 1 == NS) ? 0 : s + 1) mbar_arrive(slot_empty(s));
  };

  // S = Q K_j^T over the next dqk_slabs ring slots, one group per slab
  auto issue_s = [&](float (&s)[32]) {
    auto slab = [&](int c, auto steps) {
      mbar_wait(slot_full(slot), phase);
      const uint64_t kd = gmma_desc_sw128(sRing + slot * SLAB_BYTES, 16, 1024);
      qk_slab<decltype(steps)::value, BF16>(s, qdesc0 + (uint64_t)(c * (Q_SLAB_BYTES >> 4)), kd, c != 0);
      advance();
    };
    for (int c = 0; c + 1 < a.dqk_slabs; ++c) slab(c, std::integral_constant<int, 4>());
    slab(a.dqk_slabs - 1, std::integral_constant<int, QK_LAST>());
  };
  // O += P V over the next NVS ring slots, one group per slab
  auto issue_pv = [&](const uint32_t (&pa)[4][4]) {
#pragma unroll
    for (int vs = 0; vs < NVS; ++vs) {
      mbar_wait(slot_full(slot), phase);
      const uint64_t vd = gmma_desc_sw128(sRing + slot * SLAB_BYTES, SLAB_BYTES, 1024);
      if (vs + 1 < NVS) pv_slab<64, BF16>(o[vs], pa, vd);
      else pv_slab<PV_LAST, BF16>(o[vs], pa, vd);
      advance();
    }
  };
  // online softmax of block j on the fragment (a row's 64 columns live in the four threads of a quad): updates m and l,
  // returns the O rescale factor in alpha and the unnormalised probabilities in p. S is only read: ptxas serialises
  // every wgmma of the kernel if other instructions write accumulator registers while O += P V is in flight (C7515).
  // MASKED: the block may be the last one, whose key columns past Nk (SEG: keys of the next tile) count as -inf.
  auto softmax = [&](const float (&s)[32], int j, float (&p)[32], float (&alpha)[2], auto masked) {
    const int nvalid = Nk - j * KV_BLOCK;
    auto sv = [&](int r) {  // register r holds column 8 (r / 4) + cq + r % 2
      return (decltype(masked)::value && 8 * (r >> 2) + cq + (r & 1) >= nvalid) ? -INFINITY : s[r];
    };
    float mb[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 8; ++i) mx = fmaxf(mx, fmaxf(sv(4 * i + 2 * h), sv(4 * i + 2 * h + 1)));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx);  // finite: every block holds at least one valid key
      alpha[h] = ex2_approx((m_run[h] - m_new) * sl2);  // first block: 2^-inf = 0
      l_run[h] *= alpha[h];
      m_run[h] = m_new;
      mb[h] = m_new * sl2;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int t = 0; t < 4; ++t) p[4 * i + t] = ex2_approx(fmaf(sv(4 * i + t), sl2, -mb[t >> 1]));
      l_run[0] += p[4 * i] + p[4 * i + 1];
      l_run[1] += p[4 * i + 2] + p[4 * i + 3];
    }
  };
  // P in the A-operand fragment of m64nNk16: key step kk uses column blocks 2 kk (regs 0, 1) and 2 kk + 1 (regs 2, 3)
  uint32_t pa[4][4];
  auto pack_p = [&](const float (&p)[32]) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      pa[i >> 1][(i & 1) * 2 + 0] = T::pack(p[4 * i], p[4 * i + 1]);
      pa[i >> 1][(i & 1) * 2 + 1] = T::pack(p[4 * i + 2], p[4 * i + 3]);
    }
  };
  auto wait_o = [&](int v_first) {
    wgmma_wait<0>();
#pragma unroll
    for (int vs = 0; vs < NVS; ++vs)
#pragma unroll
      for (int i = 0; i < 32; ++i) reg_fence(o[vs][i]);
    release_from(v_first, NVS);
  };

  // Software pipeline (per warpgroup): block j's S is waited for, then O += P_{j-1} V_{j-1} is issued and runs on the
  // tensor cores while the softmax of block j runs. (Issuing S_j and that MMA back to back and waiting for S_j alone
  // measured slower on H100.) Per row, O, l and m see the same operations in the same order as with no overlap (o = o alpha_j is applied after o += P_{j-1} V_{j-1}, before o += P_j V_j).
  // The ring holds K_0, K_1, V_0, K_2, V_1, ..., V_{n-1}: consumption order. P_j stays in fp32 until the MMA, which
  // reads the 16-bit P_{j-1} from registers, is complete.
  float alpha[2];
  mbar_wait(q_full, 0);
  {
    float s[32], p[32];
    const int k_first = slot;
    issue_s(s);
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 32; ++i) reg_fence(s[i]);
    release_from(k_first, a.dqk_slabs);
    softmax(s, 0, p, alpha, std::true_type());  // alpha = 0 would scale the zero O: nothing to do
    pack_p(p);
  }
  auto step = [&](int j, auto masked) {
    float s[32], p[32];  // fresh per block, so that only wgmma defines s
    const int k_first = slot;
    issue_s(s);
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 32; ++i) reg_fence(s[i]);
    release_from(k_first, a.dqk_slabs);
    const int v_first = slot;
    issue_pv(pa);
    softmax(s, j, p, alpha, masked);
#pragma unroll
    for (int i = 0; i < 32; ++i) reg_fence(p[i]);
    wait_o(v_first);
    pack_p(p);
#pragma unroll
    for (int vs = 0; vs < NVS; ++vs)
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h) { o[vs][4 * i + 2 * h] *= alpha[h]; o[vs][4 * i + 2 * h + 1] *= alpha[h]; }
  };
  // only the last block can hold keys past Nk: the loop runs the unmasked softmax
  for (int j = 1; j < nblk - 1; ++j) step(j, std::false_type());
  if (nblk > 1) step(nblk - 1, std::true_type());
  {
    const int v_first = slot;
    issue_pv(pa);
    wait_o(v_first);
  }

  // ---- epilogue: O / l -> out[b, q, out_col0 + h * out_hstride + j]
  using TT = typename T::type;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv_l = 1.f / l;
    int q = q0 + wg * 64 + band + 8 * h;
    if (q >= (SEG ? Nk : a.Nq)) continue;
    if constexpr (SEG) {  // tile-major row -> natural row of the seg_h x seg_w grid
      const int r = q / tw, c = q - r * tw, ih = tile / nw, iw = tile - ih * nw;
      q = (ih * th + r) * a.seg_w + iw * tw + c;
    }
    TT* orow = reinterpret_cast<TT*>(a.out) + ((size_t)hb_b * a.Nq + q) * a.ldo + a.out_col0 + hb_h * a.out_hstride;
#pragma unroll
    for (int vs = 0; vs < NVS; ++vs)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int col = vs * 64 + 8 * i + cq;  // even, dv a multiple of 8: col + 1 is valid with col
        if (col < a.dv)
          *reinterpret_cast<uint32_t*>(orow + col) = T::pack(o[vs][4 * i + 2 * h] * inv_l, o[vs][4 * i + 2 * h + 1] * inv_l);
      }
  }
}

typedef void (*AttnKernel)(const AttnArgs);
// head-dim class of a pass (attention_kernel's HD): 40, 80 and 160 for the passes the UNets run, 0 for any other
static int attention_head_dim(const AttnArgs& a) {
  if (a.dqk == 40 && a.dv == 40) return 40;
  if (a.dqk == 80 && a.dv == 80) return 80;
  if (a.dqk == 160 && (a.dv == 128 || a.dv == 32)) return 160;
  return 0;
}
template <bool BF16, bool SEG> static AttnKernel attention_variant(int nvs, int hd) {
  if (hd == 40) return attention_kernel<BF16, 1, SEG, 40>;
  if (hd == 80) return attention_kernel<BF16, 2, SEG, 80>;
  if (hd == 160) return nvs == 1 ? attention_kernel<BF16, 1, SEG, 160> : attention_kernel<BF16, 2, SEG, 160>;
  return nvs == 1 ? attention_kernel<BF16, 1, SEG, 0> : attention_kernel<BF16, 2, SEG, 0>;
}
static AttnKernel attention_variant(bool bf16, int nvs, bool seg, int hd) {
  if (seg) return bf16 ? attention_variant<true, true>(nvs, hd) : attention_variant<false, true>(nvs, hd);
  return bf16 ? attention_variant<true, false>(nvs, hd) : attention_variant<false, false>(nvs, hd);
}

int attention_init() {
  static bool done = false;
  if (!done) {
    for (int b = 0; b < 2; ++b)
      for (int nvs = 1; nvs <= 2; ++nvs)
        for (int seg = 0; seg < 2; ++seg)
          for (int hd : {0, 40, 80, 160})
            SDXE_CUDA_CHECK(cudaFuncSetAttribute(attention_variant(b != 0, nvs, seg != 0, hd),
                                                 cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BUDGET));
    done = true;
  }
  return 0;
}

int attention_launch(const AttnArgs& a_in, bool bf16, cudaStream_t stream) {
  AttnArgs a = a_in;
  if (a.dv_slabs < 1 || a.dv_slabs * 64 > ATTN_MAX_DV || a.dqk_slabs < 1 || a.dqk_slabs > 8 || a.dv % 8 != 0 ||
      a.dv > a.dv_slabs * 64) {
    set_last_error(__FILE__, __LINE__, "attention: unsupported head size");
    return -1;
  }
  const size_t fixed = 1024 /*alignment*/ + (size_t)a.dqk_slabs * Q_SLAB_BYTES + 8;
  // every K slab of a block stays resident until the block's S is complete, so the ring holds at least dqk_slabs
  a.num_slots = (int)std::min<size_t>(16, (SMEM_BUDGET - fixed) / (SLAB_BYTES + 16));
  if (a.num_slots < std::max(2, a.dqk_slabs)) { set_last_error(__FILE__, __LINE__, "attention: smem"); return -1; }
  const size_t smem = fixed + (size_t)a.num_slots * (SLAB_BYTES + 16);
  if (attention_init() != 0) return -1;
  const bool seg = a.seg != nullptr;
  if (seg && (a.Nq != a.Nk || a.seg_h * a.seg_w != a.Nq || a.seg_max_tiles < 1)) {
    set_last_error(__FILE__, __LINE__, "attention: bad Hypertile geometry");
    return -1;
  }
  // a tiling into k tiles of T tokens needs k ceil(T / 128) <= ceil(Nq / 128) + k - 1 query blocks
  dim3 grid((a.Nq + 127) / 128 + (seg ? a.seg_max_tiles - 1 : 0), a.B * a.H);
  const AttnKernel kern = attention_variant(bf16, a.dv_slabs, seg, attention_head_dim(a));
  kern<<<grid, ATT_THREADS, smem, stream>>>(a);
  SDXE_LAUNCH_CHECK();
  return 0;
}

__global__ void hypertile_table_kernel(const HtDraws d, int* __restrict__ table) {
  for (int i = threadIdx.x; i < 2 * d.n; i += blockDim.x) table[i] = d.v[i];
}

int hypertile_table_launch(const HtDraws& d, int* table, cudaStream_t stream) {
  if (d.n < 1 || d.n > HT_MAX_LAYERS) { set_last_error(__FILE__, __LINE__, "hypertile: layer count"); return -1; }
  hypertile_table_kernel<<<1, 256, 0, stream>>>(d, table);
  SDXE_LAUNCH_CHECK();
  return 0;
}

// one CTA per destination row: 16-byte vectors of the row copied from its natural position
__global__ void hypertile_gather_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int N, int seg_h,
                                        int seg_w, int row_vecs, const int* __restrict__ seg) {
  const int nh = seg[0], nw = seg[1];
  const int th = seg_h / nh, tw = seg_w / nw, T = th * tw;
  const int64_t p = blockIdx.x;  // b * N + tile-major row
  const int b = (int)(p / N), l = (int)(p - (int64_t)b * N);
  const int tile = l / T, t = l - tile * T;
  const int r = t / tw, c = t - r * tw, ih = tile / nw, iw = tile - ih * nw;
  const int64_t n = (int64_t)b * N + (int64_t)(ih * th + r) * seg_w + iw * tw + c;
  const uint4* s = src + n * row_vecs;
  uint4* o = dst + p * row_vecs;
  for (int i = threadIdx.x; i < row_vecs; i += blockDim.x) o[i] = s[i];
}

int hypertile_gather_launch(const void* src, void* dst, int B, int seg_h, int seg_w, int row_elems, const int* seg,
                            cudaStream_t stream) {
  if (row_elems % 8 || B < 1 || seg_h < 1 || seg_w < 1) { set_last_error(__FILE__, __LINE__, "hypertile gather: shape"); return -1; }
  const int row_vecs = row_elems / 8;
  hypertile_gather_kernel<<<(unsigned)((int64_t)B * seg_h * seg_w), std::min(256, (row_vecs + 31) / 32 * 32), 0, stream>>>(
      (const uint4*)src, (uint4*)dst, seg_h * seg_w, seg_h, seg_w, row_vecs, seg);
  SDXE_LAUNCH_CHECK();
  return 0;
}

int attention_args(std::vector<AttnArgs>& passes, const AttnView& q, const AttnView& k, const AttnView& v, int B, int H,
                   int Nq, int Nk, int dqk, int dv, float scale, void* out, int ldo, int out_hstride) {
  passes.clear();
  for (int v0 = 0; v0 < dv; v0 += ATTN_MAX_DV) {  // the O accumulator of a pass lives in registers
    const int w = std::min(ATTN_MAX_DV, dv - v0);
    AttnArgs a;
    memset(&a, 0, sizeof(a));
    // a 64-wide box reaching past the head dim (or the pass's value columns) is zero-filled by TMA
    if (make_tmap_heads(&a.tmQ, q.p, dqk, Nq, H, B, q.tok_stride, q.head_stride, q.batch_stride, ATTN_Q_BOX_ROWS)) return -1;
    if (make_tmap_heads(&a.tmK, k.p, dqk, Nk, H, B, k.tok_stride, k.head_stride, k.batch_stride, ATTN_KV_BOX_ROWS)) return -1;
    if (make_tmap_heads(&a.tmV, (const uint16_t*)v.p + v0, w, Nk, H, B, v.tok_stride, v.head_stride, v.batch_stride,
                        ATTN_KV_BOX_ROWS))
      return -1;
    a.B = B; a.H = H; a.Nq = Nq; a.Nk = Nk;
    a.dqk_slabs = (dqk + 63) / 64;
    a.dv_slabs = (w + 63) / 64;
    a.dv = w;
    a.dqk = dqk;
    a.scale_log2 = scale * 1.4426950408889634f;
    a.out = out; a.ldo = ldo; a.out_col0 = v0; a.out_hstride = out_hstride;
    passes.push_back(a);
  }
  return 0;
}

}  // namespace sdxe
