"""Per-element fp64 bounds for the stand-alone CUDA primitives (tests/test_prims_gpu.py, the Hypertile primitive test in
tests/test_hypertile_gpu.py, and their negative controls in tests/test_prim_bounds_cpu.py).

Every reference is computed in fp64 from the exact 16-bit inputs, upcast, and every output element must satisfy
|out - ref| <= bound. The bounds follow what the kernels do: exact 16-bit products accumulated in fp32, fp32 statistics,
P rounded to 16 bit in front of the PV MMA, and the output rounded to 16 bit. `ulp16(ref)` is one ulp of the output
format at |ref|: twice the round-to-nearest error, which also covers a result that rounds up across a power of two.
A norm over the whole tensor cannot see a fault that stays in one row, one key or one tile; a per-element bound can.

This module is device-agnostic (fp64 on whatever device the inputs are on) and imports nothing from the package.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

U32 = 2.0 ** -24  # unit roundoff of fp32
GELU_ERF_ABS = 1.5e-7  # Abramowitz-Stegun 7.1.26, the erf behind gelu_fast_f (csrc/common.cuh)


def unit16(dtype) -> float:
    """Unit roundoff of the 16-bit format."""
    return 2.0 ** -11 if dtype == torch.float16 else 2.0 ** -8


def ulp16(ref: torch.Tensor, dtype) -> torch.Tensor:
    """One ulp of `dtype` at |ref| (fp64); the subnormal spacing below the smallest normal."""
    mant, emin = (10, -14) if dtype == torch.float16 else (7, -126)
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** emin)))
    return torch.exp2(e - mant)


def check(what: str, out: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, where=None) -> float:
    """Assert |out - ref| <= bound for every element. Prints and returns the worst ratio |err| / bound; on failure the
    message names its index and, through where(index) -> str, its tile coordinates. A non-finite output counts as inf."""
    o = out.double()
    ratio = ((o - ref).abs() / bound).reshape(-1)
    ratio = torch.where(torch.isfinite(o.reshape(-1)), ratio, torch.full_like(ratio, math.inf))
    i = int(torch.argmax(ratio))
    worst = float(ratio[i])
    idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), ref.shape))
    loc = f" [{where(idx)}]" if where else ""
    msg = (f"{what}: worst |err|/bound {worst:.3g} at {idx}{loc}: out {float(o.reshape(-1)[i]):.6g} "
           f"ref {float(ref.reshape(-1)[i]):.6g} bound {float(bound.reshape(-1)[i]):.3g}")
    print(msg)
    assert worst <= 1.0, msg
    return worst


# ---- GEMM, GEGLU, conv ------------------------------------------------------------------------------------------
def _acc_bound(mag: torch.Tensor, K: int, extra_adds: int) -> torch.Tensor:
    """fp32 accumulation of K exact products plus `extra_adds` epilogue additions, each rounding at most u32 of the
    running magnitude; the factor 2 leaves room for an accumulator that truncates instead of rounding to nearest."""
    return 2 * (K + extra_adds) * U32 * mag


def gemm_ref(a, w, bias=None, residual=None):
    """out = a w^T (+ bias) (+ residual), a [M, K], w [N, K]: (ref, bound) in fp64.

    bound = ulp16(ref) + 2 (K + 2) u32 (sum_k |a_ik w_jk| + |b_j| + |r_ij|): the wgmma sums K exact products in fp32,
    the epilogue adds bias and residual in fp32 and rounds once to 16 bit."""
    ad, wd = a.double(), w.double()
    ref, mag = ad @ wd.t(), ad.abs() @ wd.abs().t()
    for t in (bias, residual):
        if t is not None:
            ref = ref + t.double()
            mag = mag + t.double().abs()
    return ref, ulp16(ref, a.dtype) + _acc_bound(mag, a.shape[1], 2)


def geglu_ref(a, w, bias=None):
    """GEGLU: out[:, j] = v_j gelu(g_j), with v the first N/2 and g the last N/2 columns of a w^T + b: (ref, bound).

    v and g carry the GEMM accumulation bound e = 2 (K + 1) u32 (sum |a w| + |b|). |gelu'| <= 1.13, so gelu(g) is off
    by at most 1.13 e_g from the accumulation, plus gelu_fast_f's own error: the erf approximation's 1.5e-7 times
    |g| / 2, and at most 16 u32 |g| from its fp32 evaluation (ex2.approx, rcp.approx, six FMAs). Then
    |v gelu(g) - v_ref gelu(g_ref)| <= e_v |gelu(g_ref)| + (|v_ref| + e_v) e_gelu, one fp32 product rounding, and the
    16-bit output rounding."""
    ad, wd = a.double(), w.double()
    proj, mag = ad @ wd.t(), ad.abs() @ wd.abs().t()
    if bias is not None:
        proj, mag = proj + bias.double(), mag + bias.double().abs()
    e = _acc_bound(mag, a.shape[1], 1)
    h = proj.shape[1] // 2
    v, g, ev, eg = proj[:, :h], proj[:, h:], e[:, :h], e[:, h:]
    gl = 0.5 * g * (1 + torch.special.erf(g / math.sqrt(2)))
    egl = 1.13 * eg + (GELU_ERF_ABS / 2 + 16 * U32) * g.abs()
    ref = v * gl
    return ref, ulp16(ref, a.dtype) + ev * gl.abs() + (v.abs() + ev) * egl + U32 * ref.abs()


def conv3x3_ref(x, w, bias=None):
    """3x3 convolution, stride 1, zero padding 1: x [n, h, w, cin] NHWC, w [cout, cin, 3, 3] -> (ref, bound) NHWC.
    The implicit GEMM has K = 9 cin; the bound is gemm_ref's with one epilogue addition (the bias)."""
    n, h, wd_, cin = x.shape
    cols = F.unfold(x.double().permute(0, 3, 1, 2), 3, padding=1).transpose(1, 2)  # [n, hw, cin * 9]
    wm = w.double().reshape(w.shape[0], -1)
    ref, mag = cols @ wm.t(), cols.abs() @ wm.abs().t()
    if bias is not None:
        ref, mag = ref + bias.double(), mag + bias.double().abs()
    ref, mag = ref.reshape(n, h, wd_, -1), mag.reshape(n, h, wd_, -1)
    return ref, ulp16(ref, x.dtype) + _acc_bound(mag, 9 * cin, 1)


# ---- attention ---------------------------------------------------------------------------------------------------
def attention_ref(q, k, v, scale=None, chunk=1024):
    """softmax(q k^T scale) v for q [B, H, Nq, D], k / v [B, H, Nk, D] -> (ref, bound) as [B, Nq, H * D], in fp64,
    computed in query chunks so that 15808 x 15808 scores never exist at once.

    Derivation, following csrc/attention.cu. The kernel forms p_j = 2^(s_j sl2 - m sl2) in fp32 and sums the row's
    l = sum_j p_j from these unrounded p_j (softmax(): l_run += p before pack_p), but multiplies V by P rounded to
    16 bit (pack_p feeds the PV wgmma). So o = sum_j round16(p_j) v_j / l: the rounding of P is not compensated by
    the normalisation, and it moves o by at most u16 sum_j P_j |v_j| with P = p / l: c = 1. (Were l summed from the
    rounded p, the error would be u16 sum_j P_j |v_j - o|, up to twice that.) fp16 P below 2^-14 is subnormal, with an
    absolute rounding error of 2^-25 instead: at most 2^-25 sum_j |v_j| / l over all keys.
    The rest is fp32 arithmetic:
    * PV accumulation over Nk keys with the alpha rescales: 2 Nk u32 sum_j P_j |v_j|, as for a GEMM with K = Nk;
    * relative error eps_j of p_j: the QK^T accumulation (scale 2 D u32 sum_d |q_d k_jd|), the rounding of the ex2
      argument (u32 |s_j - m| scale log2 e, at most one ulp for each of the two fp32 operations) and ex2.approx
      (2 ulp): eps_j = scale 2 D u32 sum |q k_j| + 8 u32 (1 + scale |s_j - m|). Relative errors eps_j of the weights
      move o = sum p_j v_j / sum p_j by at most sum_j P_j eps_j (|v_j| + |o|);
    * the final o / l: 4 u32 |o|.
    bound = ulp16(o) + (u16 + 2 Nk u32) sum_j P_j |v_j| + sum_j P_j eps_j (|v_j| + |o|) + eta |v|_1 / l + 4 u32 |o|."""
    B, H, Nq, D = q.shape
    Nk = k.shape[2]
    sc = float(scale) if scale is not None else D ** -0.5
    u16 = unit16(q.dtype)
    eta = 2.0 ** -25 if q.dtype == torch.float16 else 2.0 ** -134
    ref = torch.empty(B, Nq, H, D, dtype=torch.float64, device=q.device)
    bound = torch.empty_like(ref)
    for b in range(B):
        for h in range(H):
            kd, vd = k[b, h].double(), v[b, h].double()
            ka, va = kd.abs(), vd.abs()
            v1 = va.sum(0)
            for c0 in range(0, Nq, chunk):
                qd = q[b, h, c0:c0 + chunk].double()
                s = (qd @ kd.t()) * sc
                m = s.amax(-1, keepdim=True)
                e = torch.exp(s - m)
                l = e.sum(-1, keepdim=True)
                P = e / l
                o = P @ vd
                eps = sc * 2 * D * U32 * (qd.abs() @ ka.t()) + 8 * U32 * (1 + (m - s))
                Pe = P * eps
                bd = (ulp16(o, q.dtype) + (u16 + 2 * Nk * U32) * (P @ va) + Pe @ va + Pe.sum(-1, keepdim=True) * o.abs()
                      + eta * v1 / l + 4 * U32 * o.abs())
                ref[b, c0:c0 + chunk, h] = o
                bound[b, c0:c0 + chunk, h] = bd
                del s, e, P, eps, Pe
    return ref.reshape(B, Nq, H * D), bound.reshape(B, Nq, H * D)


# ---- GroupNorm, LayerNorm ----------------------------------------------------------------------------------------
def _norm_bound(xd, mu, var, e2, absmean, gamma, beta, eps, depth, silu, dtype):
    """y = (x - mu) rstd gamma + beta (+ SiLU) with fp32 statistics whose additions form chains of at most `depth`
    roundings: dmu <= depth u32 mean|x|, dvar <= (depth + 3) u32 E[x^2] + 2 |mu| dmu + dmu^2 (this covers the
    uncentred E[x^2] - mu^2 of the streaming GroupNorm as well as the centred second pass), rstd = rsqrtf(var + eps)
    off by dvar / (2 (var + eps)) + 4 u32 (rsqrtf: 2 ulp). The output moves by |gamma| rstd dmu + |gamma x^| drstd,
    plus 3 u32 (|gamma| rstd (|x| + |mu|) + |beta|) for the scale / shift / FMA roundings. silu_f (x rcp(1 + ex2(-x
    log2 e))) adds 8 u32 (1 + |z|) |silu(z)| and passes the error of z on with |silu'| <= 1.1."""
    r = 1.0 / torch.sqrt(var + eps)
    xh = (xd - mu) * r
    z = xh * gamma + beta
    dmu = depth * U32 * absmean
    dvar = (depth + 3) * U32 * e2 + 2 * mu.abs() * dmu + dmu * dmu
    drel = dvar / (2 * (var + eps)) + 4 * U32
    ga = gamma.abs()
    ez = ga * r * dmu + (ga * xh.abs()) * drel + 3 * U32 * (ga * r * (xd.abs() + mu.abs()) + beta.abs())
    if silu:
        y = z * torch.sigmoid(z)
        ey = 1.1 * ez + 8 * U32 * (1 + z.abs()) * y.abs()
    else:
        y, ey = z, ez
    return y, ulp16(y, dtype) + ey


def gn_depth(n, hw, c, groups=32, num_sms=132):
    """Longest chain of fp32 additions behind one group's statistics in group_norm_launch (csrc/kernels.cu), for
    either path. One-pass (strip hw * C/groups * 2 B <= 48 KB): a thread's sum over its pixels (two channels per
    pixel) then the block reduction (5 + 4 shuffle levels). Streaming: a thread's sum over its rows of the block's
    pixel chunk, the shared-memory sum over rpi rows x cpg channels, the finalize lane sum over chunks and 5 shuffles.
    Returns (depth, "onepass" | "streaming")."""
    cpg = c // groups
    strip = hw * cpg * 2
    if cpg % 2 == 0 and cpg // 2 <= 256 and strip <= 48 * 1024:
        threads = 512 if strip >= 32 * 1024 else 256
        R = threads // (cpg // 2)
        return -(-hw // R) + 10, "onepass"
    V = c // 8
    rpi = max(1, 256 // V)
    while rpi > 1 and rpi * c * 8 > 96 * 1024:
        rpi -= 1
    chunks = max(1, min((num_sms * 4 + n - 1) // n, (hw + rpi * 4 - 1) // (rpi * 4)))
    ppb = -(-hw // chunks)
    chunks = -(-hw // ppb)
    return -(-ppb // rpi) + rpi * cpg + -(-chunks // 32) + 5, "streaming"


def group_norm_ref(x, gamma, beta, groups, eps, silu, depth):
    """GroupNorm (+ SiLU) of x [n, h, w, c] NHWC with fp32 gamma / beta: (ref, bound) in fp64, see _norm_bound."""
    n, h, w, c = x.shape
    cpg = c // groups
    xd = x.double().reshape(n, h * w, groups, cpg)
    red = dict(dim=(1, 3), keepdim=True)
    mu = xd.mean(**red)
    var = ((xd - mu) ** 2).mean(**red)
    e2, am = (xd * xd).mean(**red), xd.abs().mean(**red)
    y, bound = _norm_bound(xd, mu, var, e2, am, gamma.double().reshape(groups, cpg), beta.double().reshape(groups, cpg),
                           eps, depth, silu, x.dtype)
    return y.reshape(n, h, w, c), bound.reshape(n, h, w, c)


def ln_depth(c):
    """Longest chain of fp32 additions behind a row's statistics in layer_norm_launch: layer_norm5 (C = 40 G, G lanes
    per row) sums 40 values per lane then log2 G shuffles; the generic kernel 8 per vector, ceil(C / 256) vectors per
    lane, then 5 shuffles. Returns (depth, "ln5" | "generic")."""
    if c in (320, 640, 1280):
        return 40 + int(math.log2(c // 40)), "ln5"
    return 8 * (-(-(c // 8) // 32)) + 5, "generic"


def ln_rows_per_block(c):
    """Rows one 256-thread block of layer_norm_launch covers: 8 warps x 32 / G rows (layer_norm5), else 8."""
    return 8 * (32 // (c // 40)) if c in (320, 640, 1280) else 8


def layer_norm_ref(x, gamma, beta, eps, depth):
    """LayerNorm over the last dim of x [rows, c] with fp32 gamma / beta: (ref, bound) in fp64, see _norm_bound."""
    xd = x.double()
    mu = xd.mean(-1, keepdim=True)
    var = ((xd - mu) ** 2).mean(-1, keepdim=True)
    e2, am = (xd * xd).mean(-1, keepdim=True), xd.abs().mean(-1, keepdim=True)
    return _norm_bound(xd, mu, var, e2, am, gamma.double(), beta.double(), eps, depth, False, x.dtype)


# ---- guards --------------------------------------------------------------------------------------------------------
SENTINEL = 0x7DB6  # 16-bit pattern of the output tails: a NaN payload in fp16, a large normal number in bf16


def moat(t: torch.Tensor, tail: int) -> torch.Tensor:
    """t copied to the start of a buffer whose next `tail` elements are NaN; returns the (contiguous) head. Fault: a
    read past the declared extent (a tensor map larger than the tensor, a missing p < p1 bound) meets NaN instead of
    TMA's zero fill or a neighbour's finite value, and check() rejects the non-finite output."""
    flat = torch.full((t.numel() + tail,), float("nan"), dtype=t.dtype, device=t.device)
    flat[:t.numel()] = t.reshape(-1)
    return flat[:t.numel()].view(t.shape)


def out_buffer(shape, tail: int, dtype, device):
    """(view, flat): an output of `shape` at the start of a buffer whose `tail` further elements hold SENTINEL."""
    n = math.prod(shape)
    flat = torch.full((n + tail,), SENTINEL, dtype=torch.int16, device=device).view(dtype)
    return flat[:n].view(shape), flat


def sentinel_intact(flat: torch.Tensor, n: int) -> bool:
    """Fault: a store past the last output element (a last row, tile or head written out of range)."""
    return bool((flat[n:].view(torch.int16) == SENTINEL).all())


def same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Fault: a result that depends on timing (an unordered reduction, a race): replayed CUDA graphs assume the same
    inputs give the same bits."""
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


# ---- inputs with planted values ------------------------------------------------------------------------------------
# Generated on the CPU from a seed, so that the GPU tests and their CPU negative controls see the same values.
def _randn(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g, dtype=torch.float64) * scale


def gemm_inputs(M, N, K, dtype, seed):
    """a [M, K], w [N, K], bias [N] (fp32), residual [M, N], with large values planted in A's last row, in A's and W's
    column K - 1, and in W's row N - 1. Faults: a ragged last M tile that drops or misplaces row M - 1, a ragged last
    k-block whose zero fill or tail is wrong (column K - 1), and a ragged last N tile that drops column N - 1."""
    a = _randn((M, K), seed)
    w = _randn((N, K), seed + 1, 1 / math.sqrt(K))
    a[M - 1] = 4.0 * torch.sign(a[M - 1]) + a[M - 1]
    a[:, K - 1] = 8.0
    w[:, K - 1] = 2.0 * torch.sign(w[:, K - 1]) + w[:, K - 1]
    w[N - 1] = 4.0 * torch.sign(w[N - 1]) / math.sqrt(K) + w[N - 1]
    bias = _randn((N,), seed + 2).float()
    res = _randn((M, N), seed + 3)
    return a.to(dtype), w.to(dtype), bias, res.to(dtype)


def conv_inputs(n, h, w, cin, cout, dtype, seed):
    """x [n, h, w, cin] NHWC, weight [cout, cin, 3, 3], bias [cout]: large pixels at every image's four corners and
    along its first and last row and column. Fault: an implicit-GEMM tile that spans several images reading a
    neighbour image's boundary row (or column) where the zero padding belongs; with large boundary pixels such a read
    moves every output next to the boundary by O(weight x pixel)."""
    x = _randn((n, h, w, cin), seed)
    for sl in ((slice(None), 0), (slice(None), h - 1), (slice(None), slice(None), 0), (slice(None), slice(None), w - 1)):
        x[sl] = x[sl] + 4.0 * torch.sign(x[sl])
    for yy in (0, h - 1):
        for xx in (0, w - 1):
            x[:, yy, xx] = 12.0 * torch.sign(x[:, yy, xx])
    wt = _randn((cout, cin, 3, 3), seed + 1, 1 / math.sqrt(9 * cin))
    return x.to(dtype), wt.to(dtype), _randn((cout,), seed + 2).float()


def attention_planted_keys(Nk):
    """The keys that attention_inputs plants: 63 and 64 (the two sides of the first KV block edge) and Nk - 1 (the
    ragged last block)."""
    return sorted({j for j in (63, 64, Nk - 1) if 0 <= j < Nk})


def attention_inputs(B, H, Nq, Nk, D, dtype, seed, scale=None):
    """q [B, H, Nq, D], k / v [B, H, Nk, D]. Every query of the first and last 128-row Q tiles has a strong component
    along one direction u, and the planted keys (attention_planted_keys) are 12 / scale along u: their scores
    dominate these rows (the other keys' scores stay O(1)), and they share the rows' weight about equally. Each planted
    key has a distinctive value vector of size 2-6 against O(1) random values. Faults: the last key of a ragged block
    dropped or mis-masked (a key past Nk let in, a valid one masked out), a key at the 63 | 64 block edge dropped or
    duplicated, and the first or last Q tile's rows taking another tile's result: each moves the affected rows by
    O(|v|)."""
    sc = float(scale) if scale is not None else D ** -0.5
    q = _randn((B, H, Nq, D), seed) * 0.5
    k = _randn((B, H, Nk, D), seed + 1)
    v = _randn((B, H, Nk, D), seed + 2)
    u = _randn((D,), seed + 3)
    u = u / u.norm()
    amp = math.sqrt(12.0 / sc)
    rows = sorted(set(range(min(128, Nq))) | set(range((Nq - 1) // 128 * 128, Nq)))
    q[:, :, rows] += amp * u
    sign = torch.tensor([(-1.0) ** d for d in range(D)], dtype=torch.float64)
    for t, j in enumerate(attention_planted_keys(Nk)):
        k[:, :, j] = amp * u + 0.05 * k[:, :, j]
        v[:, :, j] = 2.0 * (t + 1) * torch.roll(sign, t)
    return q.to(dtype), k.to(dtype), v.to(dtype)


def hypertile_first_rows(hp, wp, nh, nw):
    """Natural row of every tile's first token, tiles in tile-major (nh, nw) order."""
    th, tw = hp // nh, wp // nw
    return [(ih * th) * wp + iw * tw for ih in range(nh) for iw in range(nw)]


def hypertile_inputs(B, H, D, hp, wp, nh, nw, dtype, seed):
    """qkv [B, hp*wp, 3 H D] (q | k | v, heads contiguous): every query has a strong component along one direction u
    and every tile's first token (tile-major) has a key of 12 / scale along u and a value vector distinct per tile. In
    tile-major order, the first key of tile t + 1 directly follows tile t's last key: when tile t's token count is not
    a multiple of 64, it lies in the masked part of tile t's last KV block. Fault: a mask that lets it in gives it the
    same dominant score as tile t's own first key, moving tile t's rows by O(|v|)."""
    N = hp * wp
    sc = D ** -0.5
    qkv = _randn((B, N, 3, H, D), seed)
    qkv[:, :, 0] *= 0.5
    u = _randn((D,), seed + 1)
    u = u / u.norm()
    amp = math.sqrt(12.0 / sc)
    qkv[:, :, 0] += amp * u
    sign = torch.tensor([(-1.0) ** d for d in range(D)], dtype=torch.float64)
    for t, r in enumerate(hypertile_first_rows(hp, wp, nh, nw)):
        qkv[:, r, 1] = amp * u
        qkv[:, r, 2] = (2.0 + (t % 5)) * torch.roll(sign, t)
    return qkv.reshape(B, N, 3 * H * D).to(dtype)


def gn_inputs(n, h, w, c, dtype, seed, offset=0.0):
    """x [n, h, w, c] with a common offset of `offset` standard deviations, gamma, beta (fp32). The last image's last
    pixel (hw - 1) holds an outlier of sqrt(hw * c / 32) sigma in every channel, which carries about half of its
    groups' variance. Fault: statistics (or the apply pass) that drop or double the last pixel of a partial pixel
    chunk, which moves the whole last image's output by a large fraction of |gamma x^|."""
    x = _randn((n, h, w, c), seed) + offset
    x[n - 1, h - 1, w - 1] = offset + math.sqrt(h * w * c / 32) * torch.sign(_randn((c,), seed + 3))
    g = _randn((c,), seed + 1).float()
    b = _randn((c,), seed + 2).float()
    return x.to(dtype), g, b


def ln_inputs(rows, c, dtype, seed):
    """x [rows, c] (mean -1, std 3), gamma, beta (fp32), with an outlier of 4 sqrt(c) in the last channel of the last
    row. Fault: a row read or written one row off at a block edge, or a last row that loses its last vector."""
    x = _randn((rows, c), seed) * 3 - 1
    x[rows - 1, c - 1] = 4 * math.sqrt(c)
    return x.to(dtype), _randn((c,), seed + 1).float(), _randn((c,), seed + 2).float()
