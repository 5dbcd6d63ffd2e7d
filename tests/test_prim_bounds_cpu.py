"""Negative controls for tests/prim_bounds.py, without a GPU: a CPU emulation of each kernel's rounding (fp32
accumulation and statistics, P rounded to 16 bit in attention, output rounded to 16 bit) passes the per-element bound
on the planted inputs the GPU tests use, and the same emulation with one simulated fault fails it. This is what shows
that the GPU tests in test_prims_gpu.py and test_hypertile_gpu.py would catch a subtly wrong kernel. Shapes are the
GPU tests' edge shapes, reduced where CPU time requires it."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import hypertile_oracle as HO  # noqa: E402
import prim_bounds as PB  # noqa: E402

DTYPES = [torch.float16, torch.bfloat16]
LOG2E = 1.4426950408889634


def _fails(what, out, ref, bound):
    with pytest.raises(AssertionError):
        PB.check(what, out, ref, bound)


# ---- emulations ------------------------------------------------------------------------------------------------------
def gemm_emul(a, w, bias=None, res=None):
    acc = a.float() @ w.float().t()
    if bias is not None:
        acc = acc + bias
    if res is not None:
        acc = acc + res.float()
    return acc.to(a.dtype)


def conv_emul(x, w, bias, neighbour_row=False):
    """fp32 implicit GEMM; neighbour_row: image i > 0 reads image i - 1's last row as its top padding row."""
    xp = F.pad(x.float().permute(0, 3, 1, 2), (1, 1, 1, 1))
    if neighbour_row:
        xp[1:, :, 0, 1:-1] = x.float().permute(0, 3, 1, 2)[:-1, :, -1]
    return (F.conv2d(xp, w.float(), bias).permute(0, 2, 3, 1)).to(x.dtype)


def attention_emul(q, k, v, scale=None):
    """[B, H, Nq, D] -> [B, Nq, H * D]: fp32 scores, p = 2^((s - m) sl2), l from the fp32 p, P V with 16-bit P."""
    B, H, Nq, D = q.shape
    sl2 = (float(scale) if scale is not None else D ** -0.5) * LOG2E
    s = q.float() @ k.float().transpose(-1, -2)
    m = s.amax(-1, keepdim=True)
    p = torch.exp2(s * sl2 - m * sl2)
    o = (p.to(q.dtype).float() @ v.float()) / p.sum(-1, keepdim=True)
    return o.to(q.dtype).transpose(1, 2).reshape(B, Nq, H * D)


def hypertile_emul(qkv, H, D, hp, wp, nh, nw, leak=False):
    """Tile-local attention; leak: tile t also sees tile t + 1's first key (a mask that lets in a key past T)."""
    q, k, v = (HO.regroup(t, hp, wp, nh, nw) for t in qkv.split(H * D, dim=-1))
    bt, T, _ = q.shape
    q, k, v = (t.reshape(bt, T, H, D).transpose(1, 2) for t in (q, k, v))
    nt = nh * nw
    outs = []
    for i in range(bt):
        kk, vv = k[i:i + 1], v[i:i + 1]
        if leak and (i % nt) + 1 < nt:
            kk, vv = torch.cat([kk, k[i + 1:i + 2, :, :1]], 2), torch.cat([vv, v[i + 1:i + 2, :, :1]], 2)
        outs.append(attention_emul(q[i:i + 1], kk, vv))
    return HO.ungroup(torch.cat(outs), hp, wp, nh, nw)


def hypertile_ref(qkv, H, D, hp, wp, nh, nw):
    q, k, v = (HO.regroup(t, hp, wp, nh, nw) for t in qkv.split(H * D, dim=-1))
    bt, T, _ = q.shape
    ref, bound = PB.attention_ref(*(t.reshape(bt, T, H, D).transpose(1, 2) for t in (q, k, v)))
    return HO.ungroup(ref, hp, wp, nh, nw), HO.ungroup(bound, hp, wp, nh, nw)


def gn_emul(x, gamma, beta, groups, eps, silu, centred, skip_last=False):
    """fp32 statistics (centred second pass, or the streaming E[x^2] - mu^2); skip_last: the statistics miss pixel
    hw - 1."""
    n, h, w, c = x.shape
    xs = x.float().reshape(n, h * w, groups, c // groups)
    st = xs[:, :-1] if skip_last else xs
    mu = st.mean((1, 3), keepdim=True)
    var = ((st - mu) ** 2).mean((1, 3), keepdim=True) if centred else ((st * st).mean((1, 3), keepdim=True) - mu * mu)
    y = (xs - mu) * torch.rsqrt(var + eps) * gamma.reshape(groups, -1) + beta.reshape(groups, -1)
    if silu:
        y = F.silu(y)
    return y.reshape(n, h, w, c).to(x.dtype)


def ln_emul(x, gamma, beta, eps, shift_from=None):
    """fp32 two-pass LayerNorm; shift_from: rows from that block edge on are written one row late."""
    y = F.layer_norm(x.float(), (x.shape[-1],), gamma, beta, eps).to(x.dtype)
    if shift_from is not None:
        y[shift_from + 1:] = y[shift_from:-1].clone()
    return y


# ---- GEMM ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,N,K", [(129, 24, 72), (127, 264, 200), (1, 8, 8), (4097, 40, 2056)])
def test_gemm_emulation_and_faults(dtype, M, N, K):
    """The fp32-accumulating emulation passes; ignoring A's last row (a ragged last M tile) or column K - 1 (a ragged
    last k-block) fails."""
    a, w, bias, res = PB.gemm_inputs(M, N, K, dtype, 7)
    ref, bound = PB.gemm_ref(a, w, bias, res)
    PB.check("gemm emulation", gemm_emul(a, w, bias, res), ref, bound)
    a_row = a.clone()
    a_row[M - 1] = 0
    _fails("last row ignored", gemm_emul(a_row, w, bias, res), ref, bound)
    a_col = a.clone()
    a_col[:, K - 1] = 0
    _fails("column K-1 ignored", gemm_emul(a_col, w, bias, res), ref, bound)
    w_row = w.clone()
    w_row[N - 1] = 0
    _fails("W row N-1 ignored", gemm_emul(a, w_row, bias, res), ref, bound)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bias", [True, False])
def test_geglu_emulation_and_fault(dtype, bias):
    """fp32 projection and exact-erf GELU pass; a gate column taken from the wrong half fails."""
    M, C = 129, 64
    a, w, b, _ = PB.gemm_inputs(M, 8 * C, C, dtype, 11)
    b = b if bias else None
    ref, bound = PB.geglu_ref(a, w, b)
    proj = a.float() @ w.float().t() + (b if bias else 0)
    val, gate = proj.chunk(2, dim=-1)
    PB.check("geglu emulation", (val * F.gelu(gate)).to(dtype), ref, bound)
    _fails("geglu last K column ignored",
           ((a.float()[:, :-1] @ w.float()[:, :-1].t() + (b if bias else 0)).chunk(2, -1)[0] * F.gelu(gate)).to(dtype),
           ref, bound)


# ---- conv ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,h,w", [(5, 8, 8), (3, 8, 8), (2, 16, 8)])
def test_conv_emulation_and_fault(dtype, n, h, w):
    """Zero-padded fp32 conv passes; a neighbour image's last row read as top padding (a tile spanning images) fails."""
    x, wt, b = PB.conv_inputs(n, h, w, 64, 32, dtype, 5)
    ref, bound = PB.conv3x3_ref(x, wt, b)
    PB.check("conv emulation", conv_emul(x, wt, b), ref, bound)
    _fails("neighbour row as padding", conv_emul(x, wt, b, neighbour_row=True), ref, bound)


# ---- attention -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Nq,Nk,D,scale", [(129, 65, 40, None), (1, 63, 8, None), (129, 1, 48, None), (257, 130, 80, None),
                                           (129, 65, 64, 0.3), (4097, 65, 8, None)])
def test_attention_emulation_and_faults(dtype, Nq, Nk, D, scale):
    """fp32 softmax with 16-bit P passes; dropping the last key (ragged last KV block), or key 64 (the block edge), or
    letting in one key past Nk fails."""
    q, k, v = PB.attention_inputs(1, 2, Nq, Nk, D, dtype, 3, scale)
    ref, bound = PB.attention_ref(q, k, v, scale)
    PB.check("attention emulation", attention_emul(q, k, v, scale), ref, bound)
    if Nk > 1:
        _fails("last key dropped", attention_emul(q, k[:, :, :-1], v[:, :, :-1], scale), ref, bound)
    if Nk > 64:
        keep = [j for j in range(Nk) if j != 64]
        _fails("key 64 dropped", attention_emul(q, k[:, :, keep], v[:, :, keep], scale), ref, bound)
    # a key past Nk that the mask lets in: the next planted-like key (what a neighbour head or tile would hold)
    q2, k2, v2 = PB.attention_inputs(1, 2, Nq, Nk + 1, D, dtype, 3, scale)
    k_in = torch.cat([k, k2[:, :, -1:]], 2)
    v_in = torch.cat([v, v2[:, :, -1:] * -1], 2)
    _fails("key past Nk let in", attention_emul(q, k_in, v_in, scale), ref, bound)


def test_attention_bound_is_not_vacuous():
    """The bound at a long sequence stays far below the planted values' effect (a third of |v| ~ 1)."""
    q, k, v = PB.attention_inputs(1, 1, 129, 4097, 64, torch.float16, 3)
    _, bound = PB.attention_ref(q, k, v)
    assert float(bound.max()) < 0.05


# ---- Hypertile -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", [(1, 2, 40, 12, 30, 2, 3), (1, 1, 64, 26, 20, 2, 2), (1, 2, 40, 13, 10, 1, 2)],
                         ids=lambda c: "B{}H{}d{}_{}x{}_{}x{}".format(*c))
def test_hypertile_emulation_and_fault(dtype, case):
    """Tile-local emulation passes; the next tile's first key leaking into a tile (a failed mask on the ragged last KV
    block) fails."""
    B, H, D, hp, wp, nh, nw = case
    qkv = PB.hypertile_inputs(B, H, D, hp, wp, nh, nw, dtype, 3)
    ref, bound = hypertile_ref(qkv, H, D, hp, wp, nh, nw)
    PB.check("hypertile emulation", hypertile_emul(qkv, H, D, hp, wp, nh, nw), ref, bound)
    _fails("next tile's first key leaks", hypertile_emul(qkv, H, D, hp, wp, nh, nw, leak=True), ref, bound)


# ---- GroupNorm -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,h,w,c,silu,offset", [(1, 39, 63, 320, True, 8.0), (1, 2, 1229, 320, False, 8.0),
                                                  (2, 26, 38, 1280, True, 0.0), (2, 52, 76, 640, False, 8.0)])
def test_group_norm_emulation_and_fault(dtype, n, h, w, c, silu, offset):
    """Centred (one-pass) and uncentred (streaming) fp32 statistics pass, at an offset of 8 sigma too; statistics that
    skip the last pixel fail."""
    x, g, b = PB.gn_inputs(n, h, w, c, dtype, 9, offset)
    depth, _ = PB.gn_depth(n, h * w, c)
    ref, bound = PB.group_norm_ref(x, g, b, 32, 1e-5, silu, depth)
    for centred in (True, False):
        PB.check(f"group norm emulation centred={centred}", gn_emul(x, g, b, 32, 1e-5, silu, centred), ref, bound)
    _fails("last pixel skipped", gn_emul(x, g, b, 32, 1e-5, silu, False, skip_last=True), ref, bound)


# ---- LayerNorm -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows,c", [(33, 320), (4097, 640), (33, 1280), (31, 8), (33, 264), (33, 768), (33, 2048)])
def test_layer_norm_emulation_and_fault(dtype, rows, c):
    """fp32 two-pass statistics pass; rows written one row late from the last block edge on fail."""
    x, g, b = PB.ln_inputs(rows, c, dtype, 13)
    depth, _ = PB.ln_depth(c)
    ref, bound = PB.layer_norm_ref(x, g, b, 1e-5, depth)
    PB.check("layer norm emulation", ln_emul(x, g, b, 1e-5), ref, bound)
    edge = (rows - 1) // PB.ln_rows_per_block(c) * PB.ln_rows_per_block(c)
    _fails("rows shifted at a block edge", ln_emul(x, g, b, 1e-5, shift_from=max(edge - 1, 0)), ref, bound)


# ---- guards ----------------------------------------------------------------------------------------------------------
def test_guards_catch_their_faults():
    """A NaN read from a moat fails check(); a store into the sentinel tail and a one-ulp difference between two calls
    are both seen."""
    x = torch.randn(16, 8).half()
    m = PB.moat(x, 32)
    flat = m.untyped_storage()
    assert torch.isnan(torch.tensor([], dtype=torch.float16).set_(flat, 16 * 8, (32,))).all()
    ref, bound = x.double(), PB.ulp16(x.double(), torch.float16)
    PB.check("identity", m, ref, bound)
    bad = m.clone()
    bad[15, 7] = float("nan")
    _fails("NaN from a moat", bad, ref, bound)
    out, oflat = PB.out_buffer((16, 8), 64, torch.bfloat16, "cpu")
    out.fill_(1.0)
    assert PB.sentinel_intact(oflat, 128)
    oflat[128] = 0
    assert not PB.sentinel_intact(oflat, 128)
    y = out.clone()
    y.view(torch.int16)[3, 3] += 1
    assert PB.same_bits(out, out.clone()) and not PB.same_bits(out, y)
