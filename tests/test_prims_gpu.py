"""GPU tests of the stand-alone CUDA primitives through the C-ABI (libsdxe.so), element by element against fp64
references of the same op on the same 16-bit inputs (tests/prim_bounds.py derives each bound from what the kernel
does). Every input carries planted values aimed at one tile-edge fault (see the input generators' docstrings), sits
at the start of a buffer with a NaN tail at least one tile long, and every output is followed by a sentinel tail that
must come back unchanged; each call runs twice and must give the same bits."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import prim_bounds as PB  # noqa: E402

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


def _dt(dtype):
    return "fp16" if dtype == torch.float16 else "bf16"


def _twice(call, out, flat):
    """Run call() twice into `out`: the second call must give the same bits, and the sentinel tail after `out` must be
    untouched. Returns the first result."""
    call()
    first = out.clone()
    call()
    torch.cuda.synchronize()
    assert PB.same_bits(first, out), "second call gave different bits"
    assert PB.sentinel_intact(flat, out.numel()), "store past the end of the output"
    return first


def _gemm(dev, a, w, bias, res, geglu=False):
    from sdwebui_b200 import lib as L

    M, K = a.shape
    N = w.shape[0]
    a, w = PB.moat(a.to(dev), 128 * K), PB.moat(w.to(dev), 256 * K)
    bias = PB.moat(bias.to(dev), 256) if bias is not None else None
    res = PB.moat(res.to(dev), 128 * N) if res is not None else None
    out, flat = PB.out_buffer((M, N // 2 if geglu else N), 128 * N, a.dtype, dev)
    lib = L.load()
    out = _twice(lambda: L.check(lib.sdxe_gemm(L.ptr(a), L.ptr(w), L.ptr(out), M, N, K, L.ptr(bias), L.ptr(res),
                                               1 if geglu else 0, L.torch_dtype_code(a.dtype), L.current_stream()),
                                 "sdxe_gemm"), out, flat)
    return out, (a, w, bias, res)


def _gemm_where(idx):
    m, n = idx
    return f"M tile {m // 128} row {m % 128}, column {n} (16-wide N tile {n // 16})"


def _check_gemm(cuda, dtype, M, N, K, bias=True, residual=True, seed=0):
    a, w, b, r = PB.gemm_inputs(M, N, K, dtype, seed)
    out, (a, w, b, r) = _gemm(cuda, a, w, b if bias else None, r if residual else None)
    ref, bound = PB.gemm_ref(a, w, b, r)
    PB.check(f"gemm {_dt(dtype)} M={M} N={N} K={K} bias={bias} res={residual}", out, ref, bound, _gemm_where)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (256, 320, 320), (1000, 328, 200), (4096, 1280, 1280), (1232, 640, 768),
                                   (65536, 320, 320), (128, 2560, 640)])
def test_gemm_plain(cuda, dtype, M, N, K):
    _check_gemm(cuda, dtype, M, N, K, seed=M + N + K)


GEMM_EDGES = [(M, N, K) for M in (1, 127, 129, 4097) for N in (8, 24, 40, 264) for K in (8, 72, 200, 2056)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,N,K", GEMM_EDGES)
def test_gemm_edges(cuda, dtype, M, N, K):
    """Ragged last M tile (127, 129, 4097 rows, and a single row), N % 16 == 8 (a half-empty last column tile), K < 64
    and K % 64 != 0 (TMA zero fill of the last k-block), with the four bias / residual combinations in turn."""
    i = GEMM_EDGES.index((M, N, K))
    _check_gemm(cuda, dtype, M, N, K, bias=i % 2 == 0, residual=(i // 2) % 2 == 0, seed=i)


@pytest.mark.parametrize("bn", [16, 32, 48, 80, 96, 160, 256])
def test_gemm_tile_widths(cuda, bn):
    """Every forced tile width through the ops.gemm wrapper, with A's last row and column K - 1 planted."""
    from sdwebui_b200 import ops

    dtype = torch.float16
    M, N, K = 640, 480, 448
    a, w, _, _ = PB.gemm_inputs(M, N, K, dtype, bn)
    a, w = a.to(cuda), w.to(cuda)
    out = ops.gemm(a, w, force_bn=bn)
    ref, bound = PB.gemm_ref(a, w)
    PB.check(f"gemm fp16 BN={bn}", out, ref, bound, _gemm_where)


def _check_geglu(cuda, dtype, M, C, bias):
    a, w, b, _ = PB.gemm_inputs(M, 8 * C, C, dtype, C)
    out, (a, w, b, _) = _gemm(cuda, a, w, b if bias else None, None, geglu=True)
    ref, bound = PB.geglu_ref(a, w, b)
    PB.check(f"geglu {_dt(dtype)} M={M} C={C} bias={bias}", out, ref, bound, _gemm_where)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,C", [(256, 64), (4096, 320), (1024, 1280)])
def test_gemm_geglu(cuda, dtype, M, C):
    _check_geglu(cuda, dtype, M, C, True)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,C", [(129, 64), (4097, 320)])
def test_gemm_geglu_no_bias(cuda, dtype, M, C):
    _check_geglu(cuda, dtype, M, C, False)


def test_gemm_geglu_untileable(cuda):
    """GEGLU needs a tile width BN % 32 == 0 that divides N; N = 48 has none, and the call must fail, not run."""
    from sdwebui_b200 import lib as L
    from sdwebui_b200 import ops

    a = torch.randn(64, 64, device=cuda).half()
    w = torch.randn(48, 64, device=cuda).half()
    with pytest.raises(L.SdxeError, match="geglu"):
        ops.gemm(a, w, geglu=True)


# ---- conv --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 8, 8, 64, 64), (1, 16, 16, 128, 320), (2, 32, 32, 64, 128), (3, 64, 64, 64, 32),
                                            (1, 128, 128, 64, 64), (2, 16, 8, 64, 64), (16, 8, 8, 1280, 1280), (1, 64, 64, 320, 320),
                                            (3, 8, 8, 128, 64),
                                            # tileable but not square: a partial last tile of several images, rows of 8
                                            # or 16 pixels, a W of two 128-pixel boxes
                                            (5, 8, 8, 64, 64), (2, 48, 16, 64, 128), (2, 24, 16, 320, 320), (1, 4, 256, 64, 64)])
def test_conv3x3(cuda, dtype, n, h, w, cin, cout):
    """Large pixels on every image's corners and borders: the multi-image tiles (W = 8 and 16) put a neighbour
    image's border next to each padding row."""
    from sdwebui_b200 import lib as L

    x, wt, b = PB.conv_inputs(n, h, w, cin, cout, dtype, n * h + cin)
    x, wt, b = PB.moat(x.to(cuda), 128 * cin), wt.to(cuda), b.to(cuda)
    wp = PB.moat(wt.permute(0, 2, 3, 1).reshape(cout, 9 * cin), 256 * 9 * cin)
    out, flat = PB.out_buffer((n, h, w, cout), 128 * cout, dtype, cuda)
    lib = L.load()
    out = _twice(lambda: L.check(lib.sdxe_conv3x3_nhwc(L.ptr(x), L.ptr(wp), L.ptr(out), n, h, w, cin, cout, L.ptr(b),
                                                       L.torch_dtype_code(dtype), L.current_stream()),
                                 "sdxe_conv3x3_nhwc"), out, flat)
    ref, bound = PB.conv3x3_ref(x, wt, b)

    def where(i):
        m = (i[0] * h + i[1]) * w + i[2]
        return f"image {i[0]} pixel ({i[1]}, {i[2]}), M tile {m // 128} row {m % 128}, channel {i[3]}"

    PB.check(f"conv3x3 {_dt(dtype)} {n}x{h}x{w} {cin}->{cout}", out, ref, bound, where)


# ---- attention ---------------------------------------------------------------------------------------------------
def _check_attention(cuda, dtype, B, H, Nq, Nk, D, scale=None):
    from sdwebui_b200 import lib as L

    q, k, v = PB.attention_inputs(B, H, Nq, Nk, D, dtype, Nq + Nk + D, scale)
    q, k, v = PB.moat(q.to(cuda), 128 * D), PB.moat(k.to(cuda), 64 * D), PB.moat(v.to(cuda), 64 * D)
    out, flat = PB.out_buffer((B, Nq, H * D), 128 * H * D, dtype, cuda)
    sc = float(scale) if scale is not None else D ** -0.5
    lib = L.load()
    out = _twice(lambda: L.check(lib.sdxe_attention(L.ptr(q), L.ptr(k), L.ptr(v), L.ptr(out), B, H, Nq, Nk, D, sc,
                                                    L.torch_dtype_code(dtype), L.current_stream()), "sdxe_attention"),
                 out, flat)
    ref, bound = PB.attention_ref(q, k, v, sc)
    nblk = (Nk + 63) // 64

    def where(i):
        return (f"batch {i[0]} head {i[2] // D} column {i[2] % D}, Q tile {i[1] // 128} row {i[1] % 128}; "
                f"{nblk} KV blocks, the last holding {Nk - 64 * (nblk - 1)} keys")

    PB.check(f"attention {_dt(dtype)} B={B} H={H} Nq={Nq} Nk={Nk} D={D} scale={sc:.4g}", out, ref, bound, where)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,H,Nq,Nk,D", [
    (1, 1, 128, 128, 64), (2, 2, 256, 256, 64), (2, 8, 1024, 1024, 40), (1, 8, 4096, 4096, 40), (2, 8, 1024, 77, 80),
    (2, 8, 256, 256, 160), (2, 8, 64, 64, 160), (2, 8, 64, 77, 160), (1, 10, 4096, 154, 64), (1, 20, 1024, 1024, 64),
    (1, 1, 1024, 1024, 512), (1, 1, 4096, 4096, 512), (1, 2, 200, 333, 64), (1, 1, 128, 300, 128),
    # short-KV persistent kernel (Nk <= 128, D <= 64): more items than SMs, ragged Nq, every key-count class
    (2, 8, 4096, 77, 40), (2, 10, 1024, 77, 64), (1, 3, 200, 77, 40), (1, 2, 128, 128, 64), (1, 2, 384, 100, 48),
    (1, 1, 64, 16, 8), (3, 5, 130, 1, 32), (16, 8, 4096, 77, 40),
    # ragged last KV blocks: SDXL's UNet at 1216x832 (3952 and 988 tokens), SD1.5's first level at 768x512 (6144), and
    # the VAE mid-block at 1216x832 (15808 tokens, d = 512 in four value passes)
    (2, 10, 3952, 3952, 64), (2, 20, 988, 988, 64), (2, 10, 3952, 77, 64), (2, 8, 6144, 6144, 40), (1, 1, 15808, 15808, 512),
])
def test_attention(cuda, dtype, B, H, Nq, Nk, D):
    _check_attention(cuda, dtype, B, H, Nq, Nk, D)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [8, 40, 48, 80, 160, 512])
@pytest.mark.parametrize("Nq", [1, 129, 4097])
@pytest.mark.parametrize("Nk", [1, 63, 65, 4097])
def test_attention_edges(cuda, dtype, Nk, Nq, D):
    """A single key, one key short of a block, one key into the next block and a ragged last block after 64 full
    ones, against a single query, a ragged second Q tile and a ragged 33rd, at every head-dim class (the 40 / 80 / 160
    kernels that skip padding, and the generic one at 8, 48 and 512 in four value passes)."""
    _check_attention(cuda, dtype, 1, 2, Nq, Nk, D)


@pytest.mark.parametrize("dtype", DTYPES)
def test_attention_scale(cuda, dtype):
    """A scale other than D^-0.5, through the ops.attention wrapper."""
    from sdwebui_b200 import ops

    q, k, v = PB.attention_inputs(2, 3, 129, 65, 64, dtype, 1, 0.3)
    q, k, v = q.to(cuda), k.to(cuda), v.to(cuda)
    out = ops.attention(q, k, v, scale=0.3)
    ref, bound = PB.attention_ref(q, k, v, 0.3)
    PB.check(f"attention {_dt(dtype)} scale=0.3", out, ref, bound)


# ---- GroupNorm ---------------------------------------------------------------------------------------------------
def _check_group_norm(cuda, dtype, n, h, w, c, silu, offset):
    from sdwebui_b200 import lib as L

    x, g, b = PB.gn_inputs(n, h, w, c, dtype, c + h, offset)
    x, g, b = PB.moat(x.to(cuda), 128 * c), g.to(cuda), b.to(cuda)
    out, flat = PB.out_buffer((n, h, w, c), 128 * c, dtype, cuda)
    lib = L.load()
    out = _twice(lambda: L.check(lib.sdxe_group_norm_nhwc(L.ptr(x), L.ptr(g), L.ptr(b), L.ptr(out), n, h * w, c, 32, 1e-5,
                                                          1 if silu else 0, L.torch_dtype_code(dtype), L.current_stream()),
                                 "sdxe_group_norm_nhwc"), out, flat)
    depth, path = PB.gn_depth(n, h * w, c, 32, torch.cuda.get_device_properties(cuda).multi_processor_count)
    ref, bound = PB.group_norm_ref(x, g, b, 32, 1e-5, silu, depth)

    def where(i):
        return f"{path} path, image {i[0]} pixel {i[1] * w + i[2]} of {h * w}, group {i[3] // (c // 32)}"

    PB.check(f"group norm {_dt(dtype)} {n}x{h}x{w}x{c} silu={silu} offset={offset} ({path})", out, ref, bound, where)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,h,w,c,silu", [(2, 8, 8, 64, True), (3, 64, 64, 320, True), (2, 32, 32, 960, False), (1, 16, 16, 2560, True),
                                           (1, 256, 256, 128, True),
                                           # UNet levels of a 1216x832 image: streaming (hw * C/32 * 2 B > 48 KB) and
                                           # one-pass (the last, SD1.5's 13x19 level)
                                           (2, 104, 152, 320, True), (2, 52, 76, 640, False), (2, 26, 38, 1280, True),
                                           (4, 13, 19, 1280, False)])
def test_group_norm(cuda, dtype, n, h, w, c, silu):
    _check_group_norm(cuda, dtype, n, h, w, c, silu, 0.25)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("offset", [0.0, 8.0])
@pytest.mark.parametrize("n,h,w,c,silu", [(1, 39, 63, 320, True), (1, 2, 1229, 320, False), (2, 13, 19, 1280, True),
                                           (2, 26, 38, 1280, False), (2, 104, 152, 320, True)])
def test_group_norm_crossover(cuda, dtype, n, h, w, c, silu, offset):
    """Both sides of the one-pass / streaming crossover at a 48 KB strip (2457 pixels x 10 channels x 2 B is the
    largest one-pass strip, 2458 the smallest streaming one, with a partial last pixel chunk), and a common offset of 8
    sigma, where the streaming path's uncentred E[x^2] - mu^2 loses the most."""
    _check_group_norm(cuda, dtype, n, h, w, c, silu, offset)


# ---- LayerNorm ---------------------------------------------------------------------------------------------------
def _check_layer_norm(cuda, dtype, rows, c):
    from sdwebui_b200 import lib as L

    x, g, b = PB.ln_inputs(rows, c, dtype, c + rows)
    x, g, b = PB.moat(x.to(cuda), 128 * c), g.to(cuda), b.to(cuda)
    out, flat = PB.out_buffer((rows, c), 128 * c, dtype, cuda)
    lib = L.load()
    out = _twice(lambda: L.check(lib.sdxe_layer_norm(L.ptr(x), L.ptr(g), L.ptr(b), L.ptr(out), rows, c, 1e-5,
                                                     L.torch_dtype_code(dtype), L.current_stream()), "sdxe_layer_norm"),
                 out, flat)
    depth, path = PB.ln_depth(c)
    rpb = PB.ln_rows_per_block(c)
    ref, bound = PB.layer_norm_ref(x, g, b, 1e-5, depth)
    PB.check(f"layer norm {_dt(dtype)} rows={rows} C={c} ({path})", out, ref, bound,
             lambda i: f"{path} kernel, row {i[0]} (block {i[0] // rpb} of {rpb} rows), channel {i[1]}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows,c", [(7, 64), (4096, 320), (1024, 1280)])
def test_layer_norm(cuda, dtype, rows, c):
    _check_layer_norm(cuda, dtype, rows, c)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows", [1, 31, 33, 4097])
@pytest.mark.parametrize("c", [320, 640, 1280, 8, 264, 768, 2048])
def test_layer_norm_edges(cuda, dtype, c, rows):
    """layer_norm5 (C = 320 / 640 / 1280) and the generic kernel (C = 8, 264, CLIP's 768, and its limit 2048) with a
    partial last block, whose rows past the end the `ok` guard keeps out."""
    _check_layer_norm(cuda, dtype, rows, c)
