"""GPU parity tests of the stand-alone CUDA primitives, through the C-ABI (libsdxe.so), against plain PyTorch
fp32 references of the same op on the same seeded inputs. Tolerances are for 16-bit storage with fp32 accumulate."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


def _tol(dtype):
    return 2e-3 if dtype == torch.float16 else 1.6e-2


def _rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item(), (a - b).abs().max().item()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (256, 320, 320), (1000, 328, 200), (4096, 1280, 1280), (1232, 640, 768),
                                   (65536, 320, 320), (128, 2560, 640)])
def test_gemm_plain(cuda, dtype, M, N, K):
    from sdwebui_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = torch.randn(M, K, device=cuda, generator=g).to(dtype)
    w = (torch.randn(N, K, device=cuda, generator=g) / math.sqrt(K)).to(dtype)
    bias = torch.randn(N, device=cuda, generator=g)
    res = torch.randn(M, N, device=cuda, generator=g).to(dtype)
    out = ops.gemm(a, w, bias=bias, residual=res)
    ref = a.float() @ w.float().t() + bias + res.float()
    rel, mx = _rel_err(out, ref)
    assert rel < _tol(dtype), (rel, mx)


@pytest.mark.parametrize("bn", [16, 32, 48, 80, 96, 160, 256])
def test_gemm_tile_widths(cuda, bn):
    from sdwebui_b200 import ops

    dtype = torch.float16
    g = torch.Generator(device="cuda").manual_seed(bn)
    M, N, K = 640, 480, 448
    a = torch.randn(M, K, device=cuda, generator=g).to(dtype)
    w = (torch.randn(N, K, device=cuda, generator=g) / math.sqrt(K)).to(dtype)
    out = ops.gemm(a, w, force_bn=bn)
    ref = a.float() @ w.float().t()
    rel, mx = _rel_err(out, ref)
    assert rel < _tol(dtype), (bn, rel, mx)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,C", [(256, 64), (4096, 320), (1024, 1280)])
def test_gemm_geglu(cuda, dtype, M, C):
    from sdwebui_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(C)
    a = torch.randn(M, C, device=cuda, generator=g).to(dtype)
    w = (torch.randn(8 * C, C, device=cuda, generator=g) / math.sqrt(C)).to(dtype)
    bias = torch.randn(8 * C, device=cuda, generator=g)
    out = ops.gemm(a, w, bias=bias, geglu=True)
    proj = a.float() @ w.float().t() + bias
    val, gate = proj.chunk(2, dim=-1)
    ref = val * torch.nn.functional.gelu(gate)
    rel, mx = _rel_err(out, ref)
    assert rel < _tol(dtype) * 1.5, (rel, mx)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 8, 8, 64, 64), (1, 16, 16, 128, 320), (2, 32, 32, 64, 128), (3, 64, 64, 64, 32),
                                            (1, 128, 128, 64, 64), (2, 16, 8, 64, 64), (16, 8, 8, 1280, 1280), (1, 64, 64, 320, 320),
                                            (3, 8, 8, 128, 64),
                                            # tileable but not square: a partial last tile of several images, rows of 8
                                            # or 16 pixels, a W of two 128-pixel boxes
                                            (5, 8, 8, 64, 64), (2, 48, 16, 64, 128), (2, 24, 16, 320, 320), (1, 4, 256, 64, 64)])
def test_conv3x3(cuda, dtype, n, h, w, cin, cout):
    from sdwebui_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(n * h + cin)
    x = torch.randn(n, cin, h, w, device=cuda, generator=g).to(dtype)
    wt = (torch.randn(cout, cin, 3, 3, device=cuda, generator=g) / math.sqrt(9 * cin)).to(dtype)
    bias = torch.randn(cout, device=cuda, generator=g)
    out = ops.conv3x3_nhwc(x.permute(0, 2, 3, 1).contiguous(), wt, bias)
    ref = torch.nn.functional.conv2d(x.float(), wt.float(), bias, padding=1).permute(0, 2, 3, 1)
    rel, mx = _rel_err(out, ref)
    assert rel < _tol(dtype), (rel, mx)


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
    from sdwebui_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(Nq + Nk + D)
    q = torch.randn(B, H, Nq, D, device=cuda, generator=g).to(dtype)
    k = torch.randn(B, H, Nk, D, device=cuda, generator=g).to(dtype)
    v = torch.randn(B, H, Nk, D, device=cuda, generator=g).to(dtype)
    out = ops.attention(q, k, v)
    ref = torch.nn.functional.scaled_dot_product_attention(q.float(), k.float(), v.float())
    ref = ref.transpose(1, 2).reshape(B, Nq, H * D)
    rel, mx = _rel_err(out, ref)
    assert rel < _tol(dtype) * 1.5, (rel, mx)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,h,w,c,silu", [(2, 8, 8, 64, True), (3, 64, 64, 320, True), (2, 32, 32, 960, False), (1, 16, 16, 2560, True),
                                           (1, 256, 256, 128, True),
                                           # UNet levels of a 1216x832 image: streaming (hw * C/32 * 2 B > 48 KB) and
                                           # one-pass (the last, SD1.5's 13x19 level)
                                           (2, 104, 152, 320, True), (2, 52, 76, 640, False), (2, 26, 38, 1280, True),
                                           (4, 13, 19, 1280, False)])
def test_group_norm(cuda, dtype, n, h, w, c, silu):
    from sdwebui_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(c)
    x = (torch.randn(n, h, w, c, device=cuda, generator=g) * 2 + 0.5).to(dtype)
    gamma = torch.randn(c, device=cuda, generator=g)
    beta = torch.randn(c, device=cuda, generator=g)
    out = ops.group_norm_nhwc(x, gamma, beta, 32, 1e-5, silu)
    ref = torch.nn.functional.group_norm(x.float().permute(0, 3, 1, 2), 32, gamma, beta, 1e-5)
    if silu:
        ref = torch.nn.functional.silu(ref)
    ref = ref.permute(0, 2, 3, 1)
    rel, mx = _rel_err(out, ref)
    assert rel < _tol(dtype), (rel, mx)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows,c", [(7, 64), (4096, 320), (1024, 1280)])
def test_layer_norm(cuda, dtype, rows, c):
    from sdwebui_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(c)
    x = (torch.randn(rows, c, device=cuda, generator=g) * 3 - 1).to(dtype)
    gamma = torch.randn(c, device=cuda, generator=g)
    beta = torch.randn(c, device=cuda, generator=g)
    out = ops.layer_norm(x, gamma, beta)
    ref = torch.nn.functional.layer_norm(x.float(), (c,), gamma, beta, 1e-5)
    rel, mx = _rel_err(out, ref)
    assert rel < _tol(dtype), (rel, mx)
