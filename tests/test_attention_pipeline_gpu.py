"""GPU parity of the flash-attention kernel on the paths its per-warpgroup pipeline and head-dim-sized MMAs add, against
fp32 scaled_dot_product_attention on the same seeded inputs (same tolerance as test_prims_gpu.test_attention)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


def _tol(dtype):
    return 2e-3 if dtype == torch.float16 else 1.6e-2


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,H,Nq,Nk,D", [
    # self-attention at d = 80: the second value slab runs O += P V at n16, QK^T at 5 k16 steps
    (2, 8, 1024, 1024, 80),
    # d = 512 (8 K slabs, four value passes) with two key blocks, the second holding a single key: the prologue and the
    # last pipelined step back to back, with the largest number of K slabs in flight
    (1, 1, 128, 65, 512),
])
def test_attention_pipeline(cuda, dtype, B, H, Nq, Nk, D):
    from sdwebui_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(Nq + Nk + D)
    q = torch.randn(B, H, Nq, D, device=cuda, generator=g).to(dtype)
    k = torch.randn(B, H, Nk, D, device=cuda, generator=g).to(dtype)
    v = torch.randn(B, H, Nk, D, device=cuda, generator=g).to(dtype)
    out = ops.attention(q, k, v)
    ref = torch.nn.functional.scaled_dot_product_attention(q.float(), k.float(), v.float())
    ref = ref.transpose(1, 2).reshape(B, Nq, H * D)
    o = out.float()
    rel = ((o - ref).norm() / (ref.norm() + 1e-12)).item()
    assert rel < _tol(dtype) * 1.5, (rel, (o - ref).abs().max().item())
