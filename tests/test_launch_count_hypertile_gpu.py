"""sdxe_launch_count with Hypertile: for a UNet forward with tiled layers (the pre-op that writes the draw table, the
gather kernels, the segmented attention) and for sdxe_hypertile_attention, the counter's increase equals the number of
kernels torch.profiler records, as test_launch_count_gpu.py checks for every other entry point. Engine profiling is on,
so the plan runs op by op rather than as a graph replay."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_launch_count_gpu import _check  # noqa: E402

pytestmark = pytest.mark.gpu


def test_hypertile_attention(cuda):
    from sdwebui_b200 import lib as L

    lib = L.load()
    B, H, D, hp, wp = 2, 4, 64, 24, 40
    qkv = torch.randn(B, hp * wp, 3 * H * D, device=cuda).half()
    tiled, out = torch.empty_like(qkv), torch.empty(B, hp * wp, H * D, device=cuda, dtype=torch.float16)
    draw = torch.tensor([3, 5], dtype=torch.int32, device=cuda)
    _check(lambda: L.check(lib.sdxe_hypertile_attention(L.ptr(qkv), L.ptr(tiled), L.ptr(draw), L.ptr(out), B, H, hp, wp, D, 16,
                                                         0.125, L.SDXE_F16, L.current_stream()), "sdxe_hypertile_attention"),
           expect_min=2)


def test_unet_forward_hypertile(cuda):
    from oracle.synth import init_module_
    from oracle.unet import UNetModel, tiny_config
    from sdwebui_b200.engine import UNetEngine, UNetSpec
    from sdwebui_b200.hypertile import attn1_layers

    cfg = tiny_config()
    spec = UNetSpec.from_any(cfg)
    eng = UNetEngine(spec, dtype=torch.float16, device=cuda)
    eng.load_state_dict(init_module_(UNetModel(cfg), 1).state_dict())
    eng.finalize()
    rows = [(24, 40, 3, 5, 16) if level == 0 else (12, 20, 2, 2, 4) for _, level in attn1_layers(spec)]
    x = torch.randn(2, 4, 24, 40, device=cuda).half()
    t = torch.tensor([10.0, 500.0], device=cuda).half()
    ctx = torch.randn(2, 77, cfg.context_dim, device=cuda).half()
    eng.profile(True)
    _check(lambda: eng.forward(x, t, ctx, hypertile=rows), expect_min=2 * len(rows))
    eng.profile(False)
    eng.close()
