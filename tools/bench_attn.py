"""Times the stand-alone attention entry (sdxe_attention) on the UNet's self-attention shapes.
  python tools/bench_attn.py [--dtype bf16] [--iters 20] [--dump DIR]
Prints us / launch, TFLOP/s (4*B*H*Nq*Nk*d) and rel-L2 error vs fp32 SDPA (first shapes only). --dump DIR saves each
shape's output (seeded inputs) as DIR/<shape>_<dtype>.npy, to compare two builds bit for bit."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import sdwebui_b200  # noqa: E402,F401
from sdwebui_b200 import ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--dtype", default="bf16")
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--shapes", default="sd15_l0,sd15_l1,sd15_l2,sdxl_l1,sdxl_l2,vae64")
ap.add_argument("--check", action="store_true")
ap.add_argument("--dump", metavar="DIR", default=None)
args = ap.parse_args()
dt = torch.bfloat16 if args.dtype == "bf16" else torch.float16
SHAPES = {  # B, H, Nq, Nk, d
    "sd15_l0": (16, 8, 4096, 4096, 40), "sd15_l1": (16, 8, 1024, 1024, 80), "sd15_l2": (16, 8, 256, 256, 160),
    "sdxl_l1": (8, 10, 4096, 4096, 64), "sdxl_l2": (8, 20, 1024, 1024, 64), "vae64": (8, 1, 4096, 4096, 512),
    "sd15_l0_b2": (2, 8, 4096, 4096, 40),
}
dev = torch.device("cuda:0")
for name in args.shapes.split(","):
    B, H, Nq, Nk, d = SHAPES[name]
    g = torch.Generator(device=dev).manual_seed(1)
    q = torch.randn(B, H, Nq, d, device=dev, dtype=dt, generator=g)
    k = torch.randn(B, H, Nk, d, device=dev, dtype=dt, generator=g)
    v = torch.randn(B, H, Nk, d, device=dev, dtype=dt, generator=g)
    for _ in range(3):
        o = ops.attention(q, k, v)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.iters):
        o = ops.attention(q, k, v)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1000.0 / args.iters
    fl = 4.0 * B * H * Nq * Nk * d
    msg = f"{name:10s} B{B} H{H} Nq{Nq} Nk{Nk} d{d}: {us:8.1f} us  {fl / us / 1e6:7.1f} TFLOP/s"
    if args.check:
        nb = min(B, 2)
        ref = torch.nn.functional.scaled_dot_product_attention(q[:nb].float(), k[:nb].float(), v[:nb].float())
        ref = ref.transpose(1, 2).reshape(nb, Nq, H * d)
        msg += f"  rel-L2 {((o[:nb].float() - ref).norm() / ref.norm()).item():.3e}"
    print(msg, flush=True)
    if args.dump:
        import numpy as np

        os.makedirs(args.dump, exist_ok=True)
        np.save(os.path.join(args.dump, f"{name}_{args.dtype}.npy"), o.view(torch.int16).cpu().numpy())
