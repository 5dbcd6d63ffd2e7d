"""Tiling (circular padding) off vs on, per engine call, bf16, synthetic weights:

  sd15_unet   SD1.5 UNet forward, CFG batch 2B = 16, 64 x 64 latent (512 x 512)
  sdxl_unet   SDXL UNet forward, 2B = 8, 128 x 128 latent (1024 x 1024)
  vae_decode  VAE decode of B = 8 latents to 512 x 512

    python tools/bench_tiling.py [--calls 20] [--reps 5] [--out results/bench_tiling.json]

After one warm-up call per setting, `reps` rounds alternate off / on; a round times `calls` back-to-back calls with a CUDA
event pair. Reported per setting: the median ms per call over the rounds (and every round). From one separate
engine-profiled call per setting (per-op CUDA events, SDXE_PROFILE_DUMP): the time of the circular-halo copies
("circpad") and of the circular im2col gathers, i.e. the launches Tiling adds. One JSON line, with the card's name and
power limit read in the same run."""
import argparse
import json
import os
import statistics
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _added_ms(dump_path):
    """ms of the ops Tiling adds (halo copies, circular im2col) in one profiled call."""
    ms = {"circpad": 0.0, "im2col": 0.0}
    for line in open(dump_path):
        _, _, desc, us = line.split(",")[:4]
        words = desc.split()
        if words and words[0] in ms and (words[0] == "circpad" or "circ=1" in words):
            ms[words[0]] += float(us) / 1000.0
    return {k: round(v, 3) for k, v in ms.items()}


def _time(eng, call, calls, reps):
    for circ in (False, True):
        eng.set_circular(circ)
        call()  # plan build + graph capture of this setting
    torch.cuda.synchronize()
    rounds = {False: [], True: []}
    for _ in range(reps):
        for circ in (False, True):
            eng.set_circular(circ)
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(calls):
                call()
            b.record()
            b.synchronize()
            rounds[circ].append(a.elapsed_time(b) / calls)
    res = {}
    for circ in (False, True):
        key = "on" if circ else "off"
        res[key] = {"ms_per_call": round(statistics.median(rounds[circ]), 3), "rounds": [round(v, 3) for v in rounds[circ]]}
        eng.set_circular(circ)
        with tempfile.TemporaryDirectory() as td:
            dump = os.path.join(td, "ops.csv")
            os.environ["SDXE_PROFILE_DUMP"] = dump
            eng.profile(True)
            call()
            torch.cuda.synchronize()
            eng.profile(False)
            del os.environ["SDXE_PROFILE_DUMP"]
            res[key]["added_ms_profiled"] = _added_ms(dump)
    res["overhead_pct"] = round(100.0 * (res["on"]["ms_per_call"] / res["off"]["ms_per_call"] - 1.0), 2)
    eng.set_circular(False)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--workloads", default="sd15_unet,sdxl_unet,vae_decode")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tiling needs a CUDA device")
    from bench_samplers import gpu_info
    from sdwebui_b200 import checkpoint as C
    from sdwebui_b200.engine import UNetEngine, UNetSpec, VAEDecoderEngine, VAESpec

    dev, dtype = torch.device("cuda:0"), torch.bfloat16
    result = {"gpu": gpu_info(), "dtype": "bf16", "calls": args.calls, "reps": args.reps, "workloads": {}}
    g = torch.Generator(device="cuda").manual_seed(0)
    for name in args.workloads.split(","):
        if name == "vae_decode":
            eng = VAEDecoderEngine(VAESpec(), dtype=dtype, device=dev)
            eng.load_state_dict(C.synthetic_state_dict(C.vae_decoder_param_shapes(VAESpec()), seed=2, device=dev, dtype=dtype))
            eng.finalize()
            z = torch.randn(8, 4, 64, 64, device=dev, generator=g).to(dtype)
            out = torch.empty(8, 3, 512, 512, device=dev, dtype=dtype)
            call = lambda: eng.decode(z, out=out)  # noqa: E731
            shape = "B=8 512x512"
        else:
            xl = name == "sdxl_unet"
            spec = UNetSpec.sdxl() if xl else UNetSpec.sd15()
            eng = UNetEngine(spec, dtype=dtype, device=dev)
            eng.load_state_dict(C.synthetic_state_dict(C.unet_param_shapes(spec), seed=1, device=dev, dtype=dtype))
            eng.finalize()
            n, hw = (8, 128) if xl else (16, 64)
            x = torch.randn(n, 4, hw, hw, device=dev, generator=g).to(dtype)
            t = torch.full((n,), 500.0, device=dev, dtype=dtype)
            ctx = torch.randn(n, 77, spec.context_dim, device=dev, generator=g).to(dtype)
            y = torch.randn(n, spec.adm_in_channels, device=dev, generator=g).to(dtype) if spec.adm_in_channels else None
            out = torch.empty_like(x)
            call = lambda: eng.forward(x, t, ctx, y, out=out, context_key=1)  # noqa: E731
            shape = f"2B={n} {hw}x{hw}"
        res = _time(eng, call, args.calls, args.reps)
        res["shape"] = shape
        result["workloads"][name] = res
        print(name, json.dumps(res), flush=True)
        eng.close()
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
