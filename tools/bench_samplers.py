"""Images/s of the samplers users pick for few-step generation, at bench.py's headline size: SD1.5 512x512, batch 8, bf16,
synthetic weights, CFG 7, full process_images (sampling + VAE decode, images left on the device).

    python tools/bench_samplers.py [--warmup 1] [--reps 3] [--out results/bench_samplers.json]

Per run it reports images/s (host clock around whole jobs ending in a synchronise), the UNet calls per job, and the
per-step time outside the UNet: CUDA events around the sampler call minus CUDA events around every UNet call, divided by
the UNet calls. It prints one JSON line with the card's name and power limit beside the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RUNS = [("Euler a", 20), ("DDIM", 20), ("PLMS", 20), ("UniPC", 20), ("UniPC", 10), ("LCM", 4), ("LCM", 8)]


def gpu_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        pl, sm = [v.strip() for v in r.stdout.strip().split(",")[:2]]
        info.update(power_limit_w=float(pl), sm_max_mhz=float(sm))
    except Exception as e:  # read-only query; the numbers are still reported without it
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_samplers needs a CUDA device")
    import sdwebui_b200  # noqa: F401
    from sdwebui_b200 import checkpoint as C
    from sdwebui_b200.engine import UNetSpec, VAEDecoderEngine, VAESpec
    from sdwebui_b200.processing import SdModel, StableDiffusionProcessingTxt2Img, process_images
    from sdwebui_b200.sd_unet import SdxeUnet

    dev, dtype, B = torch.device("cuda:0"), torch.bfloat16, args.batch
    spec = UNetSpec.sd15()
    usd = C.synthetic_state_dict(C.unet_param_shapes(spec), seed=0, device=dev, dtype=torch.float16)
    vsd = C.synthetic_state_dict(C.vae_decoder_param_shapes(VAESpec()), seed=1, device=dev, dtype=torch.float16)
    unet = SdxeUnet(usd, spec, dtype=dtype, device=dev)
    unet.activate()
    vae = VAEDecoderEngine(VAESpec(), dtype=dtype, device=dev)
    vae.load_state_dict(vsd)
    vae.finalize()
    del usd, vsd
    model = SdModel(unet, vae, is_sdxl=False, dtype_unet=dtype, device=dev)
    g = torch.Generator().manual_seed(7)
    cond = torch.randn(B, 77, 768, generator=g).to(dev, dtype)
    uncond = torch.randn(B, 77, 768, generator=g).to(dev, dtype)

    unet_events = []
    fwd = unet.forward

    def timed_forward(*a, **k):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = fwd(*a, **k)
        e.record()
        unet_events.append((s, e))
        return out

    unet.forward = timed_forward

    class Job(StableDiffusionProcessingTxt2Img):
        def sample(self, c, uc, seeds):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out = super().sample(c, uc, seeds)
            e.record()
            self.sample_events = (s, e)
            return out

    results = []
    for sampler, steps in RUNS:
        def job():
            p = Job(sd_model=model, c=cond, uc=uncond, seeds=list(range(1000, 1000 + B)), sampler_name=sampler, steps=steps,
                    width=512, height=512, randn_source="GPU", check_for_nans=False)
            process_images(p, to_host=False)
            return p

        for _ in range(args.warmup):
            job()
        torch.cuda.synchronize()
        unet_events.clear()
        outside, calls = [], []
        t0 = time.perf_counter()
        for _ in range(args.reps):
            n0 = len(unet_events)
            p = job()
            torch.cuda.synchronize()
            ev = unet_events[n0:]
            t_unet = sum(s.elapsed_time(e) for s, e in ev)
            t_sample = p.sample_events[0].elapsed_time(p.sample_events[1])
            calls.append(len(ev))
            outside.append((t_sample - t_unet) / len(ev))
        dt = time.perf_counter() - t0
        r = {"sampler": sampler, "steps": steps, "images_per_s": round(B * args.reps / dt, 3), "unet_calls": calls[0],
             "outside_unet_ms_per_call": round(sum(outside) / len(outside), 4), "job_s": round(dt / args.reps, 4)}
        print(json.dumps(r), flush=True)
        results.append(r)
    line = {"bench": "samplers", "config": {"model": "sd15", "size": 512, "batch": B, "dtype": "bf16", "weights": "synthetic",
                                            "cfg_scale": 7.0, "decode": True, "reps": args.reps, "warmup": args.warmup},
            "gpu": gpu_info(), "runs": results}
    unet.deactivate()
    vae.close()
    print(json.dumps(line))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
