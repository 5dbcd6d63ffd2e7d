"""Hypertile off vs on (the extension's defaults: max tile 256, swap size 3, max depth 3) on three workloads, bf16,
synthetic weights, CFG 7, batch 4, full process_images (sampling + VAE decode, images left on the device):

  sd15_hires   SD1.5 512x512 -> 1024x1024 latent hires, Euler a 20 + 20, Hypertile on the second pass only
  sd15_1024    SD1.5 1024x1024 txt2img, Euler a 20, Hypertile U-Net on
  sdxl_1024    SDXL 1024x1024 txt2img, Euler a 20, Hypertile U-Net on

    python tools/bench_hypertile.py [--reps 2] [--steps 20] [--out results/bench_hypertile.json]

Each workload runs off / on alternately, `reps` times each, after one warm-up job per setting. Reported per setting:
images/s (host clock around whole jobs ending in a synchronise); from one separate engine-profiled job (per-op CUDA
events, SDXE_PROFILE_DUMP) the time of the highest-resolution self-attention class and of the Hypertile gather kernels;
and the host time per UNet call spent drawing the Hypertile table. One JSON line, with the card's name and power limit."""
import argparse
import json
import os
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

WORKLOADS = {
    "sd15_hires": dict(arch="sd15", width=512, height=512, hires=True),
    "sd15_1024": dict(arch="sd15", width=1024, height=1024, hires=False),
    "sdxl_1024": dict(arch="sdxl", width=1024, height=1024, hires=False),
}


def _profile_classes(dump_path, top_tokens):
    attn_ms = gather_ms = 0.0
    for line in open(dump_path):
        _, kind, desc, us = line.split(",")[:4]
        words = desc.split()
        f = dict(w.split("=", 1) for w in words[1:] if "=" in w)
        if words and words[0] == "attn" and f.get("Nq") == f.get("Nk") and int(f["Nq"]) == top_tokens:
            attn_ms += float(us) / 1000.0
        elif words and words[0] == "ht_gather":
            gather_ms += float(us) / 1000.0
    return attn_ms, gather_ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_hypertile needs a CUDA device")
    import bench
    from bench_samplers import gpu_info
    from sdwebui_b200 import hypertile as HT
    from sdwebui_b200.processing import StableDiffusionProcessingTxt2Img, process_images
    from sdwebui_b200.sd_unet import SdxeUnet

    dev, dtype, B = torch.device("cuda:0"), torch.bfloat16, args.batch
    draw_time = {"s": 0.0, "calls": 0}
    orig_rows = SdxeUnet.hypertile_rows

    def timed_rows(self, h, w):
        t0 = time.perf_counter()
        r = orig_rows(self, h, w)
        if r is not None:
            draw_time["s"] += time.perf_counter() - t0
            draw_time["calls"] += 1
        return r

    SdxeUnet.hypertile_rows = timed_rows
    result = {"gpu": gpu_info(), "batch": B, "steps": args.steps, "dtype": "bf16", "workloads": {}}
    models = {}
    for name in args.workloads.split(","):
        w = WORKLOADS[name]
        if w["arch"] not in models:
            models.clear()
            torch.cuda.empty_cache()
            models[w["arch"]] = bench.build_model(w["arch"], dtype, dev, 0, 1)[0]
        model = models[w["arch"]]
        wl = {"ctx_dim": 2048 if w["arch"] == "sdxl" else 768, "adm": 2816 if w["arch"] == "sdxl" else 0}
        c, uc = (bench.to_dev(v, dev) for v in bench.make_conds(wl, B, dev, 7))

        def job(on):
            ht = HT.HypertileOptions(enable_unet=not w["hires"], enable_unet_secondpass=w["hires"]) if on else None
            p = StableDiffusionProcessingTxt2Img(sd_model=model, c=c, uc=uc, seeds=list(range(1000, 1000 + B)), sampler_name="Euler a",
                                                 steps=args.steps, width=w["width"], height=w["height"], enable_hr=w["hires"],
                                                 hr_scale=2.0, denoising_strength=0.7, hypertile=ht)
            return process_images(p, to_host=False)

        res = {"off": {"img_s": []}, "on": {"img_s": []}}
        for on in (False, True):
            job(on)
        torch.cuda.synchronize()
        for _ in range(args.reps):
            for on in (False, True):
                draw_time.update(s=0.0, calls=0)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                job(on)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                key = "on" if on else "off"
                res[key]["img_s"].append(round(B / dt, 3))
                if on:
                    res[key]["draw_us_per_call"] = round(1e6 * draw_time["s"] / max(1, draw_time["calls"]), 1)
        hh, ww = (w["height"] * (2 if w["hires"] else 1)) // 8, (w["width"] * (2 if w["hires"] else 1)) // 8
        top_tokens = hh * ww if w["arch"] == "sd15" else (hh // 2) * (ww // 2)
        for on in (False, True):
            with tempfile.TemporaryDirectory() as td:
                dump = os.path.join(td, "ops.csv")
                os.environ["SDXE_PROFILE_DUMP"] = dump
                model.unet.engine.profile(True)
                job(on)
                torch.cuda.synchronize()
                model.unet.engine.profile(False)
                del os.environ["SDXE_PROFILE_DUMP"]
                attn_ms, gather_ms = _profile_classes(dump, top_tokens)
            key = "on" if on else "off"
            res[key]["top_self_attention_ms_per_job"] = round(attn_ms, 2)
            res[key]["gather_ms_per_job"] = round(gather_ms, 2)
        res["top_self_attention_tokens"] = top_tokens
        result["workloads"][name] = res
        print(name, json.dumps(res), flush=True)
    SdxeUnet.hypertile_rows = orig_rows
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
