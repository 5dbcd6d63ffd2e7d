"""Writes tests/golden/hypertile_ref.json from the reference's own Hypertile extension, unmodified.

    python tests/golden/make_golden_hypertile.py <reference webui root>

It imports extensions-builtin/hypertile/hypertile.py and scripts/hypertile_script.py (with stub `modules.*` packages and
stub nn.Module trees that carry the ldm attn1 names of SD1.5 and SDXL) and records:
  * hooked:      the hooked layers and their depths (the extension's own endswith matching);
  * candidates:  find_hw_candidates for every UNet level of several image sizes;
  * regroup:     the token permutation of the regrouping for several (h', w', nh, nw);
  * jobs:        the draws "nhxnw" of every enabled layer on every UNet forward, through the script's
                 process() / before_hr() sequence, for several seeds and settings.
Needs torch and einops (both used by the reference module).
"""
import json
import os
import sys
import types

import torch
import torch.nn as nn

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hypertile_ref.json")


def attn1_names(is_sdxl):
    """ldm attn1 module names in execution order."""
    if is_sdxl:
        mult_depth = [0, 2, 10]
        middle = 10
    else:
        mult_depth = [1, 1, 1, 0]
        middle = 1
    names, idx = [], 1
    nl = len(mult_depth)
    for level in range(nl):
        for _ in range(2):
            names += [(f"input_blocks.{idx}.1.transformer_blocks.{k}.attn1", level) for k in range(mult_depth[level])]
            idx += 1
        if level != nl - 1:
            idx += 1
    names += [(f"middle_block.1.transformer_blocks.{k}.attn1", nl - 1) for k in range(middle)]
    idx = 0
    for level in reversed(range(nl)):
        for _ in range(3):
            names += [(f"output_blocks.{idx}.1.transformer_blocks.{k}.attn1", level) for k in range(mult_depth[level])]
            idx += 1
    return names


class Leaf(nn.Module):
    def forward(self, x):
        return x


def stub_tree(names):
    """DiffusionWrapper-like tree: model.diffusion_model.<ldm name>, modules registered in execution order."""
    root = nn.Module()
    for name, _ in names:
        cur = root
        parts = ("diffusion_model." + name).split(".")
        for part in parts[:-1]:
            if not hasattr(cur, part):
                cur.add_module(part, nn.Module())
            cur = getattr(cur, part)
        cur.add_module(parts[-1], Leaf())
    return root


def level_tokens(w, h, levels):
    lh, lw, out = h // 8, w // 8, []
    for _ in range(levels):
        out.append(lh * lw)
        lh, lw = (lh + 1) // 2, (lw + 1) // 2
    return out


def main(ref_root):
    ht_dir = os.path.join(ref_root, "extensions-builtin", "hypertile")
    sys.path.insert(0, ht_dir)
    shared = types.SimpleNamespace(opts=None, sd_model=None)
    modules = types.ModuleType("modules")
    modules.scripts = types.SimpleNamespace(Script=object, AlwaysVisible=object())
    modules.script_callbacks = types.SimpleNamespace(on_ui_settings=lambda f: None, on_before_ui=lambda f: None)
    modules.shared = shared
    sys.modules["modules"] = modules
    for k in ("scripts", "script_callbacks", "shared"):
        sys.modules["modules." + k] = getattr(modules, k)
    import hypertile as H  # noqa: E402
    import importlib.util

    spec = importlib.util.spec_from_file_location("hypertile_script", os.path.join(ht_dir, "scripts", "hypertile_script.py"))
    script_mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(script_mod)

    # record every draw: (current layer, result); the extension's wrapper looks random_divisor up in its module
    orig_divisor = H.random_divisor
    current = {"layer": None}
    draws = []

    def recording_divisor(value, min_value, max_options=1):
        r = orig_divisor(value, min_value, max_options)
        draws.append((current["layer"], r))
        return r

    H.random_divisor = recording_divisor
    out = {"hooked": {}, "candidates": [], "regroup": [], "jobs": []}

    # ---- hooked layers
    for model_name, is_sdxl in (("sd15", False), ("sdxl", True)):
        tree = stub_tree(attn1_names(is_sdxl))
        H.hypertile_hook_model(tree, 512, 512, enable=True, is_sdxl=is_sdxl)
        hooked = []
        for name, mod in tree.named_modules():
            prm = getattr(mod, "__webui_hypertile_params", None)
            if prm is not None:
                hooked.append([name[len("diffusion_model."):], prm.depth])
        out["hooked"][model_name] = hooked

    # ---- find_hw_candidates per level
    for w, h in ((512, 512), (768, 512), (1024, 1024), (1216, 832), (832, 1216)):
        for hw in level_tokens(w, h, 4):
            out["candidates"].append([w, h, hw, list(H.find_hw_candidates(hw, w / h))])

    # ---- regrouping permutation: the tokens the wrapped forward sees, with the draws pinned
    seen = {}

    class Probe(nn.Module):
        def forward(self, x):
            seen["x"] = x.clone()
            return x

    for hp, wp, nh, nw in ((8, 8, 2, 2), (12, 8, 3, 2), (8, 12, 2, 3), (24, 16, 3, 2), (38, 26, 2, 2), (6, 4, 3, 1), (10, 6, 1, 1)):
        prm = H.HypertileParams()
        probe = Probe()
        prm.forward = probe.forward
        prm.enabled, prm.tile_size, prm.swap_size, prm.aspect_ratio, prm.depth = True, 128, 1, hp / wp, 0
        assert H.find_hw_candidates(hp * wp, hp / wp) == (hp, wp)
        pinned = iter([nh, nw])
        H.random_divisor = lambda *a, **k: next(pinned)
        x = torch.arange(hp * wp, dtype=torch.float64).reshape(1, hp * wp, 1)
        y = H.self_attn_forward(prm)(x)
        H.random_divisor = recording_divisor
        assert torch.equal(y, x)
        out["regroup"].append([hp, wp, nh, nw, [int(v) for v in seen["x"].reshape(-1)]])

    # ---- jobs: process() -> first-pass forwards -> before_hr() -> hires forwards
    case = 0
    for model_name, is_sdxl, (w, h), (hw_, hh_) in (("sd15", False, (512, 512), (1024, 1024)),
                                                    ("sd15", False, (768, 512), (1152, 768)),
                                                    ("sdxl", True, (832, 1216), (1248, 1824))):
        names = attn1_names(is_sdxl)
        # every max depth with the default swap size and each way of enabling; swap size 1 and "all off" once each
        settings = [(d, 3, e, s) for d in range(4) for e, s in ((True, False), (False, True), (True, True))]
        settings += [(3, 1, True, False), (1, 1, False, True), (3, 3, False, False)]
        for max_depth, swap, enable, secondpass in settings:
            case += 1
            tree = stub_tree(names)
            mods = [tree.get_submodule("diffusion_model." + n) for n, _ in names]
            opts = types.SimpleNamespace(
                hypertile_enable_unet=enable, hypertile_enable_unet_secondpass=secondpass, hypertile_max_depth_unet=max_depth,
                hypertile_max_tile_unet=256, hypertile_swap_size_unet=swap, hypertile_enable_vae=False,
                hypertile_max_depth_vae=3, hypertile_max_tile_vae=128, hypertile_swap_size_vae=3)
            opts.get_default = lambda name: None
            shared.opts = opts
            shared.sd_model = types.SimpleNamespace(first_stage_model=nn.Module(), model=tree, is_sdxl=is_sdxl)
            seed = 1000 + 37 * case
            p = types.SimpleNamespace(all_seeds=[seed, seed + 1], width=w, height=h, hr_upscale_to_x=hw_,
                                      hr_upscale_to_y=hh_, extra_generation_params={})
            script = script_mod.ScriptHypertile()
            forwards = []

            def run_forwards(k, W, H_):
                tokens = level_tokens(W, H_, 4)
                for _ in range(k):
                    draws.clear()
                    for i, ((_, level), mod) in enumerate(zip(names, mods)):
                        current["layer"] = i
                        mod(torch.zeros(1, tokens[level], 1))
                    per_layer = [0] * len(names)
                    for i, r in draws:
                        per_layer[i] = [r] if per_layer[i] == 0 else per_layer[i] + [r]
                    # one string per forward: "nhxnw" per layer in execution order, "-" for a layer that drew nothing
                    forwards.append(" ".join("-" if d == 0 else "x".join(map(str, d)) for d in per_layer))

            script.process(p)
            run_forwards(2, w, h)
            script.before_hr(p)
            run_forwards(2, hw_, hh_)
            out["jobs"].append({"model": model_name, "width": w, "height": h, "hr_width": hw_, "hr_height": hh_,
                                "seed": seed, "enable_unet": enable, "enable_unet_secondpass": secondpass,
                                "max_depth": max_depth, "swap_size": swap, "max_tile": 256, "forwards": forwards})
    with open(OUT, "w") as f:
        json.dump(out, f, separators=(",", ":"))
    print(f"wrote {OUT}: {len(out['jobs'])} jobs")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit("usage: make_golden_hypertile.py <reference webui root>")
    main(sys.argv[1])
