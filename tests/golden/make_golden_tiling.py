"""Pins tests/tiling_oracle.apply_circular to the REFERENCE: StableDiffusionModelHijack.apply_circular and the `flatten`
that hijack() builds its layer list with (modules/sd_hijack.py:254-261, 311-318) are taken from the file by AST and
executed as they are on the tiny oracle UNet (both variants), VAE decoder and VAE encoder with seeded inputs. The outputs
with Tiling on, and again after turning it off, go to tiling_ref.npz.

    python tests/golden/make_golden_tiling.py   ->   tests/golden/tiling_ref.npz
"""
import ast
import os
import sys
import textwrap

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from tiling_oracle import cases  # noqa: E402


def reference_hijack():
    """A stand-in class for model_hijack with the reference's apply_circular method, and hijack()'s nested flatten, both
    unmodified."""
    src = open(os.path.join(REF, "modules", "sd_hijack.py")).read()
    tree = ast.parse(src)
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "StableDiffusionModelHijack")
    methods = {n.name: n for n in cls.body if isinstance(n, ast.FunctionDef)}
    apply_src = textwrap.dedent(ast.get_source_segment(src, methods["apply_circular"], padded=True))
    flatten = next(n for n in ast.walk(methods["hijack"]) if isinstance(n, ast.FunctionDef) and n.name == "flatten")
    flatten_src = textwrap.dedent(ast.get_source_segment(src, flatten, padded=True))
    ns = {"torch": torch}
    exec(compile(flatten_src + "\n\nclass Hijack:\n    circular_enabled = False\n    layers = None\n\n" +
                 textwrap.indent(apply_src, "    "), "sd_hijack.py", "exec"), ns)
    return ns["Hijack"], ns["flatten"]


def main():
    Hijack, flatten = reference_hijack()
    out = {}
    with torch.no_grad():
        for name, (build, inputs, run) in cases().items():
            model = build()
            h = Hijack()
            h.layers = flatten(model)
            args = inputs()
            h.apply_circular(True)
            out[f"{name}/circular"] = run(model, args).numpy()
            h.apply_circular(True)                      # unchanged: the early return
            h.apply_circular(False)
            out[f"{name}/zeros"] = run(model, args).numpy()
            print(name, out[f"{name}/circular"].shape,
                  float(np.abs(out[f"{name}/circular"] - out[f"{name}/zeros"]).max()))
    np.savez_compressed(os.path.join(HERE, "tiling_ref.npz"), **out)


if __name__ == "__main__":
    main()
