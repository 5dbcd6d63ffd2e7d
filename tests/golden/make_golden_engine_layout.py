"""Writes tests/golden/engine_layout_ref.json: the host-side layout of small seeded engines (weight-blob size and SHA-256,
activation-pool bytes after one forward, launches of a replayed call, the profiled op list, and sdxe_finalize's report
of missing weights), recorded from the cases in tests/test_engine_layout_gpu.py. Needs a CUDA GPU (an H100: the engine
is built for sm_90a) and a built libsdxe.so.

    python tests/golden/make_golden_engine_layout.py   ->   tests/golden/engine_layout_ref.json
"""
import json
import os
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import test_engine_layout_gpu as T  # noqa: E402


def main():
    if not torch.cuda.is_available():
        raise SystemExit("make_golden_engine_layout.py needs a CUDA device")
    with tempfile.TemporaryDirectory() as tmp:
        rec = T.records(torch.device("cuda:0"), tmp)
    with open(T.GOLDEN, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote {T.GOLDEN}: {len(rec) - 1} engine records")


if __name__ == "__main__":
    main()
