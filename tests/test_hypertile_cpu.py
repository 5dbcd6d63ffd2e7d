"""Hypertile's host side against the reference extension's own behaviour (tests/golden/hypertile_ref.json, written by
tests/golden/make_golden_hypertile.py from the unmodified extension): hooked layers and depths, grid candidates, the
token regrouping, and the draw sequence of whole jobs, headless and through the webui seam."""
import json
import os
import sys
import types

import pytest
import torch

from sdwebui_b200 import hypertile as HT
from sdwebui_b200 import sd_unet
from sdwebui_b200.engine import UNetSpec

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import hypertile_oracle  # noqa: E402

GOLDEN = json.load(open(os.path.join(HERE, "golden", "hypertile_ref.json")))
SPECS = {"sd15": (UNetSpec.sd15(), False), "sdxl": (UNetSpec.sdxl(), True)}


@pytest.mark.parametrize("model", ["sd15", "sdxl"])
def test_hooked_layers_and_depths(model):
    spec, is_sdxl = SPECS[model]
    ours = sorted([name, HT.layer_depth(name, is_sdxl)] for name, _ in HT.attn1_layers(spec)
                  if HT.layer_depth(name, is_sdxl) is not None)
    assert ours == sorted(GOLDEN["hooked"][model])
    counts = [sum(1 for _, d in ours if d == k) for k in range(4)]
    assert counts == ([5, 5, 5, 1] if model == "sd15" else [5, 55, 10, 0])
    assert len(HT.attn1_layers(spec)) == (16 if model == "sd15" else 70)


def test_find_hw_candidates():
    for w, h, hw, cand in GOLDEN["candidates"]:
        assert list(HT.find_hw_candidates(hw, w / h)) == cand, (w, h, hw)
    # the transposed grid of non-square images: 1216x832 level 0 is 104 x 152 tokens, the candidates are (152, 104)
    assert HT.find_hw_candidates(104 * 152, 1216 / 832) == (152, 104)


def test_divisors_and_tile_size():
    assert HT.get_divisors(96, 32, 3) == [3, 2, 1]
    assert HT.get_divisors(64, 128, 3) == [1]
    assert HT.largest_tile_size_available(1216, 832) == 64
    assert HT.largest_tile_size_available(1024, 1024) == 1024


def test_regroup_permutation_matches_reference():
    for hp, wp, nh, nw, perm in GOLDEN["regroup"]:
        n = hp * wp
        x = torch.arange(n, dtype=torch.float64).reshape(1, n, 1)
        y = hypertile_oracle.regroup(x, hp, wp, nh, nw)
        assert [int(v) for v in y.reshape(-1)] == perm, (hp, wp, nh, nw)
        assert torch.equal(hypertile_oracle.ungroup(y, hp, wp, nh, nw), x)


def _golden_rows(fwd):
    return [None if d == "-" else tuple(int(v) for v in d.split("x")) for d in fwd.split()]


def _our_rows(rows):
    return [None if mt == 0 else (nh, nw) for _, _, nh, nw, mt in rows]


def _job_p(job, unet):
    model = types.SimpleNamespace(unet=unet, is_sdxl=job["model"] == "sdxl")
    opts = HT.HypertileOptions(enable_unet=job["enable_unet"], enable_unet_secondpass=job["enable_unet_secondpass"],
                               max_depth_unet=job["max_depth"], max_tile_unet=job["max_tile"], swap_size_unet=job["swap_size"])
    return types.SimpleNamespace(sd_model=model, seeds=[job["seed"], job["seed"] + 1], width=job["width"],
                                 height=job["height"], hypertile=opts)


class _RecordingEngine:
    """Stands in for UNetEngine: records the Hypertile rows of every call."""

    def __init__(self, spec):
        self.spec = spec
        self.calls = []

    def forward(self, x, t, ctx, y=None, context_key=0, hypertile=None):
        self.calls.append(hypertile)
        return torch.zeros_like(x)


def _unet(model):
    spec, _ = SPECS[model]
    u = sd_unet.SdxeUnet({}, spec)
    u.engine = _RecordingEngine(spec)
    return u


def _call(u, w, h, batch):
    x = torch.zeros(batch, 4, h // 8, w // 8)
    u.forward(x, torch.zeros(batch), torch.zeros(batch, 77, 8))


@pytest.mark.parametrize("idx", range(len(GOLDEN["jobs"])))
def test_job_draw_sequence(idx):
    """A simulated job through SdxeUnet.forward: process() -> Heun's two calls of one step -> before_hr() -> the hires
    step's cond and uncond sub-batches. Every call's draws equal the reference's."""
    job = GOLDEN["jobs"][idx]
    u = _unet(job["model"])
    p = _job_p(job, u)
    u.hypertile = HT.begin_job(p)
    _call(u, job["width"], job["height"], 2)   # Heun: first call
    _call(u, job["width"], job["height"], 2)   # Heun: second-order call
    u.hypertile = HT.begin_hr_pass(p, job["hr_width"], job["hr_height"])
    _call(u, job["hr_width"], job["hr_height"], 1)  # cond sub-batch
    _call(u, job["hr_width"], job["hr_height"], 1)  # uncond sub-batch
    assert len(u.engine.calls) == len(job["forwards"]) == 4
    for rows, fwd in zip(u.engine.calls, job["forwards"]):
        want = _golden_rows(fwd)
        if all(v is None for v in want):
            assert rows is None  # nothing enabled: no table, the call is exactly as without Hypertile
        else:
            assert _our_rows(rows) == want
            for hp, wp, nh, nw, mt in rows:
                if mt:
                    assert hp % nh == 0 and wp % nw == 0 and nh * nw <= mt


def test_no_hypertile_makes_no_draws():
    u = _unet("sd15")
    state = HT.RNG.getstate()
    _call(u, 512, 512, 2)
    assert u.engine.calls == [None]
    assert HT.RNG.getstate() == state


def test_max_tiles_bounds_every_draw():
    spec, _ = SPECS["sd15"]
    st = HT.configure(spec, 1024, 1024, HT.HypertileOptions(enable_unet=True), True, False)
    rows = st.draw_rows(128, 128)
    lvl0 = [r for r, (_, level) in zip(rows, HT.attn1_layers(spec)) if level == 0]
    assert all(r[:2] == (128, 128) and r[4] == 16 for r in lvl0)  # nh, nw in {4, 2, 1} at 1024^2, tile 256
    assert st.structure(128, 128)[0] == (128, 128, 0, True)


# ---- webui seam -------------------------------------------------------------------------------------------------
class _Params:
    def __init__(self, depth, enabled, tile_size=256, swap_size=3, aspect_ratio=1.0):
        self.depth, self.enabled, self.tile_size, self.swap_size, self.aspect_ratio = depth, enabled, tile_size, swap_size, aspect_ratio


def _webui_tree(spec, is_sdxl, max_depth, aspect):
    root = torch.nn.Module()
    hooked = {}
    for name, _ in HT.attn1_layers(spec):
        cur = root
        parts = ("diffusion_model." + name).split(".")
        for part in parts[:-1]:
            if not hasattr(cur, part):
                cur.add_module(part, torch.nn.Module())
            cur = getattr(cur, part)
        leaf = torch.nn.Module()
        cur.add_module(parts[-1], leaf)
        depth = HT.layer_depth(name, is_sdxl)
        if depth is not None:
            setattr(leaf, "__webui_hypertile_params", _Params(depth, depth <= max_depth, aspect_ratio=aspect))
            hooked["diffusion_model." + name] = 1
    setattr(root, "__webui_hypertile_layers", hooked)
    return root


def test_webui_draws_through_the_webui_module(monkeypatch):
    """Inside the webui, the draws go through the webui's own hypertile module, in stock order, with stock arguments."""
    spec, is_sdxl = SPECS["sd15"]
    calls = []
    stub = types.ModuleType("hypertile")
    stub.find_hw_candidates = lambda hw, ar: (calls.append(("hw", hw, ar)), HT.find_hw_candidates(hw, ar))[1]
    stub.random_divisor = lambda v, lo, n: (calls.append(("div", v, lo, n)), 1)[1]
    shared = types.SimpleNamespace(sd_model=types.SimpleNamespace(model=_webui_tree(spec, is_sdxl, 1, 768 / 512)))
    monkeypatch.setitem(sys.modules, "hypertile", stub)
    monkeypatch.setitem(sys.modules, "modules", types.SimpleNamespace(shared=shared))
    monkeypatch.setitem(sys.modules, "modules.shared", shared)
    monkeypatch.setattr(sd_unet, "IN_WEBUI", True)
    u = _unet("sd15")
    _call(u, 768, 512, 2)
    rows = u.engine.calls[0]
    expect = []
    for (name, level), row in zip(HT.attn1_layers(spec), rows):
        depth = HT.layer_depth(name, is_sdxl)
        if depth is None or depth > 1:
            assert row == (0, 0, 1, 1, 0)
            continue
        tokens = HT.level_tokens(64, 96, 4)[level]
        hp, wp = HT.find_hw_candidates(tokens, 768 / 512)
        lo = 256 // 8 * 2 ** depth
        expect += [("hw", tokens, 768 / 512), ("div", hp, lo, 3), ("div", wp, lo, 3)]
        assert row[:4] == (hp, wp, 1, 1)
    assert calls == expect and len(expect) == 10 * 3


def test_webui_without_hypertile_module(monkeypatch):
    spec, is_sdxl = SPECS["sd15"]
    shared = types.SimpleNamespace(sd_model=types.SimpleNamespace(model=_webui_tree(spec, is_sdxl, 3, 1.0)))
    monkeypatch.setitem(sys.modules, "hypertile", None)  # import fails
    monkeypatch.setitem(sys.modules, "modules", types.SimpleNamespace(shared=shared))
    monkeypatch.setitem(sys.modules, "modules.shared", shared)
    monkeypatch.setattr(sd_unet, "IN_WEBUI", True)
    u = _unet("sd15")
    _call(u, 512, 512, 2)
    assert u.engine.calls == [None]


def test_webui_without_hooks(monkeypatch):
    stub = types.ModuleType("hypertile")
    shared = types.SimpleNamespace(sd_model=types.SimpleNamespace(model=torch.nn.Module()))
    monkeypatch.setitem(sys.modules, "hypertile", stub)
    monkeypatch.setitem(sys.modules, "modules", types.SimpleNamespace(shared=shared))
    monkeypatch.setitem(sys.modules, "modules.shared", shared)
    monkeypatch.setattr(sd_unet, "IN_WEBUI", True)
    u = _unet("sd15")
    _call(u, 512, 512, 2)
    assert u.engine.calls == [None]
