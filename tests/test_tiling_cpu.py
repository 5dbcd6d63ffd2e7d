"""Tiling without a GPU: the test-side apply_circular against the reference's own code (tests/golden/tiling_ref.npz, made
by tests/golden/make_golden_tiling.py from modules/sd_hijack.py:254-261,311-318), the host logic of process_images
(modules/processing.py:879-880,895) through fake engine handles, and the webui seams with a stub `modules` package."""
import contextlib
import importlib
import importlib.util
import os
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from tiling_oracle import apply_circular, cases  # noqa: E402

ROOT = os.path.dirname(HERE)
EXT = os.path.join(ROOT, "stable-diffusion-webui_b200", "webui_extension", "scripts", "sdxe_unet.py")


# ---- oracle pin ---------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "tiling_ref.npz"))


@pytest.mark.parametrize("name", list(cases()))
def test_apply_circular_matches_reference(golden, name):
    build, inputs, run = cases()[name]
    model, args = build(), inputs()
    with torch.no_grad():
        apply_circular(model, True)
        on = run(model, args).numpy()
        apply_circular(model, False)
        off = run(model, args).numpy()
    ref_on, ref_off = golden[f"{name}/circular"], golden[f"{name}/zeros"]
    # the same modules, inputs and torch ops as the generator: equal up to the CPU's own fp32 kernel choices
    np.testing.assert_allclose(on, ref_on, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(off, ref_off, rtol=1e-5, atol=1e-5)
    assert np.abs(ref_on - ref_off).max() > 0.1  # the wrap changes the result: the pin discriminates


def test_padding_zero_conv_is_untouched():
    """The VAE encoder's Downsample is Conv2d(padding=0) after a constant pad: its mode flips, its output does not."""
    from oracle.vae import Downsample

    torch.manual_seed(0)
    d = Downsample(8).eval()
    x = torch.randn(1, 8, 6, 10)
    with torch.no_grad():
        a = d(x)
        apply_circular(d, True)
        assert d.conv.padding_mode == "circular"
        assert torch.equal(d(x), a)


# ---- process_images host logic ------------------------------------------------------------------------------------
class _FakeEngine:
    def __init__(self):
        self.calls = []

    def set_circular(self, enable):
        self.calls.append(bool(enable))


def _model(with_encoder=True):
    from sdwebui_b200.processing import SdModel
    from sdwebui_b200.sd_unet import SdxeUnet

    su = SdxeUnet({}, dtype=torch.float16, device="cpu")
    su.engine = _FakeEngine()  # an activated UNet, as far as Tiling goes
    m = SdModel(su, _FakeEngine(), is_sdxl=False, device="cpu", vae_encoder=_FakeEngine() if with_encoder else None)
    return m


def _engines(m):
    return [m.unet.engine, m.vae] + ([m.vae_encoder] if m.vae_encoder is not None else [])


def _run(monkeypatch, p):
    """process_images up to the sampler: `p.sample` records the Tiling state each pass sees and stops the job."""
    from sdwebui_b200 import processing as P

    seen = []

    def sample(c, uc, seeds):
        seen.append(p.sd_model.circular_enabled)
        if p.enable_hr:
            seen.append(p.sd_model.circular_enabled)  # sample_hr_pass runs on the same model, nothing resets it
        raise _Stop()

    monkeypatch.setattr(p, "sample", sample)
    monkeypatch.setattr(p, "make_rng", lambda shape, seeds: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())  # the job's device is the CPU here
    with pytest.raises(_Stop):
        P.process_images(p)
    return seen


class _Stop(Exception):
    pass


def test_tiling_none_resolves_to_off(monkeypatch):
    from sdwebui_b200.processing import StableDiffusionProcessingTxt2Img

    m = _model()
    p = StableDiffusionProcessingTxt2Img(sd_model=m, c=torch.zeros(1), uc=torch.zeros(1))
    assert p.tiling is None
    assert _run(monkeypatch, p) == [False]
    assert p.tiling is False
    assert all(e.calls == [] for e in _engines(m))  # off -> off: apply_circular's early return


def test_tiling_reaches_all_three_engines(monkeypatch):
    from sdwebui_b200.processing import StableDiffusionProcessingImg2Img

    m = _model()
    p = StableDiffusionProcessingImg2Img(sd_model=m, c=torch.zeros(1), uc=torch.zeros(1), tiling=True)
    assert _run(monkeypatch, p) == [True]
    assert all(e.calls == [True] for e in _engines(m))
    assert m.unet.circular


def test_hires_pass_keeps_tiling(monkeypatch):
    from sdwebui_b200.processing import StableDiffusionProcessingTxt2Img

    m = _model(with_encoder=False)
    p = StableDiffusionProcessingTxt2Img(sd_model=m, c=torch.zeros(1), uc=torch.zeros(1), tiling=True, enable_hr=True)
    assert _run(monkeypatch, p) == [True, True]
    assert all(e.calls == [True] for e in _engines(m))


def test_repeated_calls_are_no_ops(monkeypatch):
    from sdwebui_b200.processing import StableDiffusionProcessingTxt2Img

    m = _model()
    for tiling in (True, True, None, False, False, True):
        _run(monkeypatch, StableDiffusionProcessingTxt2Img(sd_model=m, c=torch.zeros(1), uc=torch.zeros(1), tiling=tiling))
    assert all(e.calls == [True, False, True] for e in _engines(m))


def test_unet_keeps_tiling_across_reactivation():
    from sdwebui_b200.sd_unet import SdxeUnet

    su = SdxeUnet({}, dtype=torch.float16, device="cpu")
    su.set_circular(True)  # before activate(): remembered, applied to the engine activate() builds
    assert su.circular and su.engine is None


# ---- webui seams ----------------------------------------------------------------------------------------------------
def _stub_webui(monkeypatch, hijack):
    """A stub `modules` package with sd_unet / shared / devices / script_callbacks and, when `hijack` is not None,
    sd_hijack.model_hijack = hijack."""
    pkg = types.ModuleType("modules")
    cb = types.ModuleType("modules.script_callbacks")
    cb.registered = {}
    for name in ("on_list_unets", "on_list_optimizers", "on_model_loaded"):
        setattr(cb, name, lambda fn, *, name=None, _n=name: cb.registered.setdefault(_n, fn))
    shared = types.ModuleType("modules.shared")
    shared.device = torch.device("cpu")
    shared.opts = types.SimpleNamespace(hypertile_enable_vae=False, upcast_attn=False)
    shared.loaded_hypernetworks = []
    devices = types.ModuleType("modules.devices")
    devices.dtype_unet, devices.dtype_vae = torch.float16, torch.float16
    sd_unet = types.ModuleType("modules.sd_unet")

    class SdUnetOption:
        pass

    class SdUnet(torch.nn.Module):
        def activate(self):
            pass

        def deactivate(self):
            pass

    sd_unet.SdUnetOption, sd_unet.SdUnet = SdUnetOption, SdUnet
    sd_opt = types.ModuleType("modules.sd_hijack_optimizations")

    class SdOptimization:
        pass

    sd_opt.SdOptimization = SdOptimization
    stubs = {"modules": pkg, "modules.script_callbacks": cb, "modules.shared": shared, "modules.devices": devices,
             "modules.sd_unet": sd_unet, "modules.sd_hijack_optimizations": sd_opt}
    if hijack is not None:
        sdh = types.ModuleType("modules.sd_hijack")
        sdh.model_hijack = hijack
        stubs["modules.sd_hijack"] = sdh
        pkg.sd_hijack = sdh
    for k, v in stubs.items():
        if k != "modules":
            setattr(pkg, k.split(".")[-1], v)
        monkeypatch.setitem(sys.modules, k, v)
    if hijack is None:
        monkeypatch.setitem(sys.modules, "modules.sd_hijack", None)  # import fails
    return cb


@pytest.fixture()
def webui(monkeypatch):
    import sdwebui_b200  # noqa: F401
    from sdwebui_b200 import sd_hijack_optimizations as prod_opt
    from sdwebui_b200 import sd_unet as prod_unet

    def install(hijack):
        cb = _stub_webui(monkeypatch, hijack)
        importlib.reload(prod_unet)
        importlib.reload(prod_opt)
        spec = importlib.util.spec_from_file_location("sdxe_ext_tiling_under_test", EXT)
        ext = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(ext)
        return cb, ext, prod_unet

    yield install
    monkeypatch.undo()
    importlib.reload(prod_unet)
    importlib.reload(prod_opt)


def _webui_unet(prod_unet):
    su = prod_unet.SdxeUnet({}, dtype=torch.float16, device="cpu")
    eng = _FakeEngine()
    eng.forward = lambda *a, **k: "eps"
    su.engine = eng
    su.hypertile_rows = lambda h, w: None
    return su, eng


@pytest.mark.parametrize("attr", [True, False, "missing"])
def test_webui_unet_reads_circular_enabled_per_call(webui, attr):
    hijack = types.SimpleNamespace() if attr == "missing" else types.SimpleNamespace(circular_enabled=attr)
    _, _, prod_unet = webui(hijack)
    assert prod_unet.IN_WEBUI
    su, eng = _webui_unet(prod_unet)
    x = torch.zeros(1, 4, 8, 8)
    su.forward(x, torch.zeros(1), torch.zeros(1, 77, 8))
    if attr != "missing":
        hijack.circular_enabled = not attr  # apply_circular ran between two calls
    su.forward(x, torch.zeros(1), torch.zeros(1, 77, 8))
    # the engine follows every change (the flag is sticky on the engine: an unchanged state needs no call)
    assert eng.calls == ({True: [True, False], False: [True], "missing": []}[attr])
    assert su.circular == (False if attr == "missing" else not attr)


def test_webui_without_sd_hijack_is_off(webui):
    _, _, prod_unet = webui(None)
    su, eng = _webui_unet(prod_unet)
    su.circular = True  # left on by an earlier job
    su.forward(torch.zeros(1, 4, 8, 8), torch.zeros(1), torch.zeros(1, 77, 8))
    assert eng.calls == [False] and not su.circular


@pytest.mark.parametrize("attr", [True, "missing"])
def test_webui_vae_wrappers_read_circular_enabled_per_call(webui, attr):
    hijack = types.SimpleNamespace() if attr == "missing" else types.SimpleNamespace(circular_enabled=attr)
    cb, ext, _ = webui(hijack)
    made = []

    class FakeVae(_FakeEngine):
        def __init__(self, spec, dtype=None, device=None):
            super().__init__()
            made.append(self)

        def load_state_dict(self, sd):
            pass

        def finalize(self):
            pass

        def decode(self, z):
            return z

        def encode_moments(self, x):
            return torch.zeros(1, 8, 2, 2)

        def close(self):
            pass

    ext.VAEDecoderEngine, ext.VAEEncoderEngine = FakeVae, FakeVae
    ext.VAESpec = types.SimpleNamespace(from_state_dict=lambda sd: None)
    fs = types.SimpleNamespace(state_dict=lambda: {"decoder.x": 0, "encoder.x": 0}, decode=lambda z: "stock", encode=lambda x: "stock")
    cb.registered["on_model_loaded"](types.SimpleNamespace(first_stage_model=fs))
    dec, enc = made
    fs.decode(torch.zeros(1))
    fs.encode(torch.zeros(1))
    if attr != "missing":
        hijack.circular_enabled = False
    fs.decode(torch.zeros(1))
    fs.encode(torch.zeros(1))
    want = [False, False] if attr == "missing" else [True, False]
    assert dec.calls == want and enc.calls == want
