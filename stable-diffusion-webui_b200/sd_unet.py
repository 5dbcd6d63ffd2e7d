"""The drop-in UNet seam: `SdUnetOption` / `SdUnet` exactly as modules/sd_unet.py:63-83 defines them, backed by the
sdxe engine. Inside a running webui these classes subclass the real `modules.sd_unet` types and are registered with
`script_callbacks.on_list_unets` (see webui_extension/scripts/sdxe_unet.py and INTEGRATION.md); headless (tests, bench,
the pipeline in this package) the same classes run against the structural twins below.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import hypertile as HT
from . import lib as L
from .engine import UNetEngine, UNetSpec

try:  # inside the webui process
    from modules import sd_unet as _ref_sd_unet  # type: ignore

    _SdUnetOptionBase = _ref_sd_unet.SdUnetOption
    _SdUnetBase = _ref_sd_unet.SdUnet
    IN_WEBUI = True
except Exception:  # headless: structural twins of modules/sd_unet.py:63-83
    IN_WEBUI = False

    class _SdUnetOptionBase:
        model_name = None
        label = None

        def create_unet(self):
            raise NotImplementedError()

    class _SdUnetBase(torch.nn.Module):
        def forward(self, x, timesteps, context, *args, **kwargs):
            raise NotImplementedError()

        def activate(self):
            pass

        def deactivate(self):
            pass


def webui_circular() -> bool:
    """The webui's Tiling state: modules.sd_hijack.model_hijack.circular_enabled, which apply_circular sets
    (modules/sd_hijack.py:311-318, from modules/processing.py:895). Unreadable means off, as in a webui where
    apply_circular never ran."""
    try:
        from modules import sd_hijack  # type: ignore

        return bool(sd_hijack.model_hijack.circular_enabled)
    except Exception:
        return False


def guess_unet_spec(state_dict: Dict[str, torch.Tensor]) -> UNetSpec:
    """Architecture from the checkpoint's own keys (the webui guesses from keys too: sd_models_config.py:72-114)."""
    if "label_emb.0.0.weight" in state_dict:
        w0 = state_dict.get("input_blocks.0.0.weight")
        wk = state_dict.get("input_blocks.4.1.transformer_blocks.0.attn2.to_k.weight")
        if w0 is None or w0.shape[1] != 4 or wk is None or wk.shape[1] != 2048 or state_dict["label_emb.0.0.weight"].shape[1] != 2816:
            raise L.SdxeError("SDXL-like checkpoint the engine does not implement (inpainting / refiner layout)")
        return UNetSpec.sdxl()
    w = state_dict.get("input_blocks.1.1.transformer_blocks.0.attn2.to_k.weight")
    w0 = state_dict.get("input_blocks.0.0.weight")
    if w is not None and w0 is not None and w.shape[1] == 768 and w0.shape[0] == 320 and w0.shape[1] == 4:
        return UNetSpec.sd15()
    raise L.SdxeError("unrecognised UNet checkpoint layout: pass an explicit UNetSpec")


class SdxeUnet(_SdUnetBase):
    """SdUnet whose forward is `sdxe_unet_forward`. Owns its weights (modules/sd_unet.py:54 moves the stock UNet away)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], spec: Optional[UNetSpec] = None, dtype=torch.float16,
                 device="cuda:0", prefix: str = "", loras=None):
        """`loras`: [(lora_state_dict, unet_multiplier), ...] merged into the weights at activate() — the reference
        merges lazily inside the stock modules, which a weight-snapshotting SdUnet would never see (SURVEY N3)."""
        super().__init__()
        self._sd = state_dict
        self._prefix = prefix
        self.loras = list(loras or [])
        self.lora_reports = []
        self.spec = spec
        self.dtype = dtype
        self.device_ = torch.device(device)
        self.engine: Optional[UNetEngine] = None
        # headless Hypertile state of the running job (processing.process_images sets it); in the webui the extension's
        # hooks on the stock modules are read instead
        self.hypertile: Optional[HT.HypertileState] = None
        self._webui_ht_cache = {}
        # headless Tiling state (SdModel.apply_circular); in the webui model_hijack.circular_enabled is read per call
        self.circular = False

    def activate(self):
        if self.engine is not None:
            return
        sd = {k[len(self._prefix):]: v for k, v in self._sd.items() if k.startswith(self._prefix)}
        spec = self.spec or guess_unet_spec(sd)
        if self.loras:
            from .extra_networks_lora import merge_loras

            sd, self.lora_reports = merge_loras(sd, self.loras)
        eng = UNetEngine(spec, dtype=self.dtype, device=self.device_)
        eng.load_state_dict(sd)
        eng.finalize()
        eng.set_circular(self.circular)
        self.engine = eng
        self._sd = None  # the engine holds the packed copy

    def set_circular(self, enable: bool):
        """Tiling on the engine (sdxe_set_circular), kept across deactivate() / activate()."""
        self.circular = bool(enable)
        if self.engine is not None:
            self.engine.set_circular(self.circular)

    def deactivate(self):
        if self.engine is not None:
            self.engine.close()
            self.engine = None

    def forward(self, x, timesteps, context, *args, **kwargs):
        """Called as UNetModel.forward would be: (x, timesteps, context) for ldm, (x, timesteps=, context=, y=) for sgm
        (modules/sd_unet.py:87-91). Accepts any leading batch size; tensors arrive in devices.dtype_unet."""
        if self.engine is None:
            raise L.SdxeError("SdxeUnet.forward before activate()")
        y = kwargs.get("y", args[0] if args else None)
        if IN_WEBUI:  # the stock convs whose padding_mode apply_circular flipped never run: carry the flag to the engine
            circular = webui_circular()
            if circular != self.circular:
                self.set_circular(circular)
        # context_key: only the package's own CFGDenoiser passes one (it knows the conditioning is step-invariant);
        # called from the stock webui the key is 0 and nothing is cached across calls
        return self.engine.forward(x, timesteps, context, y, context_key=int(kwargs.get("context_key", 0)),
                                   hypertile=self.hypertile_rows(x.shape[-2], x.shape[-1]))

    def hypertile_rows(self, h: int, w: int):
        """This call's Hypertile rows (h', w', nh, nw, max_tiles) per attn1 layer, drawn in stock execution order, or None.
        Every UNet call passes through here, so the draws advance the RNG exactly as the stock hooked modules would."""
        if IN_WEBUI:
            try:
                import hypertile as webui_ht  # extensions-builtin/hypertile/hypertile.py (its RNG_INSTANCE)
                from modules import shared  # type: ignore

                model = shared.sd_model.model
            except Exception:  # no Hypertile extension (or no model): nothing is tiled
                return None
            st = HT.webui_state(self.engine.spec, model, self._webui_ht_cache)
            return st.draw_rows(h, w, webui_ht.random_divisor, webui_ht.find_hw_candidates) if st is not None else None
        return self.hypertile.draw_rows(h, w) if self.hypertile is not None else None


class SdxeUnetOption(_SdUnetOptionBase):
    def __init__(self, model_name: str, state_dict_provider, spec: Optional[UNetSpec] = None, dtype=torch.float16,
                 device="cuda:0", prefix: str = "", loras_provider=None):
        self.model_name = model_name          # "Automatic" picks this option when the checkpoint name matches
        self.label = f"[sdxe] {model_name}"
        self._provider = state_dict_provider  # callable -> state dict (read lazily, at create_unet time)
        self._loras = loras_provider          # callable -> [(lora state dict, unet multiplier)] active at activation time
        self._spec, self._dtype, self._device, self._prefix = spec, dtype, device, prefix

    def create_unet(self):
        loras = self._loras() if self._loras is not None else None
        return SdxeUnet(self._provider(), self._spec, self._dtype, self._device, self._prefix, loras=loras)
