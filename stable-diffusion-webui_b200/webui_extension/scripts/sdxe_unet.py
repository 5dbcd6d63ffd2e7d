"""webui extension entry point (drop this directory into <webui>/extensions/sdxe/): registers the sdxe UNet and the
sdxe attention optimisation through the reference's own plugin callbacks:
  script_callbacks.on_list_unets       modules/script_callbacks.py:602-606  -> modules/sd_unet.py:10-14
  script_callbacks.on_list_optimizers  modules/script_callbacks.py:594-599  -> modules/sd_hijack.py:48-56
  script_callbacks.on_model_loaded     modules/script_callbacks.py:467      -> wraps first_stage_model.decode (B3) and
                                                                              first_stage_model.encode (img2img init, N1)
Nothing in the webui itself is modified.

What the callbacks guard against (a plugin that silently changes results or crashes the stock path is worse than none):
  * the UNet option is offered only for checkpoints the engine implements — eps-prediction SD1.x or SDXL-base with a
    4-channel latent input; SD2.x / v-prediction / inpainting (9-channel) / refiner checkpoints keep the stock UNet
    (with sd_unet = "Automatic", modules/sd_unet.py:22-27, an option named like the checkpoint is selected by itself);
  * LoRA / LyCORIS networks active at activation time are merged into the engine's weights (the stock merge patches
    the torch modules' weights, which the engine does not read: modules/sd_unet.py:54 moves the stock UNet away);
  * the VAE wrappers are rebuilt whenever model_loaded fires (it also fires after a VAE swap, modules/sd_vae.py:279),
    run in devices.dtype_vae (bf16 when the webui chose it for SDXL; an fp32 VAE — --no-half-vae — is left alone),
    and anything going wrong restores the stock decode / encode;
  * Hypertile (extensions-builtin/hypertile): the UNet's tiled self-attention runs on the engine, with the draws taken
    from the extension's own RNG in stock order (sd_unet.SdxeUnet.hypertile_rows); with Hypertile VAE on, decode and
    encode go to the stock VAE, which the engine VAE does not tile;
  * Tiling (modules/sd_hijack.py:311-318 apply_circular flips padding_mode on the stock Conv2d modules, which the engine
    never runs): the UNet and both VAE wrappers read model_hijack.circular_enabled on every call and set it on their
    engine (sd_unet.webui_circular; unreadable = off). With Hypertile VAE on, the stock VAE's flipped modules do it.
"""
import os
import sys

from modules import devices, script_callbacks, shared  # type: ignore

_ROOT = os.environ.get("SDXE_ROOT", os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)

import sdwebui_b200  # noqa: E402,F401
import torch  # noqa: E402

from sdwebui_b200.engine import VAEDecoderEngine, VAEEncoderEngine, VAESpec  # noqa: E402
from sdwebui_b200.lib import SdxeError  # noqa: E402
from sdwebui_b200.sd_hijack_optimizations import SdOptimizationSdxe  # noqa: E402
from sdwebui_b200.sd_unet import SdxeUnetOption, guess_unet_spec, webui_circular  # noqa: E402


def supported_unet_spec(sd_model):
    """UNetSpec when the loaded checkpoint is one the engine implements, else None (the stock UNet keeps running)."""
    if getattr(sd_model, "parameterization", "eps") != "eps":            # v-prediction (SD2.x 768, some fine-tunes)
        return None
    if getattr(sd_model, "is_sd2", False) or getattr(sd_model, "is_sd3", False) or getattr(sd_model, "is_sdxl_inpaint", False):
        return None
    if getattr(getattr(sd_model, "model", None), "conditioning_key", "crossattn") not in (None, "crossattn"):
        return None                                                     # inpainting / instruct-pix2pix ("hybrid", "concat")
    try:
        sd = sd_model.model.diffusion_model.state_dict()
        if sd["input_blocks.0.0.weight"].shape[1] != 4:                 # 9-channel inpainting UNet
            return None
        return guess_unet_spec(sd)                                      # raises for anything but SD1.x / SDXL-base layouts
    except (SdxeError, KeyError, AttributeError):
        return None


def active_loras():
    """[(state_dict, unet_multiplier)] of the networks the built-in Lora extension currently has loaded."""
    try:
        import networks  # type: ignore  (extensions-builtin/Lora/networks.py)
    except ImportError:
        return []
    from sdwebui_b200.sd_models import read_state_dict

    out = []
    for net in getattr(networks, "loaded_networks", []):
        fn = getattr(getattr(net, "network_on_disk", None), "filename", None)
        if fn:
            out.append((read_state_dict(fn), float(getattr(net, "unet_multiplier", 1.0))))
    return out


def _list_unets(unets):
    sd_model = shared.sd_model
    info = getattr(sd_model, "sd_checkpoint_info", None)
    if info is None:
        return
    spec = supported_unet_spec(sd_model)
    if spec is None:
        return
    unets.append(SdxeUnetOption(info.model_name, lambda: sd_model.model.diffusion_model.state_dict(), spec=spec,
                                dtype=devices.dtype_unet if devices.dtype_unet in (torch.float16, torch.bfloat16) else torch.float16,
                                device=shared.device, loras_provider=active_loras))


def _list_optimizers(optimizers):
    optimizers.append(SdOptimizationSdxe())


def _restore_vae(fs):
    for name in ("decode", "encode"):
        orig = fs.__dict__.pop(f"_sdxe_orig_{name}", None)
        if orig is not None:
            setattr(fs, name, orig)
    for eng in fs.__dict__.pop("_sdxe_engines", []):
        eng.close()


def _hypertile_vae():
    return bool(getattr(shared.opts, "hypertile_enable_vae", False))


def _tiled(eng):
    """`eng` with the webui's current Tiling state applied (apply_circular may have changed it since the last call)."""
    eng.set_circular(webui_circular())
    return eng


def _model_loaded(sd_model):
    fs = getattr(sd_model, "first_stage_model", None)
    if fs is None:
        return
    _restore_vae(fs)  # a previous wrap (other checkpoint, or the same one before a VAE swap) is undone first
    dtype = devices.dtype_vae
    if dtype not in (torch.float16, torch.bfloat16):
        return  # --no-half-vae / fp32 VAE: the engine is 16-bit, the stock modules keep running
    engines = []
    try:
        sd = fs.state_dict()
        dsd = {k: v for k, v in sd.items() if k.startswith(("decoder.", "post_quant_conv."))}
        spec = VAESpec.from_state_dict(dsd)
        dec = VAEDecoderEngine(spec, dtype=dtype, device=shared.device)
        engines.append(dec)
        dec.load_state_dict(dsd)
        dec.finalize()
        fs._sdxe_orig_decode = orig_decode = fs.decode
        # precedent for patching these methods: modules/lowvram.py:64-74,136-137. With Hypertile VAE on, the stock
        # decode runs: its hooks tile the VAE attention and draw from Hypertile's RNG, which the engine VAE does not do
        fs.decode = lambda z, *a, **k: orig_decode(z, *a, **k) if _hypertile_vae() else _tiled(dec).decode(z)
        esd = {k: v for k, v in sd.items() if k.startswith(("encoder.", "quant_conv."))}
        if esd:
            enc = VAEEncoderEngine(spec, dtype=dtype, device=shared.device)
            engines.append(enc)
            enc.load_state_dict(esd)
            enc.finalize()
            fs._sdxe_orig_encode = orig_encode = fs.encode
            fs.encode = lambda x, *a, **k: orig_encode(x, *a, **k) if _hypertile_vae() else _Posterior(_tiled(enc).encode_moments(x))
        fs._sdxe_engines = engines
    except Exception as ex:  # noqa: BLE001  unknown VAE layout, out of memory, ...: the stock VAE stays in place
        fs._sdxe_engines = engines
        _restore_vae(fs)
        print(f"[sdxe] VAE not accelerated ({type(ex).__name__}: {ex}); using the stock VAE")


class _Posterior:
    """What ldm's AutoencoderKL.encode returns (DiagonalGaussianDistribution), as far as get_first_stage_encoding and
    images_tensor_to_samples (modules/sd_samplers_common.py:87-112) use it: sample() / mode()."""

    def __init__(self, moments):
        self.mean, self.logvar = torch.chunk(moments.float(), 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def sample(self):
        return self.mean + self.std * torch.randn(self.mean.shape, device=self.mean.device)

    def mode(self):
        return self.mean


script_callbacks.on_list_unets(_list_unets)
script_callbacks.on_list_optimizers(_list_optimizers)
script_callbacks.on_model_loaded(_model_loaded)
