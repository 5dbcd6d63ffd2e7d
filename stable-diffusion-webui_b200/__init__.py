"""stable-diffusion-webui_b200 — an H100-native (sm_90a) denoising engine that plugs in behind
AUTOMATIC1111/stable-diffusion-webui's own seams (modules/sd_unet.py, modules/sd_hijack_optimizations.py,
modules/processing.process_images). Import as `sdwebui_b200` (see ../sdwebui_b200.py).

Only what the hot path needs lives here: csrc/ (CUDA kernels + the C-ABI, built into libsdxe.so) and the host-side
mirror of the reference's plugin interfaces. There is no CPU path.
"""
from . import lib  # noqa: F401

__all__ = ["lib"]
