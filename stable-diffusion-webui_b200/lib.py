"""ctypes binding of libsdxe.so — the C-ABI declared in include/sdxe.h.

There is no fallback: if the shared library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsdxe.so")

SDXE_F16, SDXE_BF16, SDXE_F32 = 0, 1, 2
SDXE_MODEL_UNET, SDXE_MODEL_VAE_DECODER, SDXE_MODEL_VAE_ENCODER, SDXE_MODEL_CLIP_TEXT = 0, 1, 2, 3
SDXE_MAX_LEVELS = 8


class SdxeError(RuntimeError):
    pass


class SdxeConfig(ctypes.Structure):
    """Mirror of `struct sdxe_config` (include/sdxe.h)."""

    _fields_ = [
        ("kind", c_int32),
        ("dtype", c_int32),
        ("in_channels", c_int32),
        ("out_channels", c_int32),
        ("model_channels", c_int32),
        ("num_levels", c_int32),
        ("channel_mult", c_int32 * SDXE_MAX_LEVELS),
        ("num_res_blocks", c_int32),
        ("transformer_depth", c_int32 * SDXE_MAX_LEVELS),
        ("num_heads", c_int32),
        ("num_head_channels", c_int32),
        ("context_dim", c_int32),
        ("use_linear_in_transformer", c_int32),
        ("adm_in_channels", c_int32),
        ("transformer_depth_middle", c_int32),
        ("vae_ch", c_int32),
        ("vae_z_channels", c_int32),
        ("vae_out_ch", c_int32),
        ("clip_vocab", c_int32),
        ("clip_hidden", c_int32),
        ("clip_intermediate", c_int32),
        ("clip_layers", c_int32),
        ("clip_heads", c_int32),
        ("clip_positions", c_int32),
        ("clip_act", c_int32),
        ("reserved", c_int32 * 1),
    ]


# every symbol include/sdxe.h declares: name -> (restype, argtypes)
SYMBOLS = {
    "sdxe_last_error": (c_char_p, []),
    "sdxe_version": (c_int, []),
    "sdxe_launch_count": (c_int64, []),
    "sdxe_create": (c_int, [POINTER(SdxeConfig), POINTER(c_void_p)]),
    "sdxe_destroy": (None, [c_void_p]),
    "sdxe_set_weight": (c_int, [c_void_p, c_char_p, c_void_p, c_int, c_int, POINTER(c_int64)]),
    "sdxe_param_count": (c_int64, [c_void_p]),
    "sdxe_finalize": (c_int, [c_void_p]),
    "sdxe_weight_blob": (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_int64)]),
    "sdxe_unet_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "sdxe_vae_decode": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "sdxe_vae_encode": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "sdxe_clip_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "sdxe_clip_forward_fixes": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    "sdxe_unet_set_context_key": (c_int, [c_void_p, c_int64]),
    "sdxe_unet_set_hypertile": (c_int, [c_void_p, POINTER(c_int32), c_int]),
    "sdxe_set_plan_cache": (c_int, [c_void_p, c_int, c_int64]),
    "sdxe_pool_bytes": (c_int64, [c_void_p, POINTER(c_int64)]),
    "sdxe_profile": (c_int, [c_void_p, c_int]),
    "sdxe_profile_read": (c_int, [c_void_p, c_int, POINTER(ctypes.c_double), POINTER(ctypes.c_double), POINTER(ctypes.c_double), POINTER(c_int64)]),
    "sdxe_attention": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_int, c_void_p]),
    "sdxe_hypertile_attention": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_int, c_void_p]),
    "sdxe_gemm": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "sdxe_conv3x3_nhwc": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "sdxe_group_norm_nhwc": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_int, c_int, c_void_p]),
    "sdxe_layer_norm": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_int, c_void_p]),
    "sdxe_denoiser_in": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int64, c_int, c_void_p]),
    "sdxe_cfg_combine": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_int, c_int64, c_int, c_void_p]),
    "sdxe_cfg_combine_multi": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int64, c_int, c_void_p]),
    "sdxe_cfg_combine_affine": (c_int, [c_void_p] * 12 + [c_int, c_int64, c_int, c_void_p]),
    "sdxe_lincomb": (c_int, [c_void_p, c_void_p, c_float, c_void_p, c_float, c_void_p, c_float, c_void_p, c_float, c_int64, c_void_p]),
    "sdxe_euler_ancestral_step": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_float, c_float, c_int64, c_void_p]),
    "sdxe_dpmpp_2m_step": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_float, c_float, c_float, c_int64, c_void_p]),
}

_lib = None


def load() -> ctypes.CDLL:
    """Load libsdxe.so (once). Raises SdxeError when it has not been built — there is no CPU path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SdxeError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). This engine has no CPU or PyTorch fallback."
        )
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().sdxe_last_error()
        raise SdxeError(f"{what} failed (rc={rc}): {msg.decode() if msg else '?'}")


def torch_dtype_code(dt) -> int:
    import torch

    if dt == torch.float16:
        return SDXE_F16
    if dt == torch.bfloat16:
        return SDXE_BF16
    if dt == torch.float32:
        return SDXE_F32
    raise SdxeError(f"unsupported dtype {dt}")


def ptr(t) -> c_void_p:
    """Device (or host) pointer of a contiguous torch tensor; None -> NULL."""
    if t is None:
        return c_void_p(0)
    if not t.is_contiguous():
        raise SdxeError("tensor must be contiguous")
    return c_void_p(t.data_ptr())


def current_stream() -> c_void_p:
    import torch

    return c_void_p(torch.cuda.current_stream().cuda_stream)
