"""The drop-in attention seam: one `SdOptimization` (modules/sd_hijack_optimizations.py:25-48) whose apply() installs
sdxe-backed `CrossAttention.forward` and `AttnBlock.forward`, replacing every variant the reference ships
(xformers / sdp / sdp-no-mem / sub-quadratic / V1 / InvokeAI / Doggettx, :51-143).

Used for the VAE AttnBlock (not covered by the SdUnet seam) and as a per-layer path when the stock UNet stays active.
Inside the webui it subclasses the real `SdOptimization` and is registered through `on_list_optimizers`; headless,
`apply(classes=...)` patches whatever module classes the caller hands over (tests patch structural twins).
"""
from __future__ import annotations

import torch

from . import ops
from .lib import SdxeError

try:
    from modules import sd_hijack_optimizations as _ref  # type: ignore

    _Base = _ref.SdOptimization
except Exception:
    _ref = None

    class _Base:  # structural twin of sd_hijack_optimizations.py:25-48
        name: str = None
        label = None
        cmd_opt = None
        priority: int = 0

        def title(self):
            return self.name if self.label is None else f"{self.name} - {self.label}"

        def is_available(self):
            return True

        def apply(self):
            pass

        def undo(self):
            pass


def _webui_state():
    """(loaded hypernetworks, apply_hypernetworks, upcast_attn) from the running webui; ([], None, False) headless."""
    try:
        from modules import shared  # type: ignore
        from modules.hypernetworks import hypernetwork  # type: ignore

        return (getattr(shared, "loaded_hypernetworks", []), hypernetwork.apply_hypernetworks,
                bool(getattr(getattr(shared, "opts", None), "upcast_attn", False)))
    except Exception:
        return [], None, False


def _check_upcast(upcast):
    if upcast:  # the reference computes q k v in fp32 then (:530-532); this kernel is 16-bit by construction
        raise SdxeError('"Upcast cross attention layer to float32" is on: the sdxe attention kernels are 16-bit only — '
                        "turn the option off or pick another cross-attention optimization")


def sdxe_attention_forward(self, x, context=None, mask=None, **kwargs):
    """CrossAttention.forward — same contract as scaled_dot_product_attention_forward (:508-546): x [B,N,C],
    optional context [B,Nk,Cctx]; uses self.heads / to_q / to_k / to_v / to_out; hypernetworks are applied to the
    context like every reference variant does (:519). Masks are not supported (the webui never passes one on this
    path); upcast_attn raises."""
    if mask is not None:
        raise NotImplementedError("sdxe attention: attention masks are not supported")
    hypernets, apply_hn, upcast = _webui_state()
    _check_upcast(upcast)
    b, n, inner = x.shape
    h = self.heads
    q_in = self.to_q(x)
    context = x if context is None else context
    context_k, context_v = apply_hn(hypernets, context) if apply_hn is not None else (context, context)
    k_in = self.to_k(context_k)
    v_in = self.to_v(context_v)
    d = q_in.shape[-1] // h
    q = q_in.view(b, -1, h, d).transpose(1, 2)
    k = k_in.view(b, -1, h, d).transpose(1, 2)
    v = v_in.view(b, -1, h, d).transpose(1, 2)
    dt = q.dtype
    if dt not in (torch.float16, torch.bfloat16):
        q, k, v = q.half(), k.half(), v.half()
    out = ops.attention(q, k, v).to(dt)  # [b, n, h*d]
    out = self.to_out[0](out)
    return self.to_out[1](out)


def sdxe_attnblock_forward(self, x):
    """VAE AttnBlock.forward — contract of sdp_attnblock_forward (:637-655): x [B,C,H,W], self.norm/q/k/v/proj_out."""
    _check_upcast(_webui_state()[2])
    h_ = self.norm(x)
    q, k, v = self.q(h_), self.k(h_), self.v(h_)
    b, c, hh, ww = q.shape
    q, k, v = (t.reshape(b, c, hh * ww).transpose(1, 2).unsqueeze(1).contiguous() for t in (q, k, v))  # [b,1,hw,c]
    dt = q.dtype
    if dt not in (torch.float16, torch.bfloat16):
        q, k, v = q.half(), k.half(), v.half()
    out = ops.attention(q, k, v).to(dt)  # [b, hw, c]
    out = out.transpose(1, 2).reshape(b, c, hh, ww)
    return x + self.proj_out(out)


class SdOptimizationSdxe(_Base):
    name = "sdxe"
    label = "H100 wgmma flash attention"
    cmd_opt = "opt_sdxe_attention"
    # below the stock CUDA choices (xformers 100, Doggettx 90, sdp-no-mem 80, sdp 70; :51-143): "Automatic" keeps the
    # reference's behaviour, the user opts in through Settings -> Cross attention optimization -> sdxe. (The UNet seam,
    # sd_unet.SdxeUnet, replaces these per-layer calls wholesale; this optimizer is for the VAE AttnBlock and for
    # checkpoints the engine does not implement.)
    priority = 60

    def __init__(self):
        self._saved = []

    def is_available(self):
        # libsdxe.so holds sm_90a code only: it runs on Hopper (compute capability 9.0) and nothing else
        return torch.cuda.is_available() and torch.cuda.get_device_capability() == (9, 0)

    def apply(self, classes=None):
        """classes: optional {"CrossAttention": [cls...], "AttnBlock": [cls...]}; default = ldm + sgm classes."""
        if classes is None:
            import ldm.modules.attention  # type: ignore
            import ldm.modules.diffusionmodules.model  # type: ignore
            import sgm.modules.attention  # type: ignore
            import sgm.modules.diffusionmodules.model  # type: ignore

            classes = {
                "CrossAttention": [ldm.modules.attention.CrossAttention, sgm.modules.attention.CrossAttention],
                "AttnBlock": [ldm.modules.diffusionmodules.model.AttnBlock, sgm.modules.diffusionmodules.model.AttnBlock],
            }
        for cls in classes.get("CrossAttention", []):
            self._saved.append((cls, cls.forward))
            cls.forward = sdxe_attention_forward
        for cls in classes.get("AttnBlock", []):
            self._saved.append((cls, cls.forward))
            cls.forward = sdxe_attnblock_forward

    def undo(self):
        for cls, fwd in reversed(self._saved):
            cls.forward = fwd
        self._saved.clear()
