"""Python handles over the C-ABI engine objects (include/sdxe.h): UNetEngine and VAEDecoderEngine.

Torch supplies device memory and the current stream; all arithmetic runs in libsdxe.so. Weights are ingested by their
ldm state-dict keys (SURVEY Appendix A.3), so the same checkpoint dict that `shared.sd_model.model.diffusion_model`
exposes in the webui loads here unchanged (modules/sd_unet.py:54: the plugin must own its weights).
"""
from __future__ import annotations

import ctypes
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch

from . import lib as L


@dataclass
class UNetSpec:
    """Constructor arguments of ldm / sgm UNetModel (configs/v1-inference.yaml:29-44, configs/sd_xl_inpaint.yaml:19-37)."""

    in_channels: int = 4
    out_channels: int = 4
    model_channels: int = 320
    channel_mult: List[int] = field(default_factory=lambda: [1, 2, 4, 4])
    num_res_blocks: int = 2
    transformer_depth: List[int] = field(default_factory=lambda: [1, 1, 1, 0])
    num_heads: int = 8
    num_head_channels: int = -1
    context_dim: int = 768
    use_linear_in_transformer: bool = False
    adm_in_channels: int = 0
    middle_depth: int = 1

    @staticmethod
    def sd15() -> "UNetSpec":
        return UNetSpec()

    @staticmethod
    def sdxl() -> "UNetSpec":
        return UNetSpec(channel_mult=[1, 2, 4], transformer_depth=[0, 2, 10], num_heads=-1, num_head_channels=64,
                        context_dim=2048, use_linear_in_transformer=True, adm_in_channels=2816, middle_depth=10)

    @staticmethod
    def from_any(cfg) -> "UNetSpec":
        """Accepts any object with the same attribute names (e.g. a parsed webui yaml or a test config)."""
        return UNetSpec(**{k: (list(getattr(cfg, k)) if isinstance(getattr(cfg, k), (list, tuple)) else getattr(cfg, k))
                           for k in UNetSpec.__dataclass_fields__})


@dataclass
class VAESpec:
    """ddconfig of AutoencoderKL (configs/v1-inference.yaml:46-65)."""

    ch: int = 128
    out_ch: int = 3
    ch_mult: List[int] = field(default_factory=lambda: [1, 2, 4, 4])
    num_res_blocks: int = 2
    z_channels: int = 4

    @staticmethod
    def from_any(cfg) -> "VAESpec":
        return VAESpec(**{k: (list(getattr(cfg, k)) if isinstance(getattr(cfg, k), (list, tuple)) else getattr(cfg, k))
                          for k in VAESpec.__dataclass_fields__})

    @staticmethod
    def from_state_dict(sd) -> "VAESpec":
        """ddconfig read back from a `first_stage_model` state dict (decoder.* and / or encoder.* keys): the KL-f8 VAE of
        SD1.x / SDXL gives the defaults; anything the engine does not implement (attention outside the mid block, a
        z_channels != embed_dim pairing it cannot pack, ...) raises SdxeError so that callers keep the stock VAE."""
        side = "decoder" if any(k.startswith("decoder.") for k in sd) else "encoder"
        if f"{side}.conv_in.weight" not in sd:
            raise L.SdxeError("not an AutoencoderKL state dict (no conv_in)")
        levels = sorted({int(k.split(".")[2]) for k in sd if k.startswith(f"{side}.{'up' if side == 'decoder' else 'down'}.")})
        if not levels or levels != list(range(len(levels))):
            raise L.SdxeError("unrecognised VAE level layout")
        if any(".attn." in k and not k.startswith(f"{side}.mid.") for k in sd if k.startswith(side)):
            raise L.SdxeError("VAE with attention outside the mid block is not implemented")
        if side == "decoder":
            ch = sd["decoder.up.0.block.0.conv1.weight"].shape[0]
            mult = [sd[f"decoder.up.{l}.block.0.conv1.weight"].shape[0] // ch for l in levels]
            nres = len({int(k.split(".")[4]) for k in sd if k.startswith("decoder.up.0.block.")}) - 1
            z = sd["decoder.conv_in.weight"].shape[1]
            out_ch = sd["decoder.conv_out.weight"].shape[0]
        else:
            ch = sd["encoder.conv_in.weight"].shape[0]
            mult = [sd[f"encoder.down.{l}.block.0.conv1.weight"].shape[0] // ch for l in levels]
            nres = len({int(k.split(".")[4]) for k in sd if k.startswith("encoder.down.0.block.")})
            z = sd["encoder.conv_out.weight"].shape[0] // 2
            out_ch = sd["encoder.conv_in.weight"].shape[1]
        return VAESpec(ch=int(ch), out_ch=int(out_ch), ch_mult=[int(m) for m in mult], num_res_blocks=int(nres), z_channels=int(z))


def _dtype_code(dtype: torch.dtype) -> int:
    if dtype not in (torch.float16, torch.bfloat16):
        raise L.SdxeError("engine dtype must be torch.float16 or torch.bfloat16")
    return L.torch_dtype_code(dtype)


class _EngineBase:
    def __init__(self, cfg: L.SdxeConfig, dtype: torch.dtype, device):
        if not torch.cuda.is_available():
            raise L.SdxeError("no CUDA device: the sdxe engine has no CPU path")
        self.lib = L.load()
        self.dtype = dtype
        self.device = torch.device(device)
        self._h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            L.check(self.lib.sdxe_create(ctypes.byref(cfg), ctypes.byref(self._h)), "sdxe_create")
        self.finalized = False

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            with torch.cuda.device(self.device):
                self.lib.sdxe_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_weight(self, key: str, tensor: torch.Tensor):
        t = tensor.detach()
        if t.dtype not in (torch.float16, torch.bfloat16, torch.float32):
            t = t.float()
        t = t.contiguous()
        shape = (ctypes.c_int64 * max(1, t.ndim))(*t.shape)
        with torch.cuda.device(self.device):
            L.check(self.lib.sdxe_set_weight(self._h, key.encode(), L.ptr(t), L.torch_dtype_code(t.dtype), t.ndim, shape),
                    f"sdxe_set_weight({key})")

    def load_state_dict(self, sd: Dict[str, torch.Tensor], prefix: str = "", only: Optional[tuple] = None):
        """Ingest every tensor whose key starts with `prefix` (stripped), e.g. "model.diffusion_model." or
        "first_stage_model."; `only` optionally restricts to sub-prefixes."""
        n = 0
        for k, v in sd.items():
            if not k.startswith(prefix):
                continue
            kk = k[len(prefix):]
            if only is not None and not kk.startswith(only):
                continue
            self.set_weight(kk, v)
            n += 1
        return n

    def param_count(self) -> int:
        return int(self.lib.sdxe_param_count(self._h))

    def finalize(self):
        with torch.cuda.device(self.device):
            L.check(self.lib.sdxe_finalize(self._h), "sdxe_finalize")
        self.finalized = True

    PROFILE_KINDS = ("gemm", "conv3x3", "attention", "group_norm", "layer_norm", "other")

    def profile(self, enable: bool):
        L.check(self.lib.sdxe_profile(self._h, 1 if enable else 0), "sdxe_profile")

    def set_plan_cache(self, max_plans: int = 8, pool_limit_mb: int = 6144):
        """Bound the per-shape execution-plan cache (LRU) and the free activation pool kept after an eviction."""
        L.check(self.lib.sdxe_set_plan_cache(self._h, int(max_plans), int(pool_limit_mb)), "sdxe_set_plan_cache")

    def pool_stats(self):
        """(bytes held by the activation pool, number of cached plans)."""
        import ctypes

        n = ctypes.c_int64(0)
        b = self.lib.sdxe_pool_bytes(self._h, ctypes.byref(n))
        return int(b), int(n.value)

    def profile_read(self) -> dict:
        """{kind: {"ms", "flops", "bytes", "launches"}} accumulated since profile(True)."""
        out = {}
        for k, name in enumerate(self.PROFILE_KINDS):
            ms, fl, by, n = ctypes.c_double(), ctypes.c_double(), ctypes.c_double(), ctypes.c_int64()
            L.check(self.lib.sdxe_profile_read(self._h, k, ctypes.byref(ms), ctypes.byref(fl), ctypes.byref(by), ctypes.byref(n)),
                    "sdxe_profile_read")
            out[name] = {"ms": ms.value, "flops": fl.value, "bytes": by.value, "launches": n.value}
        return out

    def weight_blob(self) -> torch.Tensor:
        """The packed weight blob as a uint8 torch view (for the single NCCL broadcast at load)."""
        p, n = ctypes.c_void_p(), ctypes.c_int64()
        L.check(self.lib.sdxe_weight_blob(self._h, ctypes.byref(p), ctypes.byref(n)), "sdxe_weight_blob")
        return _as_tensor(p.value, n.value, self.device)


def _as_tensor(ptr: int, nbytes: int, device) -> torch.Tensor:
    """uint8 tensor aliasing device memory [ptr, ptr+nbytes) via __cuda_array_interface__."""

    class _Holder:
        pass

    h = _Holder()
    h.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}
    return torch.as_tensor(h, device=device)


class UNetEngine(_EngineBase):
    def __init__(self, spec: UNetSpec, dtype: torch.dtype = torch.float16, device="cuda:0"):
        cfg = L.SdxeConfig()
        cfg.kind = L.SDXE_MODEL_UNET
        cfg.dtype = _dtype_code(dtype)
        cfg.in_channels, cfg.out_channels, cfg.model_channels = spec.in_channels, spec.out_channels, spec.model_channels
        cfg.num_levels = len(spec.channel_mult)
        for i, m in enumerate(spec.channel_mult):
            cfg.channel_mult[i] = m
            cfg.transformer_depth[i] = spec.transformer_depth[i]
        cfg.num_res_blocks = spec.num_res_blocks
        cfg.num_heads = spec.num_heads if spec.num_heads and spec.num_heads > 0 else 0
        cfg.num_head_channels = spec.num_head_channels if spec.num_head_channels and spec.num_head_channels > 0 else 0
        cfg.context_dim = spec.context_dim
        cfg.use_linear_in_transformer = 1 if spec.use_linear_in_transformer else 0
        cfg.adm_in_channels = spec.adm_in_channels
        cfg.transformer_depth_middle = spec.middle_depth
        self.spec = spec
        super().__init__(cfg, dtype, device)

    def forward(self, x: torch.Tensor, timesteps: torch.Tensor, context: torch.Tensor, y: Optional[torch.Tensor] = None,
                out: Optional[torch.Tensor] = None, context_key: int = 0, hypertile=None) -> torch.Tensor:
        """eps = UNet(x, t, context[, y]); all tensors share x.dtype (fp16 / bf16 / fp32), x is [n,4,h,w] NCHW.
        `context_key` != 0: the caller's promise that `context` has the contents it had the last time this key was
        used — the cross-attention k | v projections are then reused (sdxe_unet_set_context_key).
        `hypertile`: rows (h', w', nh, nw, max_tiles), one per attn1 layer in execution order, tile this call's
        self-attention (sdxe_unet_set_hypertile); None leaves the call exactly as without Hypertile."""
        if not x.is_cuda:
            raise L.SdxeError("sdxe UNet needs CUDA tensors: there is no CPU fallback")
        dt = x.dtype
        x = x.contiguous()
        t = timesteps.to(dt).contiguous()
        ctx = context.to(dt).contiguous()
        yy = y.to(dt).contiguous() if y is not None else None
        n, _, h, w = x.shape
        if out is None:
            out = torch.empty_like(x)
        L.check(self.lib.sdxe_unet_set_context_key(self._h, int(context_key)), "sdxe_unet_set_context_key")
        if hypertile is not None:
            flat = [int(v) for row in hypertile for v in row]
            L.check(self.lib.sdxe_unet_set_hypertile(self._h, (ctypes.c_int32 * len(flat))(*flat), len(flat) // 5),
                    "sdxe_unet_set_hypertile")
        L.check(self.lib.sdxe_unet_forward(self._h, L.ptr(x), L.ptr(t), L.ptr(ctx), L.ptr(yy), L.ptr(out), n, h, w,
                                           ctx.shape[1], L.torch_dtype_code(dt), L.current_stream()), "sdxe_unet_forward")
        return out

    __call__ = forward


class VAEDecoderEngine(_EngineBase):
    def __init__(self, spec: VAESpec, dtype: torch.dtype = torch.float16, device="cuda:0"):
        cfg = L.SdxeConfig()
        cfg.kind = L.SDXE_MODEL_VAE_DECODER
        cfg.dtype = _dtype_code(dtype)
        cfg.num_levels = len(spec.ch_mult)
        for i, m in enumerate(spec.ch_mult):
            cfg.channel_mult[i] = m
        cfg.num_res_blocks = spec.num_res_blocks
        cfg.vae_ch, cfg.vae_z_channels, cfg.vae_out_ch = spec.ch, spec.z_channels, spec.out_ch
        self.spec = spec
        super().__init__(cfg, dtype, device)

    def load_state_dict(self, sd, prefix: str = "", only=("decoder.", "post_quant_conv.")):
        return super().load_state_dict(sd, prefix, only)

    def decode(self, z: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """AutoencoderKL.decode(z): z [n,4,h,w] (already / scale_factor) -> [n,3,8h,8w], same dtype as z."""
        if not z.is_cuda:
            raise L.SdxeError("sdxe VAE needs CUDA tensors: there is no CPU fallback")
        z = z.contiguous()
        n, _, h, w = z.shape
        up = 2 ** (len(self.spec.ch_mult) - 1)
        if out is None:
            out = torch.empty(n, self.spec.out_ch, h * up, w * up, dtype=z.dtype, device=z.device)
        L.check(self.lib.sdxe_vae_decode(self._h, L.ptr(z), L.ptr(out), n, h, w, L.torch_dtype_code(z.dtype),
                                         L.current_stream()), "sdxe_vae_decode")
        return out

    __call__ = decode


class VAEEncoderEngine(_EngineBase):
    """AutoencoderKL.encode up to the moments (encoder + quant_conv): the img2img / hires non-latent entry
    (modules/sd_samplers_common.py:87-112 images_tensor_to_samples -> model.encode_first_stage)."""

    def __init__(self, spec: VAESpec, dtype: torch.dtype = torch.float16, device="cuda:0"):
        cfg = L.SdxeConfig()
        cfg.kind = L.SDXE_MODEL_VAE_ENCODER
        cfg.dtype = _dtype_code(dtype)
        cfg.num_levels = len(spec.ch_mult)
        for i, m in enumerate(spec.ch_mult):
            cfg.channel_mult[i] = m
        cfg.num_res_blocks = spec.num_res_blocks
        cfg.vae_ch, cfg.vae_z_channels, cfg.vae_out_ch = spec.ch, spec.z_channels, spec.out_ch
        self.spec = spec
        super().__init__(cfg, dtype, device)

    def load_state_dict(self, sd, prefix: str = "", only=("encoder.", "quant_conv.")):
        return super().load_state_dict(sd, prefix, only)

    def encode_moments(self, x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """x [n,3,H,W] in [-1,1] -> moments [n, 2*z, H/f, W/f] (mean | logvar), same dtype as x."""
        if not x.is_cuda:
            raise L.SdxeError("sdxe VAE needs CUDA tensors: there is no CPU fallback")
        x = x.contiguous()
        n, _, h, w = x.shape
        f = 2 ** (len(self.spec.ch_mult) - 1)
        if out is None:
            out = torch.empty(n, 2 * self.spec.z_channels, h // f, w // f, dtype=x.dtype, device=x.device)
        L.check(self.lib.sdxe_vae_encode(self._h, L.ptr(x), L.ptr(out), n, h, w, L.torch_dtype_code(x.dtype),
                                         L.current_stream()), "sdxe_vae_encode")
        return out

    def encode(self, x: torch.Tensor, noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        """DiagonalGaussianDistribution(moments).sample() (ldm distributions.py: logvar clamped to [-30, 20],
        mean + exp(0.5 logvar) * noise); noise=None returns the mode (the mean), as `sd_vae_encode_method` "Mode"."""
        m = self.encode_moments(x).float()
        mean, logvar = torch.chunk(m, 2, dim=1)
        if noise is None:
            return mean
        return mean + torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0)) * noise.float()

    __call__ = encode_moments



@dataclass
class CLIPTextSpec:
    """transformers CLIPTextConfig as far as the text transformer needs it (CLIP-L defaults = SD1.x `cond_stage_model`)."""

    vocab_size: int = 49408
    hidden_size: int = 768
    intermediate_size: int = 3072
    num_layers: int = 12
    num_heads: int = 12
    max_positions: int = 77
    act: str = "quick_gelu"   # "gelu" for the OpenCLIP bigG tower of SDXL

    @staticmethod
    def from_any(cfg) -> "CLIPTextSpec":
        return CLIPTextSpec(**{k: getattr(cfg, k) for k in CLIPTextSpec.__dataclass_fields__ if hasattr(cfg, k)})

    @staticmethod
    def from_state_dict(sd, num_heads: Optional[int] = None, act: Optional[str] = None) -> "CLIPTextSpec":
        tok = sd["text_model.embeddings.token_embedding.weight"]
        layers = len({k.split(".")[3] for k in sd if k.startswith("text_model.encoder.layers.")})
        hidden = int(tok.shape[1])
        return CLIPTextSpec(vocab_size=int(tok.shape[0]), hidden_size=hidden,
                            intermediate_size=int(sd["text_model.encoder.layers.0.mlp.fc1.weight"].shape[0]), num_layers=layers,
                            num_heads=num_heads or hidden // 64, max_positions=int(sd["text_model.embeddings.position_embedding.weight"].shape[0]),
                            act=act or ("quick_gelu" if hidden == 768 else "gelu"))


class CLIPTextEngine(_EngineBase):
    """The text transformer behind `encode_with_transformers` (modules/sd_hijack_clip.py:351-360): token ids in, hidden
    states out. Weights by their Hugging Face names ("text_model.embeddings...", "text_model.encoder.layers.N...")."""

    def __init__(self, spec: CLIPTextSpec, dtype: torch.dtype = torch.float16, device="cuda:0"):
        cfg = L.SdxeConfig()
        cfg.kind = L.SDXE_MODEL_CLIP_TEXT
        cfg.dtype = _dtype_code(dtype)
        cfg.clip_vocab, cfg.clip_hidden, cfg.clip_intermediate = spec.vocab_size, spec.hidden_size, spec.intermediate_size
        cfg.clip_layers, cfg.clip_heads, cfg.clip_positions = spec.num_layers, spec.num_heads, spec.max_positions
        if spec.act not in ("quick_gelu", "gelu"):
            raise L.SdxeError(f"CLIP activation {spec.act!r} is not implemented")
        cfg.clip_act = 0 if spec.act == "quick_gelu" else 1
        self.spec = spec
        super().__init__(cfg, dtype, device)

    def load_state_dict(self, sd, prefix: str = "", only=("text_model.",)):
        sd = {k: v for k, v in sd.items() if "position_ids" not in k}
        return super().load_state_dict(sd, prefix, only)

    def forward(self, tokens: torch.Tensor, layer: Optional[int] = None, final_norm: bool = True,
                out_dtype: Optional[torch.dtype] = None, fixes=None) -> torch.Tensor:
        """tokens [n, T] integer -> hidden_states[layer] ([n, T, C]; layer = number of transformer layers applied, default
        all), through final_layer_norm when `final_norm`. Result in the engine's dtype (or fp32).
        `fixes`: textual-inversion replacements [(flat row = batch * T + position, vector [C]), ...] applied in order to the
        token embedding (modules/sd_hijack.py:340-366)."""
        if tokens.dim() != 2:
            raise L.SdxeError("tokens must be [n, T]")
        n, T = tokens.shape
        layer = self.spec.num_layers if layer is None else int(layer)
        ids = tokens.to(device=self.device, dtype=torch.int32).contiguous()
        odt = out_dtype or self.dtype
        out = torch.empty(n, T, self.spec.hidden_size, dtype=odt, device=self.device)
        rows = vecs = None
        n_fix = 0
        if fixes:
            for r, v in fixes:
                if not (0 <= int(r) < n * T) or v.numel() != self.spec.hidden_size:
                    raise L.SdxeError(f"textual-inversion fix: row {r} / vector of {v.numel()} values do not fit [{n} x {T}, {self.spec.hidden_size}]")
            rows = torch.tensor([int(r) for r, _ in fixes], dtype=torch.int32, device=self.device)
            vecs = torch.stack([v.reshape(-1) for _, v in fixes]).to(device=self.device, dtype=self.dtype).contiguous()
            n_fix = len(fixes)
        with torch.cuda.device(self.device):
            L.check(self.lib.sdxe_clip_forward_fixes(self._h, L.ptr(ids), L.ptr(out), n, T, layer, 1 if final_norm else 0,
                                                     L.torch_dtype_code(odt), L.ptr(rows), L.ptr(vecs), n_fix, L.current_stream()),
                    "sdxe_clip_forward_fixes")
        del rows, vecs
        return out

    __call__ = forward
