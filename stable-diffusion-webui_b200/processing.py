"""Host-side mirror of the reference pipeline boundary for the accelerated path (boundary A, SURVEY §8(b)):

  StableDiffusionProcessingTxt2Img     modules/processing.py:1166-1555  (fields used on the hot path only)
  process_images(p) -> Processed       modules/processing.py:819-1112
  decode_latent_batch                  modules/processing.py:625-672
  SdModel.apply_model                  LatentDiffusion.apply_model as patched by modules/sd_hijack_unet.py:40-54
                                       (+ DiffusionWrapper, modules/models/diffusion/ddpm_edit.py:1417-1437;
                                        SDXL: modules/sd_models_xl.py:37-43)

PNG/infotext, scripts and the UI are outside the accelerated path. Conditionings arrive either as tensors / containers
(what `p.setup_conds()` leaves in p.c / p.uc) or as prompts: with `prompts` set and a conditioner attached to the model,
`setup_conds()` (modules/processing.py:460-506, 1498-1542) builds p.c / p.uc / p.hr_c / p.hr_uc itself — prompt editing,
alternation and AND-composition through prompt_parser, text encoders on the engine. Images leave as a uint8 tensor.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import torch

from . import hypertile as HT
from . import lib as L
from . import prompt_parser
from . import samplers as S
from .engine import VAEDecoderEngine
from .rng import ImageRNG
from .sd_unet import SdxeUnet

opt_C, opt_f = 4, 8  # modules/processing.py:39-40


class SdModel:
    """What the hot path needs of `shared.sd_model`: the (replacement) UNet, the VAE decoder, the noise schedule."""

    def __init__(self, unet: SdxeUnet, vae: Optional[VAEDecoderEngine], is_sdxl: bool, dtype_unet=torch.float16,
                 device="cuda:0", scale_factor: Optional[float] = None, vae_encoder=None):
        self.unet = unet
        self.vae = vae
        self.vae_encoder = vae_encoder  # engine.VAEEncoderEngine, only needed by img2img
        self.is_sdxl = is_sdxl
        self.dtype_unet = dtype_unet
        self.dtype_vae = dtype_unet
        self.device = torch.device(device)
        self.scale_factor = scale_factor if scale_factor is not None else (0.13025 if is_sdxl else 0.18215)
        self.alphas_cumprod = S.make_alphas_cumprod().to(self.device)
        self.parameterization = "eps"
        # the conditioner (N4): SD1.x — a TextConditionalModel (sd_hijack_clip.FrozenCLIPEmbedderWithCustomWords); SDXL — the pair
        # (FrozenCLIPEmbedderForSDXLWithCustomWords, FrozenOpenCLIPEmbedder2WithCustomWords). None: conds must arrive as tensors.
        self.cond_stage_model = None
        self.sdxl_crop_top, self.sdxl_crop_left = 0, 0   # opts.sdxl_crop_top / sdxl_crop_left

    def get_learned_conditioning(self, texts):
        """LatentDiffusion.get_learned_conditioning (`cond_stage_model(texts)`); SDXL: modules/sd_models_xl.py:12-34 — width /
        height / is_negative_prompt travel on the SdConditioning list."""
        if self.cond_stage_model is None:
            raise L.SdxeError("no text encoder attached to the model (set SdModel.cond_stage_model or pass conds as tensors)")
        if not self.is_sdxl:
            return self.cond_stage_model(texts)
        from .sd_hijack_clip import sdxl_get_learned_conditioning

        clip_l, clip_g = self.cond_stage_model
        return sdxl_get_learned_conditioning(clip_l, clip_g, list(texts), width=getattr(texts, "width", None) or 1024,
                                             height=getattr(texts, "height", None) or 1024, crop_top=self.sdxl_crop_top,
                                             crop_left=self.sdxl_crop_left, is_negative_prompt=getattr(texts, "is_negative_prompt", False))

    def apply_model(self, x_noisy, t, cond=None, **kwargs):
        """cast to dtype_unet, call the UNet through the SdUnet seam (sd_hijack_unet.py:40-54)."""
        ctx = cond["crossattn"] if isinstance(cond, dict) else cond
        vec = cond.get("vector") if isinstance(cond, dict) else None
        return self.apply_model_scaled(x_noisy.to(self.dtype_unet), t, ctx, vec)

    def apply_model_scaled(self, x_in, t, context, vector=None, context_key: int = 0):
        dt = self.dtype_unet
        kwargs = {}
        if context_key:
            kwargs["context_key"] = context_key
        if vector is not None:
            kwargs["y"] = vector.to(dt)
        return self.unet.forward(x_in, t.to(dt), context.to(dt), **kwargs)

    def decode_first_stage(self, z):
        """z already divided by scale_factor upstream? No: the reference's decode_first_stage divides
        (ddpm_edit.py:726-784: z = 1/scale_factor * z). Same here."""
        if self.vae is None:
            raise L.SdxeError("no VAE decoder engine attached")
        return self.vae.decode((z.to(self.dtype_vae) / self.scale_factor).contiguous())


    # ldm LatentDiffusion.encode_first_stage / get_first_stage_encoding: moments -> scale_factor * sample
    def encode_first_stage(self, x):
        if self.vae_encoder is None:
            raise L.SdxeError("no VAE encoder engine attached (img2img needs one)")
        return self.vae_encoder.encode_moments(x.to(self.dtype_vae).contiguous())

    def get_first_stage_encoding(self, moments, noise=None):
        m = moments.float()
        mean, logvar = torch.chunk(m, 2, dim=1)
        if noise is None:  # reference: DiagonalGaussianDistribution.sample() draws from the GLOBAL torch RNG
            noise = torch.randn(mean.shape, device=mean.device, dtype=torch.float32)
        z = mean + torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0)) * noise.float()
        return self.scale_factor * z


def images_tensor_to_samples(image: torch.Tensor, model: SdModel, noise: Optional[torch.Tensor] = None) -> torch.Tensor:
    """modules/sd_samplers_common.py:87-112 ("Full" VAE encode method): image [B,3,H,W] in [0,1] -> latent [B,4,H/8,W/8].
    The reference encodes image by image; the engine takes the batch (per-sample norms / attention: same result).
    `noise` pins the posterior sample (the reference's comes from the global RNG — SURVEY N1 calls this a parity hazard)."""
    x = image.to(model.device, dtype=model.dtype_vae) * 2 - 1
    return model.get_first_stage_encoding(model.encode_first_stage(x), noise)


@dataclass
class StableDiffusionProcessingTxt2Img:
    sd_model: SdModel = None
    c: object = None                 # cond:  tensor [B,T,C] or {"crossattn","vector"} (per image)
    uc: object = None                # uncond, same form
    seeds: List[int] = field(default_factory=lambda: [1000])
    sampler_name: str = "Euler a"
    scheduler: str = "Automatic"
    steps: int = 20
    cfg_scale: float = 7.0
    width: int = 512
    height: int = 512
    eta: Optional[float] = None
    s_churn: float = 0.0
    s_tmin: float = 0.0
    s_tmax: float = float("inf")
    s_noise: float = 1.0
    hr_scheduler: Optional[str] = None
    s_min_uncond: float = 0.0
    randn_source: str = "GPU"
    subseeds: Optional[List[int]] = None     # modules/processing.py:949 — variation seeds, slerp-ed in at subseed_strength
    subseed_strength: float = 0.0
    seed_resize_from_h: int = 0
    seed_resize_from_w: int = 0
    eta_noise_seed_delta: int = 0            # opts.eta_noise_seed_delta (modules/rng.py:148-150)
    enable_hr: bool = False
    hr_scale: float = 2.0
    hr_second_pass_steps: int = 0
    denoising_strength: float = 0.75
    do_not_decode: bool = False
    check_for_nans: bool = True      # the reference checks unless --disable-nan-check (modules/devices.py:229-231)
    batch_size: int = 0
    rng: ImageRNG = None
    sampler: S.KDiffusionSampler = None
    is_hr_pass: bool = False
    # prompt-driven conditioning (modules/processing.py:460-506): one prompt per image; None -> c / uc are given
    prompts: Optional[List[str]] = None
    negative_prompts: Optional[List[str]] = None
    hr_prompts: Optional[List[str]] = None            # default: the first-pass prompts
    hr_negative_prompts: Optional[List[str]] = None
    use_old_scheduling: bool = False                  # opts.use_old_scheduling
    hr_c: object = None
    hr_uc: object = None
    step_multiplier: int = 1
    firstpass_steps: int = 0
    # Hypertile settings of the job (extensions-builtin/hypertile); None: off, no draws
    hypertile: Optional[HT.HypertileOptions] = None
    # class-level in the reference (shared between jobs so that an unchanged prompt is not re-encoded): [params, result]
    cached_uc = [None, None]
    cached_c = [None, None]
    cached_hr_uc = [None, None]
    cached_hr_c = [None, None]

    def __post_init__(self):
        self.batch_size = len(self.seeds)

    # ---- prompts -> conditioning ------------------------------------------------------------------------------------
    def cached_params(self, required_prompts, steps, hires_steps, use_old_scheduling):
        """modules/processing.py:436-458 (the options that change what the conditioner returns)."""
        m = self.sd_model
        return (tuple(required_prompts), steps, hires_steps, use_old_scheduling, id(m), id(m.cond_stage_model) if m is not None else None,
                getattr(required_prompts, "width", None), getattr(required_prompts, "height", None),
                getattr(required_prompts, "is_negative_prompt", False), getattr(m, "sdxl_crop_top", 0), getattr(m, "sdxl_crop_left", 0))

    def get_conds_with_caching(self, function, required_prompts, steps, caches, hires_steps=None):
        """:460-491 — `caches` are [params, result] pairs; a hit in any of them is returned, a miss fills the first."""
        params = self.cached_params(required_prompts, steps, hires_steps, self.use_old_scheduling)
        for cache in caches:
            if cache[0] is not None and params == cache[0]:
                return cache[1]
        cache = caches[0]
        cache[1] = function(self.sd_model, required_prompts, steps, hires_steps, self.use_old_scheduling)
        cache[0] = params
        return cache[1]

    def _total_steps(self, sampler_name, steps):
        config = S.find_sampler_config(sampler_name)   # second-order samplers call the denoiser twice per step (:497-498)
        return steps * 2 if config is not None and config[2].get("second_order", False) else steps

    def setup_conds(self):
        """:493-503 and :1513-1527."""
        if self.prompts is None:
            return
        if self.is_hr_pass:
            self.hr_c = None
            self.calculate_hr_conds()
            return
        negatives = self.negative_prompts if self.negative_prompts is not None else [""] * len(self.prompts)
        prompts = prompt_parser.SdConditioning(self.prompts, width=self.width, height=self.height)
        negative_prompts = prompt_parser.SdConditioning(negatives, width=self.width, height=self.height, is_negative_prompt=True)
        total_steps = self._total_steps(self.sampler_name, self.steps)
        self.step_multiplier = total_steps // self.steps
        self.firstpass_steps = total_steps
        cls = type(self)
        self.uc = self.get_conds_with_caching(prompt_parser.get_learned_conditioning, negative_prompts, total_steps, [cls.cached_uc])
        self.c = self.get_conds_with_caching(prompt_parser.get_multicond_learned_conditioning, prompts, total_steps, [cls.cached_c])
        self.hr_uc = None
        self.hr_c = None

    def calculate_hr_conds(self):
        """:1498-1511 — the second pass counts whole-number `when` on from the first pass's steps and fractions from 1.0."""
        if self.hr_c is not None or self.prompts is None:
            return
        tw, th = int(self.width * self.hr_scale), int(self.height * self.hr_scale)
        hr_p = self.hr_prompts if self.hr_prompts is not None else self.prompts
        hr_n = self.hr_negative_prompts if self.hr_negative_prompts is not None else (self.negative_prompts if self.negative_prompts is not None else [""] * len(hr_p))
        hr_prompts = prompt_parser.SdConditioning(hr_p, width=tw, height=th)
        hr_negative_prompts = prompt_parser.SdConditioning(hr_n, width=tw, height=th, is_negative_prompt=True)
        total_steps = self._total_steps(self.sampler_name, self.hr_second_pass_steps or self.steps)
        cls = type(self)
        self.hr_uc = self.get_conds_with_caching(prompt_parser.get_learned_conditioning, hr_negative_prompts, self.firstpass_steps,
                                                 [cls.cached_hr_uc, cls.cached_uc], total_steps)
        self.hr_c = self.get_conds_with_caching(prompt_parser.get_multicond_learned_conditioning, hr_prompts, self.firstpass_steps,
                                                [cls.cached_hr_c, cls.cached_c], total_steps)

    def get_conds(self):
        """:505-506, :1538-1542."""
        if self.is_hr_pass and self.hr_c is not None:
            return self.hr_c, self.hr_uc
        return self.c, self.uc

    def make_rng(self, shape, seeds) -> ImageRNG:
        return ImageRNG(shape, seeds, subseeds=self.subseeds, subseed_strength=self.subseed_strength,
                        seed_resize_from_h=self.seed_resize_from_h, seed_resize_from_w=self.seed_resize_from_w,
                        source=self.randn_source, device=self.sd_model.device, eta_noise_seed_delta=self.eta_noise_seed_delta)

    # modules/processing.py:1307-1362
    def sample(self, conditioning, unconditional_conditioning, seeds):
        self.sampler = S.create_sampler(self.sampler_name, self.sd_model)
        x = self.rng.next()
        samples = self.sampler.sample(self, x, conditioning, unconditional_conditioning)
        if not self.enable_hr:
            return samples
        return self.sample_hr_pass(samples, seeds)

    # modules/processing.py:1364-1463, latent upscale mode "Latent" (bilinear, antialias False: shared.py:54-56)
    def sample_hr_pass(self, samples, seeds):
        self.is_hr_pass = True
        tw, th = int(self.width * self.hr_scale), int(self.height * self.hr_scale)
        samples = torch.nn.functional.interpolate(samples, size=(th // opt_f, tw // opt_f), mode="bilinear", antialias=False)
        shape = (opt_C, th // opt_f, tw // opt_f)
        self.rng = self.make_rng(shape, seeds)                                     # processing.py:1429
        noise = self.rng.next()
        self.sampler = S.create_sampler(self.sampler_name, self.sd_model)
        self.calculate_hr_conds()                                                  # processing.py:1447 (no-op without prompts)
        if self.hypertile is not None:                                             # scripts' before_hr (processing.py:1389)
            self.sd_model.unet.hypertile = HT.begin_hr_pass(self, tw, th)
        c, uc = self.get_conds()
        return self.sampler.sample_img2img(self, samples, noise, c, uc, steps=self.hr_second_pass_steps or self.steps)


@dataclass
class StableDiffusionProcessingImg2Img(StableDiffusionProcessingTxt2Img):
    """modules/processing.py:1527-1790 restricted to the latent path: init image -> VAE encode -> noise at
    denoising_strength -> sampler.sample_img2img -> (optional latent mask blend). Resize modes, PIL mask
    pre-processing, inpainting-model conditioning and colour correction stay upstream of the path."""
    init_images: torch.Tensor = None     # [B,3,H,W] float in [0,1]
    latent_mask: torch.Tensor = None     # [B or 1, 1 or 4, H/8, W/8] float, 1 = repaint (the reference's `nmask`)
    mask_round: bool = True
    inpainting_fill: int = 1             # 1 original (0 "fill" needs the pixel-space blur), 2 latent noise, 3 latent nothing
    encode_noise: torch.Tensor = None    # pins the VAE posterior sample (None: torch.randn, as the reference)
    init_latent: torch.Tensor = None
    mask: torch.Tensor = None
    nmask: torch.Tensor = None

    def init(self, seeds):
        if self.init_images is None:
            raise L.SdxeError("img2img without init_images")
        img = self.init_images
        if img.shape[-2] != self.height or img.shape[-1] != self.width:
            raise L.SdxeError("init_images must already have the target height x width (resize modes are upstream)")
        if img.shape[0] == 1 and self.batch_size > 1:
            img = img.expand(self.batch_size, -1, -1, -1)
        self.init_latent = images_tensor_to_samples(img, self.sd_model, self.encode_noise)
        if self.latent_mask is not None:
            lat = self.latent_mask.to(self.init_latent.device, torch.float32)
            if self.mask_round:
                lat = torch.round(lat)
            lat = lat.expand(self.init_latent.shape)
            self.mask, self.nmask = 1.0 - lat, lat                                  # processing.py:1742-1743
            if self.inpainting_fill == 2:                                           # :1746-1748
                rnd = ImageRNG(tuple(self.init_latent.shape[1:]), seeds, source=self.randn_source, device=self.sd_model.device).next()
                self.init_latent = self.init_latent * self.mask + rnd * self.nmask
            elif self.inpainting_fill == 3:                                         # :1750-1752
                self.init_latent = self.init_latent * self.mask

    # modules/processing.py:1759-1779
    def sample(self, conditioning, unconditional_conditioning, seeds):
        self.init(seeds)
        x = self.rng.next()
        self.sampler = S.create_sampler(self.sampler_name, self.sd_model)
        samples = self.sampler.sample_img2img(self, self.init_latent, x, conditioning, unconditional_conditioning)
        if self.mask is not None:
            samples = samples * self.nmask + self.init_latent * self.mask
        return samples


@dataclass
class Processed:
    images: torch.Tensor = None      # uint8 [B, H, W, 3] on the host (what becomes PIL images in the reference)
    latents: torch.Tensor = None     # final latents fp32 [B,4,h,w] (device)
    seeds: List[int] = None


class NansException(Exception):
    """modules/devices.py:237-238."""


def test_for_nans(x: torch.Tensor, where: str):
    """modules/devices.py:241-265: the probe reads ONE element, `x[(0,) * x.ndim]` (a NaN anywhere in a UNet / VAE
    output spreads to the whole tensor through the next norm or attention), and raises NansException."""
    probe = x[(0,) * x.ndim] if x.ndim else x
    if not bool(torch.isnan(probe)):
        return
    if where == "unet":
        msg = "A tensor with NaNs was produced in Unet."
    elif where == "vae":
        msg = "A tensor with NaNs was produced in VAE."
    else:
        msg = "A tensor with NaNs was produced."
    raise NansException(msg + " Use --disable-nan-check commandline argument to disable this check.")


def decode_latent_batch(model: SdModel, batch: torch.Tensor, target_device=None, check_for_nans=False, batched=True):
    """modules/processing.py:625-672. The reference decodes one image at a time and probes each decoded image
    (:637-641); the engine takes the whole batch in one call (`batched=True`; per-sample GroupNorm / attention make the
    results identical either way) and probes the first element of every image with one host read. The reference's
    NaN -> fp32-VAE retry (:643-665, opt-in via auto_vae_precision) stays upstream of the engine."""
    if batched:
        out = model.decode_first_stage(batch)
    else:
        out = torch.cat([model.decode_first_stage(batch[i:i + 1]) for i in range(batch.shape[0])])
    if check_for_nans and bool(torch.isnan(out[:, 0, 0, 0]).any()):
        test_for_nans(out[int(torch.isnan(out[:, 0, 0, 0]).nonzero()[0])], "vae")
    return out if target_device is None else out.to(target_device)


@torch.no_grad()
def process_images(p: StableDiffusionProcessingTxt2Img, to_host: bool = True) -> Processed:
    """process_images_inner (modules/processing.py:863-1091) for one batch (`n_iter` == 1)."""
    S.state.interrupted = False
    S.state.skipped = False
    dev = p.sd_model.device
    unet = p.sd_model.unet
    with torch.cuda.device(dev):
        p.is_hr_pass = False
        p.setup_conds()                                                                       # processing.py:966 (no-op without prompts)
        p.rng = p.make_rng((opt_C, p.height // opt_f, p.width // opt_f), p.seeds)           # processing.py:949
        if p.hypertile is not None:                                                           # scripts' process() (:939)
            unet.hypertile = HT.begin_job(p)
        try:
            samples = p.sample(p.c, p.uc, p.seeds)
        finally:
            if p.hypertile is not None:
                unet.hypertile = None
        if p.do_not_decode:
            return Processed(None, samples, list(p.seeds))
        if p.check_for_nans:  # devices.test_for_nans(samples_ddim, "unet"), processing.py:998 (on unless --disable-nan-check)
            test_for_nans(samples, "unet")
        x = decode_latent_batch(p.sd_model, samples, check_for_nans=p.check_for_nans)      # :1002
        x = torch.clamp((x.float() + 1.0) / 2.0, min=0.0, max=1.0)                         # :1004-1005
        # :1034-1035 `x_sample = 255. * ...; x_sample.astype(np.uint8)` — numpy's float -> uint8 cast TRUNCATES
        img = (x.permute(0, 2, 3, 1) * 255.0).to(torch.uint8)
        if not to_host:
            return Processed(img, samples, list(p.seeds))
        host = torch.empty(img.shape, dtype=torch.uint8, pin_memory=True)
        host.copy_(img, non_blocking=False)
    return Processed(host, samples, list(p.seeds))
