"""Host-side mirror of the reference's sampler stack for the accelerated path, with the same names, argument meaning
and error behaviour, so parity tests read like the reference's own:

  KDiffusionSampler            modules/sd_samplers_kdiffusion.py:68-234  (get_sigmas / sample / sample_img2img)
  CFGDenoiser.forward          modules/sd_samplers_cfg_denoiser.py:156-311 — signature kept:
                               forward(x, sigma, uncond, cond, cond_scale, s_min_uncond, image_cond)
  CompVisDenoiser              k_diffusion/external.py (un-vendored; constructed at sd_samplers_kdiffusion.py:61-62)
  sample_euler_ancestral,
  sample_dpmpp_2m              k_diffusion/sampling.py (un-vendored; selected at sd_samplers_kdiffusion.py:11-27)
  setup_img2img_steps          modules/sd_samplers_common.py:22-31
  InterruptedException         modules/sd_samplers_common.py (raised when state.interrupted, cfg_denoiser.py:157-158)
  Sampler                      modules/sd_samplers_common.py:229-332 (initialize / launch_sampling / callback_state)
  create_sampler,
  find_sampler_config          modules/sd_samplers.py:11-33 — one table of the k-diffusion samplers below, the timestep
                               samplers (sd_samplers_timesteps.py: DDIM, DDIM CFG++, PLMS, UniPC) and LCM (sd_samplers_lcm.py)

What is new: the UNet behind `inner_model` is the sdxe engine, and the per-step latent-space elementwise work
(2B batch build + c_in, x + eps*c_out + CFG combine, sampler update) runs as three fused CUDA kernels from
libsdxe.so instead of ~15 small PyTorch launches (SURVEY K9). The sigma schedule stays on the host
(modules/sd_samplers_kdiffusion.py:127,132). CFGDenoiser keeps the three denoiser-specific steps in overridable methods
(model_inputs: c_in and the UNet timestep; combine; last_latent) so that the timestep and LCM denoisers add only their
differences; their combine is sdxe_cfg_combine_affine.
"""
from __future__ import annotations

import math
from typing import Callable, Optional

import numpy as np
import torch

from . import lib as L


class InterruptedException(BaseException):
    pass


class SamplerState:
    """The two cooperative-cancel flags the reference polls each denoiser call (modules/shared_state.py:79)."""

    interrupted = False
    skipped = False
    sampling_step = 0
    sampling_steps = 0


state = SamplerState()


# ------------------------------------------------------------------------------------------------------------------
# k-diffusion schedule / denoiser wrapper
# ------------------------------------------------------------------------------------------------------------------
def make_alphas_cumprod(linear_start=0.00085, linear_end=0.012, timesteps=1000) -> torch.Tensor:
    """ldm 'linear' (scaled-linear) beta schedule; configs/v1-inference.yaml:5-9, ddpm_edit.py:133-141."""
    betas = np.linspace(linear_start ** 0.5, linear_end ** 0.5, timesteps, dtype=np.float64) ** 2
    return torch.tensor(np.cumprod(1.0 - betas, axis=0), dtype=torch.float32)


class DiscreteSchedule:
    def __init__(self, alphas_cumprod: torch.Tensor, device):
        self.sigmas = (((1 - alphas_cumprod) / alphas_cumprod) ** 0.5).to(device)
        self.log_sigmas = self.sigmas.log()

    def get_sigmas(self, n: int) -> torch.Tensor:
        t_max = len(self.sigmas) - 1
        t = torch.linspace(t_max, 0, n, device=self.sigmas.device)
        return torch.cat([self.t_to_sigma(t), t.new_zeros([1])])

    def sigma_to_t(self, sigma: torch.Tensor) -> torch.Tensor:
        log_sigma = sigma.log()
        dists = log_sigma - self.log_sigmas[:, None]
        low_idx = dists.ge(0).cumsum(dim=0).argmax(dim=0).clamp(max=self.log_sigmas.shape[0] - 2)
        high_idx = low_idx + 1
        low, high = self.log_sigmas[low_idx], self.log_sigmas[high_idx]
        w = ((low - log_sigma) / (low - high)).clamp(0, 1)
        t = (1 - w) * low_idx + w * high_idx
        return t.view(sigma.shape)

    def t_to_sigma(self, t: torch.Tensor) -> torch.Tensor:
        t = t.float()
        low_idx, high_idx, w = t.floor().long(), t.ceil().long(), t.frac()
        return ((1 - w) * self.log_sigmas[low_idx] + w * self.log_sigmas[high_idx]).exp()


class CompVisDenoiser(DiscreteSchedule):
    """eps-prediction wrapper: D(x, sigma) = x + eps(x * c_in, t(sigma)) * c_out."""

    sigma_data = 1.0

    def __init__(self, sd_model, quantize: bool = False):
        super().__init__(sd_model.alphas_cumprod, sd_model.device)
        self.inner_model = sd_model
        if quantize:
            raise NotImplementedError("enable_quantization is off by default (shared_options.py:176) and not mirrored")

    def get_scalings(self, sigma):
        return -sigma, 1 / (sigma ** 2 + self.sigma_data ** 2) ** 0.5

    def forward(self, x, sigma, **kwargs):
        c_out, c_in = [s.view(-1, 1, 1, 1) for s in self.get_scalings(sigma)]
        eps = self.inner_model.apply_model(x * c_in, self.sigma_to_t(sigma), **kwargs)
        return x + eps * c_out

    __call__ = forward


def get_sigmas_karras(n, sigma_min, sigma_max, rho=7.0, device="cpu"):
    ramp = torch.linspace(0, 1, n, device=device)
    min_inv_rho, max_inv_rho = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
    sigmas = (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** rho
    return torch.cat([sigmas, sigmas.new_zeros([1])])


def setup_img2img_steps(p, steps=None):
    """modules/sd_samplers_common.py:22-31 (img2img_fix_steps is off by default)."""
    if steps is not None:
        requested = steps or p.steps
        steps = int(requested / min(p.denoising_strength, 0.999)) if p.denoising_strength > 0 else 0
        t_enc = requested - 1
    else:
        steps = p.steps
        t_enc = int(min(p.denoising_strength, 0.999) * steps)
    return steps, t_enc


# ------------------------------------------------------------------------------------------------------------------
# CFG denoiser
# ------------------------------------------------------------------------------------------------------------------
def _cond_tensor(c):
    return c["crossattn"] if isinstance(c, dict) else c


def catenate_conds(conds):
    """sd_samplers_cfg_denoiser.py:11-15."""
    if not isinstance(conds[0], dict):
        return torch.cat(conds)
    return {key: torch.cat([x[key] for x in conds]) for key in conds[0].keys()}


def subscript_cond(cond, a, b):
    """sd_samplers_cfg_denoiser.py:18-22."""
    if not isinstance(cond, dict):
        return cond[a:b]
    return {key: vec[a:b] for key, vec in cond.items()}


def pad_cond(tensor, repeats, empty):
    """sd_samplers_cfg_denoiser.py:25-30: append `repeats` copies of the empty-prompt embedding along the token axis."""
    if not isinstance(tensor, dict):
        return torch.cat([tensor, empty.repeat((tensor.shape[0], repeats, 1))], axis=1)
    tensor["crossattn"] = pad_cond(tensor["crossattn"], repeats, empty)
    return tensor


class CFGDenoiserOptions:
    """The `shared.opts` fields CFGDenoiser.forward reads (defaults: modules/shared_options.py)."""

    batch_cond_uncond = True
    pad_cond_uncond = False
    pad_cond_uncond_v0 = False
    s_min_uncond_all = False
    skip_early_cond = 0.0


class CFGDenoiser:
    """Classifier-free-guidance denoiser with the reference's call signature and batching rules
    (modules/sd_samplers_cfg_denoiser.py:156-311).

    `cond`: a `prompt_parser.MulticondLearnedConditioning` (AND-composed, weighted, step-scheduled prompts — what
    `p.setup_conds()` leaves in `p.c`) or, already reconstructed, one cond per image as a tensor [B,T,C] / SDXL dict
    {"crossattn": [B,T,C], "vector": [B,2816]}. `uncond`: list of prompt schedules or a tensor / dict likewise.
    InstructPix2Pix ("edit") checkpoints and inpainting `image_cond` are outside the accelerated path."""

    _key_counter = 0  # context keys handed to the engine's cross-attention k|v cache (unique per process)

    def __init__(self, sampler):
        self.sampler = sampler
        self.model_wrap = None
        self.mask = None
        self.nmask = None
        self.init_latent = None
        self.steps = None
        self.total_steps = None
        self.step = 0
        self.image_cfg_scale = None
        self.p = None
        self.mask_before_denoising = False
        self.cond_scale_miltiplier = 1.0
        self.padded_cond_uncond = False
        self.padded_cond_uncond_v0 = False
        self.need_last_noise_uncond = False
        self.last_noise_uncond = None
        self.opts = CFGDenoiserOptions()
        self._dev_cache = {}
        self._ctx_keys = {}
        self._ctx_refs = None
        self.on_cfg_denoiser = []   # callables(x, sigma_in, cond_in) -> None       (script_callbacks.on_cfg_denoiser)
        self.on_cfg_denoised = []   # callables(eps)                                (on_cfg_denoised)
        self.on_cfg_after_cfg = []  # callables(denoised) -> denoised | None        (on_cfg_after_cfg)

    @property
    def inner_model(self):
        if self.model_wrap is None:
            self.model_wrap = CompVisDenoiser(self.sampler.sd_model, quantize=False)
        return self.model_wrap

    def combine_denoised(self, x_out, conds_list, uncond, cond_scale):
        """sd_samplers_cfg_denoiser.py:74-82 (torch form; the hot path runs the same arithmetic in sdxe_cfg_combine*)."""
        denoised_uncond = x_out[-uncond.shape[0]:]
        denoised = torch.clone(denoised_uncond)
        for i, conds in enumerate(conds_list):
            for cond_index, weight in conds:
                denoised[i] += (x_out[cond_index] - denoised_uncond[i]) * (weight * cond_scale)
        return denoised

    def pad_cond_uncond(self, cond, uncond):
        """:100-111 — pad the shorter of cond / uncond with empty-prompt chunks (`sd_model.cond_stage_model_empty_prompt`)."""
        empty = getattr(self.sampler.sd_model, "cond_stage_model_empty_prompt", None)
        if empty is None:
            raise L.SdxeError("pad_cond_uncond needs sd_model.cond_stage_model_empty_prompt (the empty prompt's embedding)")
        num_repeats = (cond.shape[1] - uncond.shape[1]) // empty.shape[1]
        if num_repeats < 0:
            cond = pad_cond(cond, -num_repeats, empty)
            self.padded_cond_uncond = True
        elif num_repeats > 0:
            uncond = pad_cond(uncond, num_repeats, empty)
            self.padded_cond_uncond = True
        return cond, uncond

    def pad_cond_uncond_v0(self, cond, uncond):
        """:113-154 — pre-1.6.0 behaviour: repeat uncond's last token vector / truncate it to cond's token count."""
        is_dict = isinstance(uncond, dict)
        u = uncond["crossattn"] if is_dict else uncond
        if u.shape[1] < cond.shape[1]:
            u = torch.hstack([u, u[:, -1:].repeat([1, cond.shape[1] - u.shape[1], 1])])
            self.padded_cond_uncond_v0 = True
        elif u.shape[1] > cond.shape[1]:
            u = u[:, :cond.shape[1]]
            self.padded_cond_uncond_v0 = True
        if is_dict:
            uncond["crossattn"] = u
        else:
            uncond = u
        return cond, uncond

    def _apply_blend(self, latent):
        return latent * self.nmask + self.init_latent * self.mask

    def _dev(self, key, build):
        t = self._dev_cache.get(key)
        if t is None:
            if len(self._dev_cache) > 64:
                self._dev_cache.clear()
            t = self._dev_cache[key] = build()
        return t

    def _run_unet(self, x_in, t, cond_in, key=0):
        sd = self.sampler.sd_model
        ctx = _cond_tensor(cond_in)
        vec = cond_in.get("vector") if isinstance(cond_in, dict) else None
        return sd.apply_model_scaled(x_in, t, ctx, vec, context_key=key)  # engine UNet through the SdUnet seam

    def _context_key(self, cond, uncond, tag):
        """A key that identifies the CONTENTS of the conditioning sent to the UNet this step: the cond / uncond objects of the
        job (kept alive by sampler_extra_args), which scheduled prompts are active at this step, and which rows are sent."""
        from . import prompt_parser

        def active(c):
            if isinstance(c, prompt_parser.MulticondLearnedConditioning):
                return tuple(prompt_parser._active(cp.schedules, self.step) for prompts in c.batch for cp in prompts)
            if isinstance(c, (list, tuple)):
                return tuple(prompt_parser._active(sched, self.step) for sched in c)
            return ()

        ident = (id(cond), id(uncond), active(cond), active(uncond), tag)
        key = self._ctx_keys.get(ident)
        if key is None:
            CFGDenoiser._key_counter += 1
            key = self._ctx_keys[ident] = CFGDenoiser._key_counter
            self._ctx_refs = (cond, uncond)  # the ids stay unique while the denoiser holds the objects
        return key

    def model_inputs(self, sigma_in):
        """Per UNet row: the input scaling c_in and the timestep the UNet sees (CompVisDenoiser.forward)."""
        _, c_in = self.inner_model.get_scalings(sigma_in)
        return c_in, self.inner_model.sigma_to_t(sigma_in)

    def _csr(self, x, conds_list, skip_uncond, scale):
        """Device tables of the general combine: row_ptr [B+1], cond_rows, cond_w (weight * scale), uncond_rows [B]."""
        repeats = [len(c) for c in conds_list]
        n_cond, batch_size = sum(repeats), len(conds_list)
        wkey = ("csr", tuple(repeats), skip_uncond, tuple(w for c in conds_list for _, w in c), scale)

        def build():
            ptr, k = [0], 0
            for n in repeats:
                k += n
                ptr.append(k)
            # skipped uncond: the reference puts each image's FIRST cond result where the uncond result would be
            urows = [c[0][0] for c in conds_list] if skip_uncond else [n_cond + i for i in range(batch_size)]
            return (torch.tensor(ptr, device=x.device, dtype=torch.int32),
                    torch.tensor([j for c in conds_list for j, _ in c], device=x.device, dtype=torch.int32),
                    torch.tensor([w * scale for c in conds_list for _, w in c], device=x.device, dtype=torch.float32),
                    torch.tensor(urows, device=x.device, dtype=torch.int32))

        return self._dev(wkey, build)

    def combine(self, x, eps, sigma, sigma_in, conds_list, skip_uncond, scale):
        """x_out = x_in + eps * c_out and the CFG combine, fused (:272-289). `scale`: cond_scale * cond_scale_miltiplier."""
        lib = L.load()
        stream = L.current_stream()
        batch_size, elems = len(conds_list), x[0].numel()
        n_cond = sum(len(c) for c in conds_list)
        if self.need_last_noise_uncond and not skip_uncond:
            c_out, _ = self.inner_model.get_scalings(sigma_in)
            self.last_noise_uncond = x + eps[n_cond:].float() * c_out[n_cond:].view(-1, 1, 1, 1)
        if skip_uncond:
            scale = 1.0
        denoised = torch.empty_like(x)
        if n_cond == batch_size and not skip_uncond and all(c[0][1] == 1.0 for c in conds_list):
            L.check(lib.sdxe_cfg_combine(L.ptr(x), L.ptr(eps), L.ptr(sigma), scale, L.ptr(denoised), batch_size, elems,
                                         L.torch_dtype_code(eps.dtype), stream), "sdxe_cfg_combine")
        else:
            row_ptr, cond_rows, cond_w, uncond_rows = self._csr(x, conds_list, skip_uncond, scale)
            L.check(lib.sdxe_cfg_combine_multi(L.ptr(x), L.ptr(eps), L.ptr(sigma), L.ptr(row_ptr), L.ptr(cond_rows), L.ptr(cond_w),
                                               L.ptr(uncond_rows), L.ptr(denoised), batch_size, elems,
                                               L.torch_dtype_code(eps.dtype), stream), "sdxe_cfg_combine_multi")
        return denoised

    def combine_affine(self, x, eps, conds_list, skip_uncond, scale, cx, ce, x0_coef=None, want_uncond=False):
        """The CFG combine of a denoiser whose output per row is cx[b] * x[b] + ce[b] * eps[r] (sdxe_cfg_combine_affine).
        Returns (out, pred_x0 of each image's first cond or None, uncond eps as fp32 or None)."""
        row_ptr, cond_rows, cond_w, uncond_rows = self._csr(x, conds_list, skip_uncond, 1.0 if skip_uncond else scale)
        out = torch.empty_like(x)
        x0 = torch.empty_like(x) if x0_coef is not None else None
        unc = torch.empty_like(x) if want_uncond else None
        L.check(L.load().sdxe_cfg_combine_affine(L.ptr(x), L.ptr(eps), L.ptr(row_ptr), L.ptr(cond_rows), L.ptr(cond_w), L.ptr(uncond_rows),
                                                 L.ptr(cx), L.ptr(ce), L.ptr(out), L.ptr(x0_coef), L.ptr(x0), L.ptr(unc), len(conds_list),
                                                 x[0].numel(), L.torch_dtype_code(eps.dtype), L.current_stream()), "sdxe_cfg_combine_affine")
        return out, x0, unc

    def last_latent(self, denoised):
        """What an interrupted job returns (the sampler's last_latent)."""
        return denoised

    def forward(self, x, sigma, uncond, cond, cond_scale, s_min_uncond, image_cond):
        if state.interrupted or state.skipped:
            raise InterruptedException
        from . import prompt_parser

        sd = self.sampler.sd_model
        lib = L.load()
        opts = self.opts
        cond_obj, uncond_obj = cond, uncond
        # ---- per-step conditioning (:168-169)
        if isinstance(cond, prompt_parser.MulticondLearnedConditioning):
            conds_list, tensor = prompt_parser.reconstruct_multicond_batch(cond, self.step)
        else:
            tensor = cond
            conds_list = [[(i, 1.0)] for i in range(_cond_tensor(cond).shape[0])]
        if isinstance(uncond, (list, tuple)):
            uncond = prompt_parser.reconstruct_cond_batch(uncond, self.step)
        if self.mask_before_denoising and self.mask is not None:
            x = self._apply_blend(x)
        batch_size = len(conds_list)
        if x.shape[0] != batch_size or _cond_tensor(uncond).shape[0] != batch_size:
            raise L.SdxeError(f"CFGDenoiser: {x.shape[0]} latents, {batch_size} conds, {_cond_tensor(uncond).shape[0]} unconds")
        repeats = [len(c) for c in conds_list]
        n_cond = sum(repeats)
        x = x.float().contiguous()
        sigma = sigma.float().contiguous()
        # ---- uncond skipping (:213-227)
        skip_uncond = False
        if opts.skip_early_cond != 0.0 and self.step / max(1, self.total_steps or 1) <= opts.skip_early_cond:
            skip_uncond = True
        elif (self.step % 2 or opts.s_min_uncond_all) and s_min_uncond > 0 and float(sigma[0]) < s_min_uncond:
            skip_uncond = True
        rows = n_cond if skip_uncond else n_cond + batch_size
        key = (tuple(repeats), skip_uncond)
        src = self._dev(("src",) + key, lambda: torch.tensor(
            [i for i, n in enumerate(repeats) for _ in range(n)] + ([] if skip_uncond else list(range(batch_size))),
            device=x.device, dtype=torch.int32))
        plain = n_cond == batch_size  # one cond per image: rows [0,B) cond, [B,2B) uncond
        sigma_in = (sigma if skip_uncond else torch.cat([sigma, sigma])) if plain else sigma[src.long()]
        for cb in self.on_cfg_denoiser:
            cb(x, sigma_in, tensor)
        # ---- token-count reconciliation (:229-234)
        self.padded_cond_uncond = False
        self.padded_cond_uncond_v0 = False
        if opts.pad_cond_uncond_v0 and tensor.shape[1] != uncond.shape[1]:
            tensor, uncond = self.pad_cond_uncond_v0(tensor, uncond)
        elif opts.pad_cond_uncond and tensor.shape[1] != uncond.shape[1]:
            tensor, uncond = self.pad_cond_uncond(tensor, uncond)
        # ---- fused: x_in[r] = x[src[r]] * c_in[r] in the UNet's dtype (:203 + CompVisDenoiser c_in + the dtype cast of
        #      sd_hijack_unet.py:43-50)
        c_in, t = self.model_inputs(sigma_in)
        elems = x[0].numel()
        x_in = torch.empty((rows,) + tuple(x.shape[1:]), dtype=sd.dtype_unet, device=x.device)
        stream = L.current_stream()
        L.check(lib.sdxe_denoiser_in(L.ptr(x), L.ptr(src), L.ptr(c_in), L.ptr(x_in), rows, elems,
                                     L.torch_dtype_code(sd.dtype_unet), stream), "sdxe_denoiser_in")
        # ---- UNet call(s) (:236-267)
        if _cond_tensor(tensor).shape[1] == _cond_tensor(uncond).shape[1] or skip_uncond:
            cond_in = tensor if skip_uncond else catenate_conds([tensor, uncond])
            cacheable = not self.on_cfg_denoiser and not self.padded_cond_uncond and not self.padded_cond_uncond_v0
            if opts.batch_cond_uncond:
                eps = self._run_unet(x_in, t, cond_in, self._context_key(cond_obj, uncond_obj, ("all", skip_uncond)) if cacheable else 0)
            else:
                eps = torch.empty_like(x_in)
                for a in range(0, rows, batch_size):
                    b = min(a + batch_size, rows)
                    eps[a:b] = self._run_unet(x_in[a:b], t[a:b], subscript_cond(cond_in, a, b))
        else:  # cond / uncond token counts differ: they cannot share a batch
            eps = torch.empty_like(x_in)
            sub = batch_size * 2 if opts.batch_cond_uncond else batch_size
            for a in range(0, n_cond, sub):
                b = min(a + sub, n_cond)
                eps[a:b] = self._run_unet(x_in[a:b], t[a:b], subscript_cond(tensor, a, b))
            eps[n_cond:] = self._run_unet(x_in[n_cond:], t[n_cond:], uncond)
        for cb in self.on_cfg_denoised:
            cb(eps)
        denoised = self.combine(x, eps, sigma, sigma_in, conds_list, skip_uncond, float(cond_scale) * self.cond_scale_miltiplier)
        if not self.mask_before_denoising and self.mask is not None:
            denoised = self._apply_blend(denoised)
        self.sampler.last_latent = self.last_latent(denoised)
        for cb in self.on_cfg_after_cfg:
            r = cb(denoised)
            if r is not None:
                denoised = r
        self.step += 1
        return denoised

    __call__ = forward


# ------------------------------------------------------------------------------------------------------------------
# sampler loops (k_diffusion.sampling restated; the update itself is one fused kernel per step)
# ------------------------------------------------------------------------------------------------------------------
def get_ancestral_step(sigma_from: float, sigma_to: float, eta: float = 1.0):
    if not eta:
        return sigma_to, 0.0
    sigma_up = min(sigma_to, eta * (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5)
    sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
    return sigma_down, sigma_up


@torch.no_grad()
def sample_euler_ancestral(model, x, sigmas, extra_args=None, callback=None, disable=None, eta=1.0, s_noise=1.0,
                           noise_sampler: Optional[Callable] = None):
    """noise_sampler(sigma, sigma_next) -> noise like x; the webui routes it to p.rng.next() (sd_samplers_common.py:225)."""
    extra_args = {} if extra_args is None else extra_args
    lib = L.load()
    x = x.float().contiguous().clone()
    s_in = x.new_ones([x.shape[0]])
    sig = [float(s) for s in sigmas]  # host schedule
    for i in range(len(sig) - 1):
        denoised = model(x, s_in * sig[i], **extra_args)
        sigma_down, sigma_up = get_ancestral_step(sig[i], sig[i + 1], eta=eta)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": denoised})
        noise = None
        if sig[i + 1] > 0:
            noise = noise_sampler(sigmas[i], sigmas[i + 1]).float().contiguous()
        L.check(lib.sdxe_euler_ancestral_step(L.ptr(x), L.ptr(denoised.contiguous()), L.ptr(noise), sig[i], sigma_down,
                                              sigma_up * s_noise if sig[i + 1] > 0 else 0.0, x.numel(),
                                              L.current_stream()), "sdxe_euler_ancestral_step")
    return x


@torch.no_grad()
def sample_dpmpp_2m(model, x, sigmas, extra_args=None, callback=None, disable=None):
    extra_args = {} if extra_args is None else extra_args
    lib = L.load()
    x = x.float().contiguous().clone()
    s_in = x.new_ones([x.shape[0]])
    sig = [float(s) for s in sigmas]

    def t_fn(s):
        return -math.log(s) if s > 0 else math.inf

    old_denoised = None
    for i in range(len(sig) - 1):
        denoised = model(x, s_in * sig[i], **extra_args).contiguous()
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": denoised})
        t, t_next = t_fn(sig[i]), t_fn(sig[i + 1])
        h = t_next - t
        ratio = sig[i + 1] / sig[i]
        neg_expm1 = -math.expm1(-h) if math.isfinite(h) else 1.0
        if old_denoised is None or sig[i + 1] == 0:
            c0, c1 = 1.0, 0.0
        else:
            h_last = t - t_fn(sig[i - 1])
            r = h_last / h
            c0, c1 = 1 + 1 / (2 * r), -1 / (2 * r)
        L.check(lib.sdxe_dpmpp_2m_step(L.ptr(x), L.ptr(denoised), L.ptr(old_denoised), ratio, neg_expm1, c0, c1, x.numel(),
                                       L.current_stream()), "sdxe_dpmpp_2m_step")
        old_denoised = denoised
    return x


def _lincomb(lib, out, terms, n):
    """out = sum(c * p) over up to four (tensor, coefficient) terms — one fused launch (sdxe_lincomb)."""
    terms = list(terms) + [(None, 0.0)] * (4 - len(terms))
    (p0, c0), (p1, c1), (p2, c2), (p3, c3) = terms
    L.check(lib.sdxe_lincomb(L.ptr(out), L.ptr(p0), float(c0), L.ptr(p1), float(c1), L.ptr(p2), float(c2), L.ptr(p3), float(c3), n,
                             L.current_stream()), "sdxe_lincomb")
    return out


def _churn(sig, i, s_churn, s_tmin, s_tmax):
    gamma = min(s_churn / (len(sig) - 1), 2 ** 0.5 - 1) if s_tmin <= sig[i] <= s_tmax else 0.0
    return gamma, sig[i] * (gamma + 1)


def _prep(x, sigmas, extra_args):
    return ({} if extra_args is None else extra_args), L.load(), x.float().contiguous().clone(), [float(s) for s in sigmas]


@torch.no_grad()
def sample_euler(model, x, sigmas, extra_args=None, callback=None, disable=None, s_churn=0.0, s_tmin=0.0, s_tmax=float("inf"),
                 s_noise=1.0, noise_sampler: Optional[Callable] = None):
    """k-diffusion sample_euler: x += (x - D(x, sigma_hat)) / sigma_hat * (sigma_next - sigma_hat)."""
    extra_args, lib, x, sig = _prep(x, sigmas, extra_args)
    s_in, n = x.new_ones([x.shape[0]]), x.numel()
    for i in range(len(sig) - 1):
        gamma, sigma_hat = _churn(sig, i, s_churn, s_tmin, s_tmax)
        if gamma > 0:
            _lincomb(lib, x, [(x, 1.0), (noise_sampler(sigmas[i], sigmas[i + 1]).float().contiguous(), s_noise * (sigma_hat ** 2 - sig[i] ** 2) ** 0.5)], n)
        denoised = model(x, s_in * sigma_hat, **extra_args).contiguous()
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigma_hat, "denoised": denoised})
        r = sig[i + 1] / sigma_hat
        _lincomb(lib, x, [(x, r), (denoised, 1.0 - r)], n)   # x + (x - den) / s * (s' - s)
    return x


@torch.no_grad()
def sample_heun(model, x, sigmas, extra_args=None, callback=None, disable=None, s_churn=0.0, s_tmin=0.0, s_tmax=float("inf"),
                s_noise=1.0, noise_sampler: Optional[Callable] = None):
    extra_args, lib, x, sig = _prep(x, sigmas, extra_args)
    s_in, n = x.new_ones([x.shape[0]]), x.numel()
    x2 = torch.empty_like(x)
    for i in range(len(sig) - 1):
        gamma, sigma_hat = _churn(sig, i, s_churn, s_tmin, s_tmax)
        if gamma > 0:
            _lincomb(lib, x, [(x, 1.0), (noise_sampler(sigmas[i], sigmas[i + 1]).float().contiguous(), s_noise * (sigma_hat ** 2 - sig[i] ** 2) ** 0.5)], n)
        denoised = model(x, s_in * sigma_hat, **extra_args).contiguous()
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigma_hat, "denoised": denoised})
        dt = sig[i + 1] - sigma_hat
        a = dt / sigma_hat                                     # d * dt = (x - den) * a
        if sig[i + 1] == 0:
            _lincomb(lib, x, [(x, 1.0 + a), (denoised, -a)], n)
        else:
            _lincomb(lib, x2, [(x, 1.0 + a), (denoised, -a)], n)
            denoised_2 = model(x2, s_in * sig[i + 1], **extra_args).contiguous()
            b = dt / sig[i + 1]                                # d_2 * dt = (x_2 - den_2) * b
            # x + (d + d_2) / 2 * dt
            _lincomb(lib, x, [(x, 1.0 + a / 2), (denoised, -a / 2), (x2, b / 2), (denoised_2, -b / 2)], n)
    return x


@torch.no_grad()
def sample_dpm_2(model, x, sigmas, extra_args=None, callback=None, disable=None, s_churn=0.0, s_tmin=0.0, s_tmax=float("inf"),
                 s_noise=1.0, noise_sampler: Optional[Callable] = None):
    extra_args, lib, x, sig = _prep(x, sigmas, extra_args)
    s_in, n = x.new_ones([x.shape[0]]), x.numel()
    x2 = torch.empty_like(x)
    for i in range(len(sig) - 1):
        gamma, sigma_hat = _churn(sig, i, s_churn, s_tmin, s_tmax)
        if gamma > 0:
            _lincomb(lib, x, [(x, 1.0), (noise_sampler(sigmas[i], sigmas[i + 1]).float().contiguous(), s_noise * (sigma_hat ** 2 - sig[i] ** 2) ** 0.5)], n)
        denoised = model(x, s_in * sigma_hat, **extra_args).contiguous()
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigma_hat, "denoised": denoised})
        if sig[i + 1] == 0:
            a = (sig[i + 1] - sigma_hat) / sigma_hat
            _lincomb(lib, x, [(x, 1.0 + a), (denoised, -a)], n)
        else:
            sigma_mid = math.exp(0.5 * (math.log(sigma_hat) + math.log(sig[i + 1])))
            a = (sigma_mid - sigma_hat) / sigma_hat
            _lincomb(lib, x2, [(x, 1.0 + a), (denoised, -a)], n)
            denoised_2 = model(x2, s_in * sigma_mid, **extra_args).contiguous()
            b = (sig[i + 1] - sigma_hat) / sigma_mid           # x + d_2 * dt_2, d_2 = (x_2 - den_2) / sigma_mid
            _lincomb(lib, x, [(x, 1.0), (x2, b), (denoised_2, -b)], n)
    return x


@torch.no_grad()
def sample_dpm_2_ancestral(model, x, sigmas, extra_args=None, callback=None, disable=None, eta=1.0, s_noise=1.0,
                           noise_sampler: Optional[Callable] = None):
    extra_args, lib, x, sig = _prep(x, sigmas, extra_args)
    s_in, n = x.new_ones([x.shape[0]]), x.numel()
    x2 = torch.empty_like(x)
    for i in range(len(sig) - 1):
        denoised = model(x, s_in * sig[i], **extra_args).contiguous()
        sigma_down, sigma_up = get_ancestral_step(sig[i], sig[i + 1], eta=eta)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": denoised})
        if sigma_down == 0:
            a = (sigma_down - sig[i]) / sig[i]
            _lincomb(lib, x, [(x, 1.0 + a), (denoised, -a)], n)
        else:
            sigma_mid = math.exp(0.5 * (math.log(sig[i]) + math.log(sigma_down)))
            a = (sigma_mid - sig[i]) / sig[i]
            _lincomb(lib, x2, [(x, 1.0 + a), (denoised, -a)], n)
            denoised_2 = model(x2, s_in * sigma_mid, **extra_args).contiguous()
            b = (sigma_down - sig[i]) / sigma_mid
            noise = noise_sampler(sigmas[i], sigmas[i + 1]).float().contiguous()
            _lincomb(lib, x, [(x, 1.0), (x2, b), (denoised_2, -b), (noise, s_noise * sigma_up)], n)
    return x


@torch.no_grad()
def sample_dpmpp_2s_ancestral(model, x, sigmas, extra_args=None, callback=None, disable=None, eta=1.0, s_noise=1.0,
                              noise_sampler: Optional[Callable] = None):
    extra_args, lib, x, sig = _prep(x, sigmas, extra_args)
    s_in, n = x.new_ones([x.shape[0]]), x.numel()
    x2 = torch.empty_like(x)
    for i in range(len(sig) - 1):
        denoised = model(x, s_in * sig[i], **extra_args).contiguous()
        sigma_down, sigma_up = get_ancestral_step(sig[i], sig[i + 1], eta=eta)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": denoised})
        noise = noise_sampler(sigmas[i], sigmas[i + 1]).float().contiguous() if sig[i + 1] > 0 else None
        tail = [(noise, s_noise * sigma_up)] if noise is not None else []
        if sigma_down == 0:
            a = (sigma_down - sig[i]) / sig[i]
            _lincomb(lib, x, [(x, 1.0 + a), (denoised, -a)] + tail, n)
        else:
            t, t_next = -math.log(sig[i]), -math.log(sigma_down)
            h = t_next - t
            s_mid = t + 0.5 * h
            _lincomb(lib, x2, [(x, math.exp(-s_mid) / math.exp(-t)), (denoised, -math.expm1(-h * 0.5))], n)
            denoised_2 = model(x2, s_in * math.exp(-s_mid), **extra_args).contiguous()
            _lincomb(lib, x, [(x, math.exp(-t_next) / math.exp(-t)), (denoised_2, -math.expm1(-h))] + tail, n)
    return x


def linear_multistep_coeff(order, t, i, j):
    from scipy import integrate

    if order - 1 > i:
        raise ValueError(f"Order {order} too high for step {i}")

    def fn(tau):
        prod = 1.0
        for k in range(order):
            if j != k:
                prod *= (tau - t[i - k]) / (t[i - j] - t[i - k])
        return prod

    return integrate.quad(fn, t[i], t[i + 1], epsrel=1e-4)[0]


@torch.no_grad()
def sample_lms(model, x, sigmas, extra_args=None, callback=None, disable=None, order=4):
    extra_args, lib, x, sig = _prep(x, sigmas, extra_args)
    s_in, n = x.new_ones([x.shape[0]]), x.numel()
    t_cpu = sigmas.detach().cpu().numpy()
    ds = []
    for i in range(len(sig) - 1):
        denoised = model(x, s_in * sig[i], **extra_args).contiguous()
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": denoised})
        d = torch.empty_like(x)
        _lincomb(lib, d, [(x, 1.0 / sig[i]), (denoised, -1.0 / sig[i])], n)   # to_d
        ds.append(d)
        if len(ds) > order:
            ds.pop(0)
        cur = min(i + 1, order)
        coeffs = [linear_multistep_coeff(cur, t_cpu, i, j) for j in range(cur)]
        hist = list(reversed(ds))[:cur]
        _lincomb(lib, x, [(x, 1.0)] + [(d_j, c_j) for c_j, d_j in zip(coeffs[:3], hist[:3])], n)
        if cur == 4:
            _lincomb(lib, x, [(x, 1.0), (hist[3], coeffs[3])], n)
    return x


@torch.no_grad()
def restart_sampler(model, x, sigmas, extra_args=None, callback=None, disable=None, s_noise=1.0, restart_list=None,
                    noise_sampler: Optional[Callable] = None):
    """modules/sd_samplers_extra.py:7-74 ("Restart Sampling for Improving Generative Processes"): Heun steps over a Karras
    schedule with restart segments that re-noise the sample back up to sigma 2. restart_list: {min_sigma: [steps, times,
    max_sigma]}; None picks it from the step count exactly as the reference does. The re-noising draw is
    `k_diffusion.sampling.torch.randn_like` in the reference, i.e. TorchHijack -> p.rng.next() = noise_sampler here."""
    from . import sd_schedulers

    extra_args = {} if extra_args is None else extra_args
    lib = L.load()
    x = x.float().contiguous().clone()
    s_in, n = x.new_ones([x.shape[0]]), x.numel()
    x2 = torch.empty_like(x)
    step_id = 0

    def heun_step(old_sigma, new_sigma, second_order=True):
        nonlocal step_id
        old, new = float(old_sigma), float(new_sigma)
        denoised = model(x, s_in * old, **extra_args).contiguous()
        if callback is not None:
            callback({"x": x, "i": step_id, "sigma": new_sigma, "sigma_hat": old_sigma, "denoised": denoised})
        dt = new - old
        a = dt / old
        if new == 0 or not second_order:
            _lincomb(lib, x, [(x, 1.0 + a), (denoised, -a)], n)
        else:
            _lincomb(lib, x2, [(x, 1.0 + a), (denoised, -a)], n)
            denoised_2 = model(x2, s_in * new, **extra_args).contiguous()
            b = dt / new
            _lincomb(lib, x, [(x, 1.0 + a / 2), (denoised, -a / 2), (x2, b / 2), (denoised_2, -b / 2)], n)
        step_id += 1

    steps = sigmas.shape[0] - 1
    if restart_list is None:
        if steps >= 20:
            restart_steps, restart_times = 9, 1
            if steps >= 36:
                restart_steps, restart_times = steps // 4, 2
            sigmas = sd_schedulers.get_sigmas_karras(steps - restart_steps * restart_times, sigmas[-2].item(), sigmas[0].item(), device=sigmas.device)
            restart_list = {0.1: [restart_steps + 1, restart_times, 2]}
        else:
            restart_list = {}
    restart_list = {int(torch.argmin(abs(sigmas - key), dim=0)): value for key, value in restart_list.items()}
    step_list = []
    for i in range(len(sigmas) - 1):
        step_list.append((sigmas[i], sigmas[i + 1]))
        if i + 1 in restart_list:
            restart_steps, restart_times, restart_max = restart_list[i + 1]
            min_idx = i + 1
            max_idx = int(torch.argmin(abs(sigmas - restart_max), dim=0))
            if max_idx < min_idx:
                sigma_restart = sd_schedulers.get_sigmas_karras(restart_steps, sigmas[min_idx].item(), sigmas[max_idx].item(), device=sigmas.device)[:-1]
                while restart_times > 0:
                    restart_times -= 1
                    step_list.extend(zip(sigma_restart[:-1], sigma_restart[1:]))
    last_sigma = None
    for old_sigma, new_sigma in step_list:
        if last_sigma is None:
            last_sigma = old_sigma
        elif last_sigma < old_sigma:
            noise = noise_sampler(last_sigma, old_sigma).float().contiguous()
            _lincomb(lib, x, [(x, 1.0), (noise, s_noise * float(old_sigma ** 2 - last_sigma ** 2) ** 0.5)], n)
        heun_step(old_sigma, new_sigma)
        last_sigma = new_sigma
    return x


# label, function, aliases, options — modules/sd_samplers_kdiffusion.py:11-27. The SDE family (DPM++ SDE / 2M SDE / 3M SDE:
# BrownianTreeNoiseSampler over torchsde) and DPM fast / adaptive are not mirrored.
samplers_k_diffusion = [
    ("DPM++ 2M", sample_dpmpp_2m, ["k_dpmpp_2m"], {"scheduler": "karras"}),
    ("DPM++ 2S a", sample_dpmpp_2s_ancestral, ["k_dpmpp_2s_a"], {"scheduler": "karras", "uses_ensd": True, "second_order": True}),
    ("Euler a", sample_euler_ancestral, ["k_euler_a", "k_euler_ancestral"], {"uses_ensd": True}),
    ("Euler", sample_euler, ["k_euler"], {}),
    ("LMS", sample_lms, ["k_lms"], {}),
    ("Heun", sample_heun, ["k_heun"], {"second_order": True}),
    ("DPM2", sample_dpm_2, ["k_dpm_2"], {"scheduler": "karras", "discard_next_to_last_sigma": True, "second_order": True}),
    ("DPM2 a", sample_dpm_2_ancestral, ["k_dpm_2_a"], {"scheduler": "karras", "discard_next_to_last_sigma": True, "uses_ensd": True, "second_order": True}),
    ("Restart", restart_sampler, ["restart"], {"scheduler": "karras", "second_order": True}),
]
sampler_extra_params = {  # modules/sd_samplers_kdiffusion.py:36-46
    sample_euler: ["s_churn", "s_tmin", "s_tmax", "s_noise"],
    sample_heun: ["s_churn", "s_tmin", "s_tmax", "s_noise"],
    sample_dpm_2: ["s_churn", "s_tmin", "s_tmax", "s_noise"],
    sample_dpm_2_ancestral: ["s_noise"],
    sample_dpmpp_2s_ancestral: ["s_noise"],
}
_sampler_map = {}
for _label, _fn, _aliases, _opts in samplers_k_diffusion:
    _sampler_map[_label.lower()] = (_label, _fn, _opts)
    for _a in _aliases:
        _sampler_map[_a.lower()] = (_label, _fn, _opts)
_sampler_map["dpm++ 2m karras"] = _sampler_map["dpm++ 2m"]  # pre-1.9 name (infotext compatibility)


class SchedulerOptions:
    """the `shared.opts` fields get_sigmas reads (defaults of modules/shared_options.py)."""

    always_discard_next_to_last_sigma = False
    use_old_karras_scheduler_sigmas = False
    sigma_min = 0.0
    sigma_max = 0.0
    rho = 0.0
    beta_dist_alpha = 0.6
    beta_dist_beta = 0.6
    sgm_noise_multiplier = False


class Sampler:
    """What every sampler shares (modules/sd_samplers_common.py:229-332 Sampler): per-job initialisation, the
    interrupt-to-last_latent rule and the step callback."""

    eta_default = 1.0  # opts.eta_ancestral; the timestep samplers use opts.eta_ddim

    def initialize(self, p) -> dict:
        """modules/sd_samplers_common.py:288-333: per-job state + the sampler function's optional arguments."""
        import inspect

        self.p = p
        cfg = self.model_wrap_cfg
        cfg.p = p
        cfg.mask = getattr(p, "mask", None)
        cfg.nmask = getattr(p, "nmask", None)
        cfg.step = 0
        self.eta = p.eta if getattr(p, "eta", None) is not None else self.eta_default
        self.s_min_uncond = getattr(p, "s_min_uncond", 0.0)
        params = inspect.signature(self.func).parameters
        kw = {}
        for name in sampler_extra_params.get(self.func, []):
            if hasattr(p, name) and name in params:
                kw[name] = getattr(p, name)
        if "s_tmax" in kw and not kw["s_tmax"]:
            kw["s_tmax"] = float("inf")  # 0 = inf
        if "eta" in params:
            kw["eta"] = self.eta
        if "noise_sampler" in params:
            kw["noise_sampler"] = lambda sigma, sigma_next: p.rng.next()  # TorchHijack.randn_like -> p.rng.next()
        return kw

    def launch_sampling(self, steps, func):
        self.model_wrap_cfg.steps = steps
        self.model_wrap_cfg.total_steps = steps
        state.sampling_steps = steps
        state.sampling_step = 0
        try:
            return func()
        except InterruptedException:
            return self.last_latent

    def callback_state(self, d):
        state.sampling_step = d["i"]


class KDiffusionSampler(Sampler):
    def __init__(self, funcname_or_label, sd_model, options=None):
        """funcname_or_label: a label or alias of the k-diffusion table, or a sampler function (options then start empty)."""
        if callable(funcname_or_label):
            self.label, self.func, self.options = funcname_or_label.__name__, funcname_or_label, {}
        else:
            key = funcname_or_label.lower() if isinstance(funcname_or_label, str) else None
            if key not in _sampler_map:
                raise L.SdxeError(f"sampler {funcname_or_label!r} is not mirrored (available: " + ", ".join(x[0] for x in samplers_k_diffusion) + ")")
            self.label, self.func, self.options = _sampler_map[key]
        if options:
            self.options = {**self.options, **options}
        self.sd_model = sd_model
        self.sched_opts = SchedulerOptions()
        self.model_wrap_cfg = CFGDenoiser(self)
        self.model_wrap = self.model_wrap_cfg.inner_model
        self.last_latent = None
        self.eta = 1.0
        self.s_noise = 1.0
        self.s_min_uncond = 0.0
        self.p = None
        self.sampler_extra_args = None

    # -- sigma schedule (modules/sd_samplers_kdiffusion.py:79-132) ------------------------------------------------
    def get_sigmas(self, p, steps: int) -> torch.Tensor:
        from . import sd_schedulers

        o = self.sched_opts
        discard = bool(self.options.get("discard_next_to_last_sigma", False)) or o.always_discard_next_to_last_sigma
        steps += 1 if discard else 0
        scheduler_name = (getattr(p, "hr_scheduler", None) if getattr(p, "is_hr_pass", False) else getattr(p, "scheduler", None)) or "Automatic"
        if scheduler_name == "Automatic":
            scheduler_name = self.options.get("scheduler", None)
        scheduler = sd_schedulers.schedulers_map.get(scheduler_name)
        if scheduler is None and scheduler_name is not None:
            raise L.SdxeError(f"unknown scheduler {scheduler_name!r}")
        m_sigma_min, m_sigma_max = self.model_wrap.sigmas[0].item(), self.model_wrap.sigmas[-1].item()
        sigma_min, sigma_max = (0.1, 10) if o.use_old_karras_scheduler_sigmas else (m_sigma_min, m_sigma_max)
        override = getattr(p, "sampler_noise_scheduler_override", None)
        if override:
            sigmas = override(steps)
        elif scheduler is None or scheduler.function is None:
            sigmas = self.model_wrap.get_sigmas(steps)
        else:
            kw = {"sigma_min": sigma_min, "sigma_max": sigma_max}
            if o.sigma_min != 0 and o.sigma_min != m_sigma_min:
                kw["sigma_min"] = o.sigma_min
            if o.sigma_max != 0 and o.sigma_max != m_sigma_max:
                kw["sigma_max"] = o.sigma_max
            if scheduler.default_rho != -1 and o.rho != 0 and o.rho != scheduler.default_rho:
                kw["rho"] = o.rho
            if scheduler.need_inner_model:
                kw["inner_model"] = self.model_wrap
            if scheduler.name == "align_your_steps":
                kw["is_sdxl"] = bool(getattr(self.sd_model, "is_sdxl", False))
            if scheduler.name == "beta":
                kw["alpha"], kw["beta"] = o.beta_dist_alpha, o.beta_dist_beta
            sigmas = scheduler.function(n=steps, **kw, device="cpu")
        if discard:
            sigmas = torch.cat([sigmas[:-2], sigmas[-1:]])
        return sigmas.cpu()

    def sample(self, p, x, conditioning, unconditional_conditioning, steps=None, image_conditioning=None):
        steps = steps or p.steps
        sigmas = self.get_sigmas(p, steps)
        if self.sched_opts.sgm_noise_multiplier:
            x = x * torch.sqrt(1.0 + sigmas[0] ** 2.0)
        else:
            x = x * sigmas[0]
        extra = self.initialize(p)
        self.last_latent = x
        self.sampler_extra_args = {"cond": conditioning, "image_cond": image_conditioning, "uncond": unconditional_conditioning,
                                   "cond_scale": p.cfg_scale, "s_min_uncond": self.s_min_uncond}
        return self.launch_sampling(steps, lambda: self.func(self.model_wrap_cfg, x, extra_args=self.sampler_extra_args,
                                                             disable=False, callback=self.callback_state, sigmas=sigmas, **extra))

    def sample_img2img(self, p, x, noise, conditioning, unconditional_conditioning, steps=None, image_conditioning=None):
        steps, t_enc = setup_img2img_steps(p, steps)
        sigmas = self.get_sigmas(p, steps)
        sigma_sched = sigmas[steps - t_enc - 1:]
        xi = x + noise * sigma_sched[0]
        extra = self.initialize(p)
        self.model_wrap_cfg.init_latent = x
        self.last_latent = x
        self.sampler_extra_args = {"cond": conditioning, "image_cond": image_conditioning, "uncond": unconditional_conditioning,
                                   "cond_scale": p.cfg_scale, "s_min_uncond": self.s_min_uncond}
        return self.launch_sampling(t_enc + 1, lambda: self.func(self.model_wrap_cfg, xi, extra_args=self.sampler_extra_args,
                                                                 disable=False, callback=self.callback_state,
                                                                 sigmas=sigma_sched, **extra))


def _all_samplers():
    """label / alias (lower case) -> (label, function, options, constructor) over the k-diffusion, timestep and LCM tables
    (modules/sd_samplers.py:11-16)."""
    global _all_sampler_map
    if _all_sampler_map is None:
        from . import sd_samplers_lcm, sd_samplers_timesteps

        table = {}
        for rows, ctor in ((samplers_k_diffusion, KDiffusionSampler), (sd_samplers_timesteps.samplers_timesteps, sd_samplers_timesteps.CompVisSampler),
                           (sd_samplers_lcm.samplers_lcm, sd_samplers_lcm.LCMSampler)):
            for label, fn, aliases, opts in rows:
                for name in [label] + aliases:
                    table[name.lower()] = (label, fn, opts, ctor)
        table["dpm++ 2m karras"] = table["dpm++ 2m"]  # pre-1.9 name (infotext compatibility)
        _all_sampler_map = table
    return _all_sampler_map


_all_sampler_map = None


def find_sampler_config(name):
    """modules/sd_samplers.py:18-24 — (label, function, options) of a sampler by label or alias, None when unknown."""
    entry = _all_samplers().get(str(name).lower())
    return None if entry is None else entry[:3]


def create_sampler(name, model) -> Sampler:
    """modules/sd_samplers.py:33."""
    entry = _all_samplers().get(str(name).lower())
    if entry is None:
        raise L.SdxeError(f"sampler {name!r} is not mirrored (available: " + ", ".join(sorted({e[0] for e in _all_samplers().values()})) + ")")
    return entry[3](entry[0], model)
