"""The LCM sampler on the engine (modules/sd_samplers_lcm.py): latent consistency models sample in 4-8 steps with
LCM-distilled weights or an LCM LoRA (merged at SdxeUnet.activate()).

LCMCompVisDenoiser keeps every 20th step of the 1000-step schedule (50 entries) and turns the eps prediction into the
consistency output c_out' * (x - sigma * eps) + c_skip' * x with sigma_data = 0.5 and the timestep scaled by 10. That output
is affine in (x, eps) with the same coefficients for every UNet row of an image, so the CFG combine is one
sdxe_cfg_combine_affine launch; the step itself (x = denoised + sigma_next * noise) is one sdxe_lincomb.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

from . import lib as L
from . import samplers as S


class LCMCompVisDenoiser(S.CompVisDenoiser):
    sigma_data_lcm = 0.5

    def __init__(self, sd_model):
        timesteps, original_timesteps = 1000, 50
        self.skip_steps = timesteps // original_timesteps
        ac = sd_model.alphas_cumprod
        valid = torch.stack([ac[timesteps - 1 - (original_timesteps - 1 - i) * self.skip_steps] for i in range(original_timesteps)])
        S.DiscreteSchedule.__init__(self, valid.float(), sd_model.device)
        self.inner_model = sd_model

    def get_sigmas(self, n=None):
        """n sigmas linear in timestep from the largest to the smallest kept step, then 0; None: the 50 kept sigmas."""
        if n is None:
            return torch.cat([self.sigmas.flip(0), self.sigmas.new_zeros([1])])
        start, end = self.sigma_to_t(self.sigmas[-1]), self.sigma_to_t(self.sigmas[0])
        t = torch.linspace(float(start), float(end), n, device=self.sigmas.device)
        return torch.cat([self.t_to_sigma(t), t.new_zeros([1])])

    def sigma_to_t(self, sigma):
        """the nearest kept step (in log sigma), as a timestep of the 1000-step schedule."""
        dists = sigma.log() - self.log_sigmas[:, None]
        return dists.abs().argmin(dim=0).view(sigma.shape) * self.skip_steps + (self.skip_steps - 1)

    def t_to_sigma(self, t):
        t = torch.clamp(((t - (self.skip_steps - 1)) / self.skip_steps).float(), min=0, max=len(self.sigmas) - 1)
        return super().t_to_sigma(t)

    def lcm_scalings(self, sigma):
        """(c_skip', c_out') of the consistency parameterisation at sigma."""
        ts = self.sigma_to_t(sigma).float() * 10.0
        sd2 = self.sigma_data_lcm ** 2
        return sd2 / (ts ** 2 + sd2), ts / (ts ** 2 + sd2) ** 0.5

    def forward(self, x, sigma, **kwargs):
        c_out, c_in = [s.view(-1, 1, 1, 1) for s in self.get_scalings(sigma)]
        eps = self.inner_model.apply_model(x * c_in, self.sigma_to_t(sigma), **kwargs)
        c_skip2, c_out2 = [s.view(-1, 1, 1, 1) for s in self.lcm_scalings(sigma)]
        return c_out2 * (x + eps * c_out) + c_skip2 * x

    __call__ = forward


class CFGDenoiserLCM(S.CFGDenoiser):
    @property
    def inner_model(self):
        if self.model_wrap is None:
            self.model_wrap = LCMCompVisDenoiser(self.sampler.sd_model)
        return self.model_wrap

    def combine(self, x, eps, sigma, sigma_in, conds_list, skip_uncond, scale):
        # per row: c_out' (x - sigma eps) + c_skip' x = (c_out' + c_skip') x + (-sigma c_out') eps
        c_skip, c_out = self.inner_model.lcm_scalings(sigma)
        cx, ce = (c_out + c_skip).contiguous(), (-sigma * c_out).contiguous()
        return self.combine_affine(x, eps, conds_list, skip_uncond, scale, cx, ce)[0]


class LCMSampler(S.KDiffusionSampler):
    def __init__(self, funcname, sd_model, options=None):
        super().__init__(sample_lcm, sd_model, options)
        self.label = "LCM"
        self.model_wrap_cfg = CFGDenoiserLCM(self)
        self.model_wrap = self.model_wrap_cfg.inner_model


@torch.no_grad()
def sample_lcm(model, x, sigmas, extra_args=None, callback=None, disable=None, noise_sampler: Optional[Callable] = None):
    """x <- denoised, plus sigma_next * fresh noise while sigma_next > 0. noise_sampler(sigma, sigma_next) -> noise like x
    (the webui's randn_like, i.e. p.rng.next())."""
    extra_args, lib, x, sig = S._prep(x, sigmas, extra_args)
    if noise_sampler is None:
        noise_sampler = lambda sigma, sigma_next: torch.randn_like(x)  # noqa: E731
    s_in, n = x.new_ones([x.shape[0]]), x.numel()
    for i in range(len(sig) - 1):
        denoised = model(x, s_in * sig[i], **extra_args).contiguous()
        if callback is not None:
            callback({"x": x, "i": i, "sigma": sigmas[i], "sigma_hat": sigmas[i], "denoised": denoised})
        if sig[i + 1] > 0:
            x = S._lincomb(lib, torch.empty_like(x), [(denoised, 1.0), (noise_sampler(sigmas[i], sigmas[i + 1]).float().contiguous(), sig[i + 1])], n)
        else:
            x = denoised
    return x


# label, function, aliases, options — modules/sd_samplers_lcm.py:100
samplers_lcm = [("LCM", sample_lcm, ["k_lcm"], {})]
