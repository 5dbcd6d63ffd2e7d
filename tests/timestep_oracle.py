"""fp32 torch reference for the timestep samplers (DDIM, DDIM CFG++, PLMS, UniPC) and LCM end to end: the webui glue of
modules/sd_samplers_timesteps.py and modules/sd_samplers_lcm.py on top of oracle.pipeline.OraclePipeline and
oracle.cfg_denoiser.CFGDenoiser. The step formulas are plain torch; UniPC's host-side coefficients come from
sdwebui_b200.sd_samplers_timesteps, which tests/golden/timesteps_ref.npz pins to the reference's own solver."""
import math

import torch
import torch.nn.functional as F

from oracle import kdiffusion as K
from oracle.cfg_denoiser import CFGDenoiser, make_apply_model
from oracle.pipeline import OraclePipeline
from oracle.rng import ImageRNG

TIMESTEP_SAMPLERS = ("DDIM", "DDIM CFG++", "PLMS", "UniPC")


class CFGTimesteps(CFGDenoiser):
    """CFGDenoiserTimesteps: raw eps from the UNet, the latent mask blended in BEFORE the model call; keeps the
    uncond eps for CFG++ (scale multiplier 1 / 12.5)."""

    def __init__(self, apply_model, mask=None, nmask=None, init_latent=None, cond_scale_mult=1.0):
        self.uncond_eps = None

        def inner(x, t, **kw):
            out = apply_model(x, t, **kw).float()
            self.uncond_eps = out[-x.shape[0] // 2:] if not self._skip else None
            return out

        super().__init__(inner)
        self.blend = (mask, nmask, init_latent)
        self.mult = cond_scale_mult
        self._skip = False

    def __call__(self, x, sigma, uncond, cond, cond_scale, s_min_uncond=0.0, **kw):
        mask, nmask, init_latent = self.blend
        if mask is not None:
            x = x * nmask + init_latent * mask
        self._skip = bool(self.step % 2 and s_min_uncond > 0 and sigma[0] < s_min_uncond)
        return super().__call__(x, sigma, uncond, cond, cond_scale * self.mult, s_min_uncond, **kw)


class LCMDenoiser(K.DiscreteSchedule):
    """LCMCompVisDenoiser: 50 kept steps, nearest-step timesteps, consistency output with sigma_data 0.5."""

    def __init__(self, apply_model, alphas_cumprod):
        super().__init__(torch.stack([alphas_cumprod[999 - (49 - i) * 20] for i in range(50)]))
        self.apply_model = apply_model

    def get_sigmas(self, n):
        start, end = self.sigma_to_t(self.sigmas[-1]), self.sigma_to_t(self.sigmas[0])
        t = torch.linspace(float(start), float(end), n, device=self.sigmas.device)
        return torch.cat([self.t_to_sigma(t), t.new_zeros([1])])

    def sigma_to_t(self, sigma):
        return (sigma.log() - self.log_sigmas.to(sigma.device)[:, None]).abs().argmin(dim=0).view(sigma.shape) * 20 + 19

    def t_to_sigma(self, t):
        return super().t_to_sigma(torch.clamp((t - 19) / 20, 0, 49).float())

    def __call__(self, x, sigma, **kwargs):
        s = sigma.view(-1, 1, 1, 1)
        eps = self.apply_model(x / (s ** 2 + 1) ** 0.5, self.sigma_to_t(sigma), **kwargs).float()
        ts = self.sigma_to_t(sigma).float().view(-1, 1, 1, 1) * 10
        return ts / (ts ** 2 + 0.25) ** 0.5 * (x - s * eps) + 0.25 / (ts ** 2 + 0.25) * x


def get_timesteps(steps):
    return torch.clip(torch.arange(0, 1000, 1000 // steps) + 1, 0, 999)


def ddim(model, x, timesteps, ac, extra, eta=0.0, noise=None, cfgpp=False):
    ts = [int(t) for t in timesteps]
    a = ac[ts].double().cpu()
    a_prev = ac[[0] + ts[:-1]].double().cpu()
    sig = eta * ((1 - a_prev) / (1 - a) * (1 - a / a_prev)).sqrt()
    s_in = x.new_ones([x.shape[0]])
    for i in range(len(ts) - 1):
        k = len(ts) - 1 - i
        e = model(x, ts[k] * s_in, **extra)
        pred_x0 = (x - math.sqrt(1 - a[k]) * e) / math.sqrt(a[k])
        d = model.uncond_eps if cfgpp else e
        x = math.sqrt(a_prev[k]) * pred_x0 + math.sqrt(1 - a_prev[k] - sig[k] ** 2) * d
        if sig[k] != 0:
            x = x + float(sig[k]) * noise()
    return x


def plms(model, x, timesteps, ac, extra):
    ts = [int(t) for t in timesteps]
    a = ac[ts].double().cpu()
    a_prev = ac[[0] + ts[:-1]].double().cpu()
    s_in = x.new_ones([x.shape[0]])

    def step(x, e, k):
        return math.sqrt(a_prev[k]) * (x - math.sqrt(1 - a[k]) * e) / math.sqrt(a[k]) + math.sqrt(1 - a_prev[k]) * e

    old = []
    for i in range(len(ts) - 1):
        k = len(ts) - 1 - i
        e = model(x, ts[k] * s_in, **extra)
        if not old:
            e_p = (e + model(step(x, e, k), ts[max(k - 1, 0)] * s_in, **extra)) / 2
        elif len(old) == 1:
            e_p = (3 * e - old[-1]) / 2
        elif len(old) == 2:
            e_p = (23 * e - 16 * old[-1] + 5 * old[-2]) / 12
        else:
            e_p = (55 * e - 59 * old[-1] + 37 * old[-2] - 9 * old[-3]) / 24
        x = step(x, e_p, k)
        old = (old + [e])[-3:]
    return x


def unipc(model, x, timesteps, ac, extra, is_img2img=False, variant="bh1", skip_type="time_uniform", order=3, lower_order_final=True):
    from sdwebui_b200 import sd_samplers_timesteps as T

    ns = T.NoiseScheduleVP("discrete", alphas_cumprod=ac)
    coef = T.UniPCSampler.__new__(T.UniPCSampler)
    coef.ns, coef.variant = ns, variant
    s_in = x.new_ones([x.shape[0]])

    def model_fn(x, t):
        e = model(x, s_in * ((t - 1 / 1000) * 1000), **extra)
        return (x - float(ns.marginal_std(t)) * e) / float(ns.marginal_alpha(t))

    def update(x, ms, tl, t, o, corr):
        c_x, c_m0, rks, w_p, w_c, w_t = coef._coefficients(tl, t, o, corr)
        d = lambda w: sum(w[k] * (ms[-(k + 2)] - ms[-1]) / rks[k] for k in range(len(w)))  # noqa: E731
        base = c_x * x + c_m0 * ms[-1]
        x_t = base + (d(w_p) if w_p is not None else 0)
        m_t = None
        if corr:
            m_t = model_fn(x_t, t)
            x_t = base + (d(w_c) if o > 1 else 0) + w_t * (m_t - ms[-1])
        return x_t, m_t

    steps = len(timesteps)
    t_T = float(timesteps[-1]) / 1000 + 1 / 1000 if is_img2img else 1.0
    grid = [float(v) for v in T.get_time_steps(ns, skip_type, t_T, 1 / 1000, steps)]
    ms, tl = [model_fn(x, grid[0])], [grid[0]]
    for o in range(1, order):
        x, m = update(x, ms, tl, grid[o], o, True)
        ms.append(m)
        tl.append(grid[o])
    for step in range(order, steps + 1):
        o = min(order, steps + 1 - step) if lower_order_final else order
        x, m = update(x, ms, tl, grid[step], o, step != steps)
        ms, tl = ms[1:] + ms[-1:], tl[1:] + [grid[step]]
        if step < steps:
            ms[-1] = m
    return x


def sample_lcm(model, x, sigmas, extra, noise):
    s_in = x.new_ones([x.shape[0]])
    for i in range(len(sigmas) - 1):
        x = model(x, sigmas[i] * s_in, **extra)
        if sigmas[i + 1] > 0:
            x = x + sigmas[i + 1] * noise()
    return x


class SamplerOraclePipeline(OraclePipeline):
    """OraclePipeline with the timestep samplers and LCM: txt2img (+ hires pass) and latent-masked img2img."""

    def __init__(self, unet, vae, device, dtype_unet=torch.float32, dtype_vae=None, autocast=False, eta=0.0, s_min_uncond=0.0):
        super().__init__(unet, vae, device, dtype_unet, dtype_vae, autocast)
        self.apply_model = make_apply_model(unet, dtype_unet, autocast)
        self.eta, self.s_min_uncond = eta, s_min_uncond

    def _loop(self, name, x, cond, uncond, cfg_scale, rng, steps, t_enc=None, blend=(None, None, None)):
        extra = {"cond": cond, "uncond": uncond, "cond_scale": cfg_scale, "s_min_uncond": self.s_min_uncond}
        ac = self.alphas_cumprod
        if name == "LCM":
            den = LCMDenoiser(self.apply_model, ac)
            sig = den.get_sigmas(steps).to(x.device)
            cfg = CFGDenoiser(den, *blend) if blend[0] is not None else CFGDenoiser(den)
            if t_enc is None:
                return sample_lcm(cfg, x * sig[0], sig, extra, rng.next)
            sched = sig[steps - t_enc - 1:]
            return sample_lcm(cfg, x[0] + x[1] * sched[0], sched, extra, rng.next)
        cfg = CFGTimesteps(self.apply_model, *blend, cond_scale_mult=1 / 12.5 if name == "DDIM CFG++" else 1.0)
        ts = get_timesteps(steps)
        if t_enc is not None:
            a = ac[int(ts[t_enc])]
            x = x[0] * a.sqrt() + x[1] * (1 - a).sqrt()
            ts = ts[:t_enc]
        if name in ("DDIM", "DDIM CFG++"):
            return ddim(cfg, x, ts, ac, extra, eta=self.eta, noise=rng.next, cfgpp=name == "DDIM CFG++")
        if name == "PLMS":
            return plms(cfg, x, ts, ac, extra)
        return unipc(cfg, x, ts, ac, extra, is_img2img=t_enc is not None)

    @torch.no_grad()
    def sample(self, p, cond, uncond, y_cond=None, y_uncond=None):
        B = len(p.seeds)
        rng = ImageRNG((4, p.height // 8, p.width // 8), p.seeds, source=p.randn_source, device=self.device)
        samples = self._loop(p.sampler, rng.next(), cond, uncond, p.cfg_scale, rng, p.steps)
        if not p.enable_hr:
            return samples
        th, tw = int(p.height * p.hr_scale) // 8, int(p.width * p.hr_scale) // 8
        samples = F.interpolate(samples, size=(th, tw), mode="bilinear", antialias=False)
        rng2 = ImageRNG((4, th, tw), p.seeds, source=p.randn_source, device=self.device)
        noise = rng2.next()
        steps, t_enc = K.setup_img2img_steps(p.hr_second_pass_steps or p.steps, p.denoising_strength)
        assert B == samples.shape[0]
        return self._loop(p.sampler, (samples, noise), cond, uncond, p.cfg_scale, rng2, steps, t_enc)

    @torch.no_grad()
    def img2img_latent(self, p, init_latent, cond, uncond, latent_mask=None):
        """img2img from a given init latent (the VAE encode is shared with the k-diffusion tests)."""
        rng = ImageRNG((4, p.height // 8, p.width // 8), p.seeds, source=p.randn_source, device=self.device)
        noise = rng.next()
        steps, t_enc = K.setup_img2img_steps(p.steps, p.denoising_strength, steps_given=False)
        blend = (None, None, None)
        if latent_mask is not None:
            nmask = torch.round(latent_mask.to(self.device, torch.float32)).expand(init_latent.shape)
            blend = (1.0 - nmask, nmask, init_latent)
        out = self._loop(p.sampler, (init_latent, noise), cond, uncond, p.cfg_scale, rng, steps, t_enc, blend)
        if latent_mask is not None:
            out = out * blend[1] + init_latent * blend[0]
        return out
