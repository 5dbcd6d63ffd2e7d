"""The toy models, inputs and draw sequences shared by tests/golden/make_golden_timesteps.py (which runs the reference's
timestep and LCM samplers on them) and the tests that replay them through the product."""
import torch

STEPS = (4, 10, 20)
LCM_STEPS = (4, 8)
UNIPC_VARIANTS = ("bh1", "bh2", "vary_coeff")
UNIPC_SKIPS = ("time_uniform", "time_quadratic", "logSNR")
UNIPC_ORDERS = (1, 2, 3)
LATENT = (4, 4, 4)   # per-image latent shape of the toy runs


def img2img_t_enc(steps):
    """t_enc of setup_img2img_steps at denoising strength 0.75."""
    return int(0.75 * steps)


def x_init(B, steps, img2img):
    return torch.randn((B,) + LATENT, generator=torch.Generator().manual_seed(steps * 2 + int(img2img)))


class CountingNoise:
    """randn_like replacement: a fixed, seeded sequence of draws."""

    def __init__(self, shape, seed, device="cpu"):
        self.g = torch.Generator().manual_seed(seed)
        self.shape, self.device = shape, device

    def randn_like(self, x=None):
        return torch.randn(self.shape, generator=self.g).to(self.device)

    def __call__(self, *a):
        return self.randn_like()


class ToyTimestepModel:
    """Stands in for CFGDenoiserTimesteps: a smooth, nonlinear guided eps(x, t) at cond_scale 7, with the attributes the
    timestep samplers touch (alphas_cumprod behind inner_model.inner_model, CFG++'s scale multiplier and uncond eps)."""

    def __init__(self, alphas_cumprod):
        self.inner_model = type("W", (), {})()
        self.inner_model.inner_model = type("M", (), {})()
        self.inner_model.inner_model.alphas_cumprod = alphas_cumprod
        self.cond_scale_miltiplier = 1.0
        self.need_last_noise_uncond = False
        self.last_noise_uncond = None
        self.calls = []

    def __call__(self, x, t, **kwargs):
        self.calls.append(float(t[0]))
        s = (t.float() / 1000.0).view(-1, 1, 1, 1).to(x.device)
        e_c = x * (0.3 + 0.5 * s) + 0.2 * torch.tanh(x) * (1 - s)
        e_u = 0.9 * x * (0.3 + 0.5 * s) + 0.1 * torch.sin(x)
        if self.need_last_noise_uncond:
            self.last_noise_uncond = e_u
        return e_u + (e_c - e_u) * (7.0 * self.cond_scale_miltiplier)


def lcm_toy_apply_model(x, t, **kwargs):
    """eps(x, t) for the LCM denoiser's UNet slot."""
    s = (t.float() / 1000.0).view(-1, 1, 1, 1).to(x.device)
    return 0.7 * x + 0.1 * torch.tanh(x) * s
