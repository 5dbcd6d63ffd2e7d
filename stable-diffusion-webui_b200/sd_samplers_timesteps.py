"""The timestep samplers DDIM, DDIM CFG++, PLMS and UniPC on the engine, with the reference's names and behaviour:

  CompVisTimestepsDenoiser, CFGDenoiserTimesteps, CompVisSampler   modules/sd_samplers_timesteps.py
  ddim, ddim_cfgpp, plms, unipc                                    modules/sd_samplers_timesteps_impl.py
  NoiseScheduleVP ('discrete'), the UniPC multistep solver         modules/models/diffusion/uni_pc/uni_pc.py

The UNet sees raw timesteps (c_in = 1) and returns eps. The CFG combine, the first cond's pred_x0 (what an interrupted job
returns) and, for CFG++, the uncond eps come out of one sdxe_cfg_combine_affine launch per denoiser call. Every update is
sdxe_lincomb with scalars computed on the host; UniPC's small linear solve for its coefficients runs on the host too.

Reproduced as the reference has them: DDIM and PLMS make len(timesteps) - 1 denoiser calls (the lowest timestep is never
visited) and PLMS calls the model twice on its first step; s_min_uncond is compared against the timestep value; UniPC's
img2img start time is timesteps[-1] / 1000 + 1 / 1000. v-prediction checkpoints stay unsupported, as on the k-diffusion
path. The reference's vary_coeff solver only runs with one image per batch; here it runs with any batch size.
"""
from __future__ import annotations

import inspect
import math

import numpy as np
import torch

from . import lib as L
from . import samplers as S


# ------------------------------------------------------------------------------------------------------------------
# denoiser
# ------------------------------------------------------------------------------------------------------------------
class CompVisTimestepsDenoiser:
    """eps(x, t) of the model at integer-scaled timesteps t in [0, 1000)."""

    def __init__(self, sd_model):
        if getattr(sd_model, "parameterization", "eps") == "v":
            raise L.SdxeError("v-prediction checkpoints are not supported by the engine")
        self.inner_model = sd_model
        self.alphas_cumprod = sd_model.alphas_cumprod

    def __call__(self, x, timesteps, **kwargs):
        return self.inner_model.apply_model(x, timesteps, **kwargs)


class CFGDenoiserTimesteps(S.CFGDenoiser):
    """CFGDenoiser over CompVisTimestepsDenoiser: the mask is blended in before the model call, the returned value is the
    guided eps, and the sampler's last_latent is the first cond's pred_x0."""

    def __init__(self, sampler):
        super().__init__(sampler)
        self.alphas = sampler.sd_model.alphas_cumprod
        self.mask_before_denoising = True
        self._pred_x0 = None

    @property
    def inner_model(self):
        if self.model_wrap is None:
            self.model_wrap = CompVisTimestepsDenoiser(self.sampler.sd_model)
        return self.model_wrap

    def get_pred_x0(self, x_in, x_out, sigma):
        """x0 implied by eps x_out at timestep sigma (torch form of what the combine kernel writes as x0_out)."""
        a_t = self.alphas[sigma.to(dtype=torch.int64)][:, None, None, None]
        return (x_in - (1 - a_t).sqrt() * x_out) / a_t.sqrt()

    def model_inputs(self, sigma_in):
        ones = self._dev(("ones", sigma_in.shape[0]), lambda: torch.ones(sigma_in.shape[0], device=sigma_in.device))
        return ones, sigma_in

    def combine(self, x, eps, sigma, sigma_in, conds_list, skip_uncond, scale):
        B = x.shape[0]
        cx, ce = self._dev(("eps_coef", B), lambda: (torch.zeros(B, device=x.device), torch.ones(B, device=x.device)))
        a_t = self.alphas[sigma.to(dtype=torch.int64)]
        x0_coef = torch.stack([a_t.rsqrt(), -(1 - a_t).sqrt() / a_t.sqrt()], dim=1).contiguous()
        out, self._pred_x0, unc = self.combine_affine(x, eps, conds_list, skip_uncond, scale, cx, ce, x0_coef,
                                                      want_uncond=self.need_last_noise_uncond)
        if unc is not None:
            self.last_noise_uncond = unc
        return out

    def last_latent(self, denoised):
        return self._pred_x0


# ------------------------------------------------------------------------------------------------------------------
# sampler loops
# ------------------------------------------------------------------------------------------------------------------
def _lincomb(lib, out, terms, n):
    """out = sum(c * t) over any number of (tensor, coefficient) terms: four per sdxe_lincomb launch, chained through out."""
    terms = [(t, c) for t, c in terms if c != 0.0] or [(terms[0][0], 0.0)]
    S._lincomb(lib, out, terms[:4], n)
    for i in range(4, len(terms), 3):
        S._lincomb(lib, out, [(out, 1.0)] + terms[i:i + 3], n)
    return out


def _ddim_tables(alphas_cumprod, timesteps, eta):
    """Per index into timesteps: alpha_t (fp32 as stored), alpha_prev (alpha of the previous timestep, alphas_cumprod[0] for
    the first) and sigma_t = eta * sqrt((1 - a_prev) / (1 - a_t) * (1 - a_t / a_prev))."""
    ac = alphas_cumprod.detach().float().cpu().numpy()
    ts = [int(t) for t in timesteps]
    a = np.array([ac[t] for t in ts], dtype=np.float64)
    a_prev = np.array([ac[0]] + [ac[t] for t in ts[:-1]], dtype=np.float64)
    sig = eta * np.sqrt((1 - a_prev) / (1 - a) * (1 - a / a_prev))
    return ts, a, a_prev, sig


def _ddim_loop(model, x, timesteps, extra_args, callback, eta, noise_sampler, cfgpp):
    extra_args = {} if extra_args is None else extra_args
    lib = L.load()
    x = x.float().contiguous().clone()
    s_in, n = x.new_ones([x.shape[0]]), x.numel()
    ts, a, a_prev, sig = _ddim_tables(model.inner_model.inner_model.alphas_cumprod, timesteps, eta)
    if noise_sampler is None:
        noise_sampler = lambda sigma, sigma_next: torch.randn_like(x)  # noqa: E731
    if cfgpp:
        model.cond_scale_miltiplier = 1 / 12.5
        model.need_last_noise_uncond = True
    for i in range(len(ts) - 1):
        index = len(ts) - 1 - i
        e_t = model(x, ts[index] * s_in, **extra_args).contiguous()
        sq_at, sq_prev = math.sqrt(a[index]), math.sqrt(a_prev[index])
        s1m = math.sqrt(1 - a[index])
        dir_c = math.sqrt(1.0 - a_prev[index] - sig[index] ** 2)
        # x' = sqrt(a_prev) * pred_x0 + dir_c * (eps or CFG++'s uncond eps) + sigma_t * noise, pred_x0 = (x - s1m eps) / sqrt(a_t)
        terms = [(x, sq_prev / sq_at), (e_t, -sq_prev * s1m / sq_at + (0.0 if cfgpp else dir_c))]
        if cfgpp:
            terms.append((model.last_noise_uncond, dir_c))
        if sig[index] != 0:
            terms.append((noise_sampler(None, None).float().contiguous(), float(sig[index])))
        if callback is not None:
            pred_x0 = _lincomb(lib, torch.empty_like(x), [(x, 1 / sq_at), (e_t, -s1m / sq_at)], n)
        x = _lincomb(lib, torch.empty_like(x), terms, n)
        if callback is not None:
            callback({"x": x, "i": i, "sigma": 0, "sigma_hat": 0, "denoised": pred_x0})
    return x


@torch.no_grad()
def ddim(model, x, timesteps, extra_args=None, callback=None, disable=None, eta=0.0, noise_sampler=None):
    """DDIM (Song et al. 2020) over the given timesteps, from the last one down to the second; eta scales the fresh noise.
    noise_sampler() -> noise like x (the webui's randn_like, i.e. p.rng.next()); not called when eta is 0."""
    return _ddim_loop(model, x, timesteps, extra_args, callback, eta, noise_sampler, cfgpp=False)


@torch.no_grad()
def ddim_cfgpp(model, x, timesteps, extra_args=None, callback=None, disable=None, eta=0.0, noise_sampler=None):
    """CFG++ (Chung et al. 2024) on DDIM: the guidance scale is divided by 12.5 and the step direction uses the uncond
    eps instead of the guided one."""
    return _ddim_loop(model, x, timesteps, extra_args, callback, eta, noise_sampler, cfgpp=True)


@torch.no_grad()
def plms(model, x, timesteps, extra_args=None, callback=None, disable=None):
    """Pseudo linear multistep (Liu et al. 2022): Adams-Bashforth combinations of up to four past eps in the DDIM step;
    the first step is a pseudo improved Euler step with a second model call."""
    extra_args = {} if extra_args is None else extra_args
    lib = L.load()
    x = x.float().contiguous().clone()
    s_in, n = x.new_ones([x.shape[0]]), x.numel()
    ts, a, a_prev, _ = _ddim_tables(model.inner_model.inner_model.alphas_cumprod, timesteps, 0.0)

    def step_terms(e, index):  # x_prev = sqrt(a_prev) (x - sqrt(1 - a_t) e) / sqrt(a_t) + sqrt(1 - a_prev) e
        sq_at, sq_prev, s1m = math.sqrt(a[index]), math.sqrt(a_prev[index]), math.sqrt(1 - a[index])
        return [(x, sq_prev / sq_at), (e, math.sqrt(1 - a_prev[index]) - sq_prev * s1m / sq_at)]

    old_eps = []
    for i in range(len(ts) - 1):
        index = len(ts) - 1 - i
        e_t = model(x, ts[index] * s_in, **extra_args).contiguous()
        e_prime = torch.empty_like(x)
        if not old_eps:
            x_prev = _lincomb(lib, torch.empty_like(x), step_terms(e_t, index), n)
            e_next = model(x_prev, ts[max(index - 1, 0)] * s_in, **extra_args).contiguous()
            _lincomb(lib, e_prime, [(e_t, 0.5), (e_next, 0.5)], n)
        elif len(old_eps) == 1:
            _lincomb(lib, e_prime, [(e_t, 1.5), (old_eps[-1], -0.5)], n)
        elif len(old_eps) == 2:
            _lincomb(lib, e_prime, [(e_t, 23 / 12), (old_eps[-1], -16 / 12), (old_eps[-2], 5 / 12)], n)
        else:
            _lincomb(lib, e_prime, [(e_t, 55 / 24), (old_eps[-1], -59 / 24), (old_eps[-2], 37 / 24), (old_eps[-3], -9 / 24)], n)
        x_new = _lincomb(lib, torch.empty_like(x), step_terms(e_prime, index), n)
        if callback is not None:
            sq_at, s1m = math.sqrt(a[index]), math.sqrt(1 - a[index])
            pred_x0 = _lincomb(lib, torch.empty_like(x), [(x, 1 / sq_at), (e_prime, -s1m / sq_at)], n)
        old_eps.append(e_t)
        if len(old_eps) >= 4:
            old_eps.pop(0)
        x = x_new
        if callback is not None:
            callback({"x": x, "i": i, "sigma": 0, "sigma_hat": 0, "denoised": pred_x0})
    return x


# ------------------------------------------------------------------------------------------------------------------
# UniPC (Zhao et al. 2023, "UniPC: A Unified Predictor-Corrector Framework for Fast Sampling of Diffusion Models")
# ------------------------------------------------------------------------------------------------------------------
class NoiseScheduleVP:
    """The discrete VP schedule as a function of continuous time: step n of N sits at t = (n + 1) / N, and
    log alpha_t = 0.5 * log(alphas_cumprod) is interpolated linearly in t (extrapolated from the end segments)."""

    def __init__(self, schedule="discrete", alphas_cumprod=None):
        if schedule != "discrete":
            raise L.SdxeError(f"NoiseScheduleVP: only the 'discrete' schedule is supported, not {schedule!r}")
        ac = np.asarray(torch.as_tensor(alphas_cumprod).detach().double().cpu(), dtype=np.float64)
        self.total_N = len(ac)
        self.T = 1.0
        self.t_array = np.arange(1, self.total_N + 1, dtype=np.float64) / self.total_N
        self.log_alpha_array = 0.5 * np.log(ac)

    @staticmethod
    def _interp(x, xp, yp):
        """piecewise linear through (xp, yp), xp increasing, continued linearly beyond both ends."""
        x = np.asarray(x, dtype=np.float64)
        i = np.clip(np.searchsorted(xp, x) - 1, 0, len(xp) - 2)
        return yp[i] + (x - xp[i]) * (yp[i + 1] - yp[i]) / (xp[i + 1] - xp[i])

    def marginal_log_mean_coeff(self, t):
        return self._interp(t, self.t_array, self.log_alpha_array)

    def marginal_alpha(self, t):
        return np.exp(self.marginal_log_mean_coeff(t))

    def marginal_std(self, t):
        return np.sqrt(1.0 - np.exp(2.0 * self.marginal_log_mean_coeff(t)))

    def marginal_lambda(self, t):
        lmc = self.marginal_log_mean_coeff(t)
        return lmc - 0.5 * np.log(1.0 - np.exp(2.0 * lmc))

    def inverse_lambda(self, lamb):
        log_alpha = -0.5 * np.logaddexp(0.0, -2.0 * np.asarray(lamb, dtype=np.float64))
        return self._interp(log_alpha, self.log_alpha_array[::-1], self.t_array[::-1])


class UniPCOptions:
    """The `shared.opts` fields the UniPC sampler reads (defaults: modules/shared_options.py:402-405)."""

    uni_pc_variant = "bh1"              # bh1 | bh2 | vary_coeff
    uni_pc_skip_type = "time_uniform"   # time_uniform | time_quadratic | logSNR
    uni_pc_order = 3
    uni_pc_lower_order_final = True


def get_time_steps(ns: NoiseScheduleVP, skip_type, t_T, t_0, N):
    """N + 1 times from t_T down to t_0: uniform in t, uniform in sqrt(t), or uniform in logSNR (lambda)."""
    if skip_type == "logSNR":
        lam = np.linspace(float(ns.marginal_lambda(t_T)), float(ns.marginal_lambda(t_0)), N + 1)
        return ns.inverse_lambda(lam)
    if skip_type == "time_uniform":
        return np.linspace(t_T, t_0, N + 1)
    if skip_type == "time_quadratic":
        return np.linspace(t_T ** 0.5, t_0 ** 0.5, N + 1) ** 2
    raise L.SdxeError(f"unsupported UniPC skip type {skip_type!r} (logSNR, time_uniform or time_quadratic)")


class UniPCSampler:
    """Multistep UniPC in data-prediction form (thresholding off): each model evaluation returns
    x0 = (x - sigma_t * eps) / alpha_t; every update is a linear combination of x and past x0 with host coefficients."""

    def __init__(self, cfg_model, extra_args, callback, ns: NoiseScheduleVP, variant="bh1"):
        if variant not in ("bh1", "bh2", "vary_coeff"):
            raise L.SdxeError(f"unsupported UniPC variant {variant!r} (bh1, bh2 or vary_coeff)")
        self.cfg_model, self.extra_args, self.callback = cfg_model, extra_args, callback
        self.ns, self.variant = ns, variant
        self.index = 0
        self.lib = L.load()

    def model_fn(self, x, t):
        """x0 from the guided eps at continuous time t; the CFG denoiser sees the timestep (t - 1/N) * 1000."""
        s_in = x.new_ones([x.shape[0]])
        eps = self.cfg_model(x, s_in * ((t - 1.0 / self.ns.total_N) * 1000.0), **self.extra_args).contiguous()
        alpha_t, sigma_t = float(self.ns.marginal_alpha(t)), float(self.ns.marginal_std(t))
        return _lincomb(self.lib, torch.empty_like(x), [(x, 1.0 / alpha_t), (eps, -sigma_t / alpha_t)], x.numel())

    def _coefficients(self, t_prev_list, t, order, use_corrector):
        """-> (coefficient of x, of model_prev_list[-1], of model_prev_list[-(k + 2)] for the predictor and for the corrector
        (k < order - 1), of the corrector's model_t)."""
        ns = self.ns
        t_prev_0 = t_prev_list[-1]
        lambda_prev_0, lambda_t = float(ns.marginal_lambda(t_prev_0)), float(ns.marginal_lambda(t))
        sigma_prev_0, sigma_t = float(ns.marginal_std(t_prev_0)), float(ns.marginal_std(t))
        alpha_t = float(ns.marginal_alpha(t))
        h = lambda_t - lambda_prev_0
        rks = [(float(ns.marginal_lambda(t_prev_list[-(i + 1)])) - lambda_prev_0) / h for i in range(1, order)] + [1.0]
        hh = -h
        h_phi_1 = math.expm1(hh)
        # the x_t_ part, x * sigma_t / sigma_prev_0 - alpha_t * h_phi_1 * m0, is common to predictor and corrector; D1_k =
        # (m_{-(k+2)} - m0) / rks[k] enter with weights w[k], the corrector's (model_t - m0) with w_t:
        if self.variant == "vary_coeff":
            K = order
            C = np.array([[r ** j / math.factorial(j + 1) for j in range(K)] for r in rks], dtype=np.float64)
            h_phi_ks, h_phi_k, fact = [], h_phi_1, 1
            for k in range(1, K + 2):
                h_phi_ks.append(h_phi_k)
                h_phi_k = h_phi_k / hh - 1 / fact
                fact *= k + 1
            w_p = None
            if K > 1:
                A_p = np.linalg.inv(C[:-1, :-1])
                w_p = [-alpha_t * sum(h_phi_ks[k + 1] * A_p[k][j] for k in range(K - 1)) for j in range(K - 1)]
            w_c = w_t = None
            if use_corrector:
                A_c = np.linalg.inv(C)
                w_c = [-alpha_t * sum(h_phi_ks[k + 1] * A_c[k][j] for k in range(K - 1)) for j in range(K - 1)]
                w_t = -alpha_t * h_phi_ks[K] * A_c[max(K - 2, 0)][-1]   # the reference's row: the loop's last k (0 if none)
        else:
            B_h = hh if self.variant == "bh1" else math.expm1(hh)
            R = np.array([[r ** (i - 1) for r in rks] for i in range(1, order + 1)], dtype=np.float64)
            b, h_phi_k, fact = [], h_phi_1 / hh - 1, 1
            for i in range(1, order + 1):
                b.append(h_phi_k * fact / B_h)
                fact *= i + 1
                h_phi_k = h_phi_k / hh - 1 / fact
            b = np.array(b, dtype=np.float64)
            w_p = None
            if order > 1:
                rhos_p = np.array([0.5]) if order == 2 else np.linalg.solve(R[:-1, :-1], b[:-1])
                w_p = [-alpha_t * B_h * r for r in rhos_p]
            w_c = w_t = None
            if use_corrector:
                rhos_c = np.array([0.5]) if order == 1 else np.linalg.solve(R, b)
                w_c = [-alpha_t * B_h * r for r in rhos_c[:-1]]
                w_t = -alpha_t * B_h * rhos_c[-1]
        c_x, c_m0 = sigma_t / sigma_prev_0, -alpha_t * h_phi_1
        return c_x, c_m0, rks, w_p, w_c, w_t

    def update(self, x, model_prev_list, t_prev_list, t, order, use_corrector=True):
        """one multistep predictor (+ corrector) step to time t -> (x_t, model_t or None)."""
        lib, n = self.lib, x.numel()
        c_x, c_m0, rks, w_p, w_c, w_t = self._coefficients(t_prev_list, t, order, use_corrector)
        m0 = model_prev_list[-1]

        def d_terms(w):  # sum_k w[k] * (m_{-(k+2)} - m0) / rks[k]
            terms = [(model_prev_list[-(k + 2)], w[k] / rks[k]) for k in range(len(w))]
            return terms, -sum(w[k] / rks[k] for k in range(len(w)))

        extra, c0 = d_terms(w_p) if w_p is not None else ([], 0.0)
        x_t = _lincomb(lib, torch.empty_like(x), [(x, c_x), (m0, c_m0 + c0)] + extra, n)
        model_t = None
        if use_corrector:
            model_t = self.model_fn(x_t, t)
            extra, c0 = d_terms(w_c) if order > 1 else ([], 0.0)
            x_t = _lincomb(lib, x_t, [(x, c_x), (m0, c_m0 + c0 - w_t), (model_t, w_t)] + extra, n)
        return x_t, model_t

    def after_update(self, x, model_x):
        if self.callback is not None:
            self.callback({"x": x, "i": self.index, "sigma": 0, "sigma_hat": 0, "denoised": model_x})
        self.index += 1

    def sample(self, x, steps=20, t_start=None, t_end=None, order=3, skip_type="time_uniform", lower_order_final=True):
        t_0 = 1.0 / self.ns.total_N if t_end is None else t_end
        t_T = self.ns.T if t_start is None else t_start
        if steps < order:
            raise L.SdxeError(f"UniPC order must be < sampling steps (order {order}, {steps} steps)")
        x = x.float().contiguous().clone()
        timesteps = [float(v) for v in get_time_steps(self.ns, skip_type, t_T, t_0, steps)]
        model_prev_list = [self.model_fn(x, timesteps[0])]
        t_prev_list = [timesteps[0]]
        for init_order in range(1, order):   # the first `order` values come from lower-order steps
            t = timesteps[init_order]
            x, model_x = self.update(x, model_prev_list, t_prev_list, t, init_order, use_corrector=True)
            self.after_update(x, model_x)
            model_prev_list.append(model_x)
            t_prev_list.append(t)
        for step in range(order, steps + 1):
            t = timesteps[step]
            step_order = min(order, steps + 1 - step) if lower_order_final else order
            x, model_x = self.update(x, model_prev_list, t_prev_list, t, step_order, use_corrector=step != steps)
            self.after_update(x, model_x)
            model_prev_list = model_prev_list[1:] + model_prev_list[-1:]
            t_prev_list = t_prev_list[1:] + [t]
            if step < steps:   # no model call for the final value
                model_prev_list[-1] = model_x
        return x


@torch.no_grad()
def unipc(model, x, timesteps, extra_args=None, callback=None, disable=None, is_img2img=False, variant="bh1",
          skip_type="time_uniform", order=3, lower_order_final=True):
    """UniPC over len(timesteps) steps of the discrete schedule; img2img starts at timesteps[-1] / 1000 + 1 / 1000."""
    ns = NoiseScheduleVP("discrete", alphas_cumprod=model.inner_model.inner_model.alphas_cumprod)
    t_start = float(timesteps[-1]) / 1000 + 1 / 1000 if is_img2img else None
    sampler = UniPCSampler(model, {} if extra_args is None else extra_args, callback, ns, variant=variant)
    return sampler.sample(x, steps=len(timesteps), t_start=t_start, skip_type=skip_type, order=order,
                          lower_order_final=lower_order_final)


# label, function, aliases, options — modules/sd_samplers_timesteps.py:11-16
samplers_timesteps = [
    ("DDIM", ddim, ["ddim"], {}),
    ("DDIM CFG++", ddim_cfgpp, ["ddim_cfgpp"], {}),
    ("PLMS", plms, ["plms"], {}),
    ("UniPC", unipc, ["unipc"], {}),
]
_timestep_map = {name.lower(): (label, fn, opts) for label, fn, aliases, opts in samplers_timesteps for name in [label] + aliases}


class CompVisSampler(S.Sampler):
    """modules/sd_samplers_timesteps.py:75-163: a timestep grid instead of a sigma schedule, eta from opts.eta_ddim."""

    eta_default = 0.0

    def __init__(self, funcname_or_label, sd_model, options=None):
        key = funcname_or_label.lower() if isinstance(funcname_or_label, str) else None
        if key not in _timestep_map:
            raise L.SdxeError(f"timestep sampler {funcname_or_label!r} is unknown (available: "
                              + ", ".join(x[0] for x in samplers_timesteps) + ")")
        self.label, self.func, self.options = _timestep_map[key]
        if options:
            self.options = {**self.options, **options}
        self.sd_model = sd_model
        self.sched_opts = S.SchedulerOptions()
        self.unipc_opts = UniPCOptions()
        self.model_wrap_cfg = CFGDenoiserTimesteps(self)
        self.model_wrap = self.model_wrap_cfg.inner_model
        self.last_latent = None
        self.eta = 0.0
        self.s_min_uncond = 0.0
        self.p = None
        self.sampler_extra_args = None

    def get_timesteps(self, p, steps: int) -> torch.Tensor:
        """int64 [steps]: 1, 1 + 1000 // steps, ... clipped to 999 (one more step with discard_next_to_last_sigma)."""
        discard = bool(self.options.get("discard_next_to_last_sigma", False)) or self.sched_opts.always_discard_next_to_last_sigma
        steps += 1 if discard else 0
        return torch.clip(torch.arange(0, 1000, 1000 // steps) + 1, 0, 999)

    def initialize(self, p) -> dict:
        kw = super().initialize(p)
        if self.func is unipc:
            o = self.unipc_opts
            kw.update(variant=o.uni_pc_variant, skip_type=o.uni_pc_skip_type, order=o.uni_pc_order,
                      lower_order_final=o.uni_pc_lower_order_final)
        return kw

    def _extra_args(self, p, conditioning, unconditional_conditioning, image_conditioning):
        return {"cond": conditioning, "image_cond": image_conditioning, "uncond": unconditional_conditioning,
                "cond_scale": p.cfg_scale, "s_min_uncond": self.s_min_uncond}

    def sample_img2img(self, p, x, noise, conditioning, unconditional_conditioning, steps=None, image_conditioning=None):
        steps, t_enc = S.setup_img2img_steps(p, steps)
        timesteps = self.get_timesteps(p, steps)
        a = self.sd_model.alphas_cumprod[int(timesteps[t_enc])]
        xi = x * torch.sqrt(a) + noise * torch.sqrt(1 - a)
        extra = self.initialize(p)
        params = inspect.signature(self.func).parameters
        extra["timesteps"] = timesteps[:t_enc]
        if "is_img2img" in params:
            extra["is_img2img"] = True
        self.model_wrap_cfg.init_latent = x
        self.last_latent = x
        self.sampler_extra_args = self._extra_args(p, conditioning, unconditional_conditioning, image_conditioning)
        return self.launch_sampling(t_enc + 1, lambda: self.func(self.model_wrap_cfg, xi, extra_args=self.sampler_extra_args,
                                                                 disable=False, callback=self.callback_state, **extra))

    def sample(self, p, x, conditioning, unconditional_conditioning, steps=None, image_conditioning=None):
        steps = steps or p.steps
        timesteps = self.get_timesteps(p, steps)
        extra = self.initialize(p)
        extra["timesteps"] = timesteps
        self.last_latent = x
        self.sampler_extra_args = self._extra_args(p, conditioning, unconditional_conditioning, image_conditioning)
        return self.launch_sampling(steps, lambda: self.func(self.model_wrap_cfg, x, extra_args=self.sampler_extra_args,
                                                             disable=False, callback=self.callback_state, **extra))
