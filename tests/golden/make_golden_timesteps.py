"""Pins sdwebui_b200/sd_samplers_timesteps.py and sd_samplers_lcm.py to the REFERENCE's in-tree code
(modules/sd_samplers_timesteps.py, modules/sd_samplers_timesteps_impl.py, modules/models/diffusion/uni_pc/uni_pc.py,
modules/sd_samplers_lcm.py), executed unmodified from /root/reference with stub `modules.*` packages and a stub
`k_diffusion` (a seeded randn_like sequence, default_noise_sampler, trange, append_zero, append_dims, and
DiscreteEpsDDPMDenoiser assembled from oracle/kdiffusion.py):

    python tests/golden/make_golden_timesteps.py   ->   tests/golden/timesteps_ref.npz

Recorded: CompVisSampler.get_timesteps with and without discard_next_to_last_sigma; the LCM sigma tables and sigma_to_t;
UniPC's time grids; and, on a toy eps model, ddim (eta 0 and 0.7), ddim_cfgpp, plms and unipc (every variant x skip type
x order 1-3 x lower_order_final) for txt2img and img2img at 4, 10 and 20 steps, and sample_lcm at 4 and 8 steps.
The toy model and the draw sequences are restated by tests/test_timestep_samplers_*.py.
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

from timestep_toys import (LATENT, STEPS, LCM_STEPS, UNIPC_ORDERS, UNIPC_SKIPS, UNIPC_VARIANTS, CountingNoise, ToyTimestepModel,  # noqa: E402
                           img2img_t_enc, lcm_toy_apply_model, x_init)


def main():
    import oracle.kdiffusion as OK

    def pkg(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        return m

    noise_holder = types.SimpleNamespace(randn_like=None)

    def default_noise_sampler(x):
        return lambda sigma, sigma_next: noise_holder.randn_like(x)

    def append_zero(x):
        return torch.cat([x, x.new_zeros([1])])

    def append_dims(x, target_dims):
        return x[(...,) + (None,) * (target_dims - x.ndim)]

    class DiscreteEpsDDPMDenoiser(OK.DiscreteSchedule):
        """k_diffusion.external.DiscreteEpsDDPMDenoiser over the oracle's DiscreteSchedule."""

        def __init__(self, model, alphas_cumprod, quantize):
            super().__init__(alphas_cumprod)
            self.inner_model = model
            self.sigma_data = 1.0

        def get_scalings(self, sigma):
            return -sigma, 1 / (sigma ** 2 + self.sigma_data ** 2) ** 0.5

        def get_eps(self, *args, **kwargs):
            return self.inner_model(*args, **kwargs)

        def __call__(self, *args, **kwargs):  # torch.nn.Module.__call__ -> forward
            return self.forward(*args, **kwargs)

    kd_sampling = pkg("k_diffusion.sampling", torch=noise_holder, default_noise_sampler=default_noise_sampler,
                      trange=lambda n, disable=None: range(n), append_zero=append_zero)
    kd_utils = pkg("k_diffusion.utils", append_dims=append_dims)
    kd_external = pkg("k_diffusion.external", DiscreteEpsDDPMDenoiser=DiscreteEpsDDPMDenoiser)
    kd = pkg("k_diffusion", sampling=kd_sampling, utils=kd_utils, external=kd_external)

    opts = types.SimpleNamespace(uni_pc_variant="bh1", uni_pc_skip_type="time_uniform", uni_pc_order=3,
                                 uni_pc_lower_order_final=True, eta_ddim=0.0, always_discard_next_to_last_sigma=False,
                                 img2img_extra_noise=0.0)
    from sdwebui_b200.samplers import make_alphas_cumprod

    sd_model = types.SimpleNamespace(alphas_cumprod=make_alphas_cumprod(), parameterization="eps", device="cpu")
    shared = pkg("modules.shared", opts=opts, sd_model=sd_model)

    class SamplerStub:
        def __init__(self, funcname):
            self.funcname, self.func, self.config = funcname, funcname, None

    class CFGDenoiserStub:
        def __init__(self, sampler):
            self.sampler, self.model_wrap = sampler, None

    common = pkg("modules.sd_samplers_common", Sampler=SamplerStub, SamplerData=lambda *a, **k: a,
                 setup_img2img_steps=None, InterruptedException=Exception)
    cfg_den = pkg("modules.sd_samplers_cfg_denoiser", CFGDenoiser=CFGDenoiserStub)
    kdiff = pkg("modules.sd_samplers_kdiffusion", KDiffusionSampler=SamplerStub)
    callbacks = pkg("modules.script_callbacks", ExtraNoiseParams=None, extra_noise_callback=None)
    devices = pkg("modules.devices", device="cpu")
    torch_utils = pkg("modules.torch_utils", float64=lambda t: torch.float64)
    modules = pkg("modules", shared=shared, sd_samplers_common=common, sd_samplers_cfg_denoiser=cfg_den,
                  sd_samplers_kdiffusion=kdiff, script_callbacks=callbacks, devices=devices, torch_utils=torch_utils)
    models = pkg("modules.models")
    diffusion = pkg("modules.models.diffusion")
    uni_pc_pkg = pkg("modules.models.diffusion.uni_pc")
    stubs = {"k_diffusion": kd, "k_diffusion.sampling": kd_sampling, "k_diffusion.utils": kd_utils,
             "k_diffusion.external": kd_external, "modules": modules, "modules.shared": shared,
             "modules.sd_samplers_common": common, "modules.sd_samplers_cfg_denoiser": cfg_den,
             "modules.sd_samplers_kdiffusion": kdiff, "modules.script_callbacks": callbacks, "modules.devices": devices,
             "modules.torch_utils": torch_utils, "modules.models": models, "modules.models.diffusion": diffusion,
             "modules.models.diffusion.uni_pc": uni_pc_pkg}
    saved = {k: sys.modules.get(k) for k in list(stubs) + ["modules.models.diffusion.uni_pc.uni_pc",
                                                             "modules.sd_samplers_timesteps_impl", "modules.sd_samplers_compvis"]}
    sys.modules.update(stubs)

    def load(name, rel):
        spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
        return mod

    out = {}
    try:
        uni_pc = load("modules.models.diffusion.uni_pc.uni_pc", "modules/models/diffusion/uni_pc/uni_pc.py")
        uni_pc_pkg.uni_pc = uni_pc
        impl = load("modules.sd_samplers_timesteps_impl", "modules/sd_samplers_timesteps_impl.py")
        modules.sd_samplers_timesteps_impl = impl
        ts_mod = load("ref_sd_samplers_timesteps", "modules/sd_samplers_timesteps.py")
        lcm = load("ref_sd_samplers_lcm", "modules/sd_samplers_lcm.py")

        # -- get_timesteps tables ------------------------------------------------------------------------------------
        sampler = ts_mod.CompVisSampler(impl.ddim, sd_model)
        p = types.SimpleNamespace(extra_generation_params={})
        for discard in (False, True):
            opts.always_discard_next_to_last_sigma = discard
            for n in (1, 2, 3, 4, 5, 7, 10, 13, 20, 25, 30, 33, 50, 64, 100, 150):
                out[f"timesteps_{n}{'_discard' if discard else ''}"] = sampler.get_timesteps(p, n).numpy()
        opts.always_discard_next_to_last_sigma = False

        # -- LCM sigma tables --------------------------------------------------------------------------------------
        lcm_den = lcm.LCMCompVisDenoiser(sd_model)
        out["lcm_sigmas_table"] = lcm_den.sigmas.numpy()
        out["lcm_sigmas_none"] = lcm_den.get_sigmas().numpy()
        for n in (1, 2, 3, 4, 5, 6, 8, 10, 20, 50):
            out[f"lcm_sigmas_{n}"] = lcm_den.get_sigmas(n).numpy()
        probe = torch.exp(torch.linspace(-4.0, 3.0, 97))
        out["lcm_probe_sigmas"] = probe.numpy()
        out["lcm_sigma_to_t"] = lcm_den.sigma_to_t(probe).numpy()

        # -- UniPC time grids --------------------------------------------------------------------------------------
        ns = uni_pc.NoiseScheduleVP("discrete", alphas_cumprod=sd_model.alphas_cumprod)
        unipc_obj = uni_pc.UniPC(None, ns)
        for skip in UNIPC_SKIPS:
            for n in (3, 4, 10, 15, 20, 50):
                for t_T, tag in ((ns.T, ""), (0.702, "_i2i")):
                    out[f"unipc_grid_{skip}_{n}{tag}"] = unipc_obj.get_time_steps(skip, t_T, 1.0 / ns.total_N, n, "cpu").numpy()

        # -- the samplers on the toy eps model ----------------------------------------------------------------------
        def run(name, fn, steps, img2img, B, **kw):
            toy = ToyTimestepModel(sd_model.alphas_cumprod)
            timesteps = sampler.get_timesteps(p, steps)
            if img2img:
                timesteps = timesteps[:img2img_t_enc(steps)]
            noise_holder.randn_like = CountingNoise((B,) + LATENT, 500 + steps).randn_like
            x = x_init(B, steps, img2img)
            res = fn(toy, x.clone(), timesteps, extra_args={}, callback=lambda d: None, disable=True, **kw)
            out[name] = res.numpy()
            out[name + "_calls"] = np.array(toy.calls, dtype=np.float64)

        for steps in STEPS:
            for img2img in (False, True):
                tag = f"{steps}{'_i2i' if img2img else ''}"
                run(f"ddim_{tag}", impl.ddim, steps, img2img, 2, eta=0.0)
                run(f"ddim_eta07_{tag}", impl.ddim, steps, img2img, 2, eta=0.7)
                run(f"ddim_cfgpp_{tag}", impl.ddim_cfgpp, steps, img2img, 2, eta=0.0)
                run(f"plms_{tag}", impl.plms, steps, img2img, 2)
                for variant in UNIPC_VARIANTS:
                    for skip in UNIPC_SKIPS:
                        for order in UNIPC_ORDERS:
                            for lof in (True, False):
                                opts.uni_pc_variant, opts.uni_pc_skip_type = variant, skip
                                opts.uni_pc_order, opts.uni_pc_lower_order_final = order, lof
                                # the reference's vary_coeff solver only broadcasts over a batch of one image
                                run(f"unipc_{variant}_{skip}_o{order}_{'lof' if lof else 'nolof'}_{tag}", impl.unipc, steps,
                                    img2img, 1 if variant == "vary_coeff" else 2, is_img2img=img2img)

        # -- sample_lcm through LCMCompVisDenoiser on a toy eps model -------------------------------------------------
        lcm_model = types.SimpleNamespace(apply_model=lcm_toy_apply_model, alphas_cumprod=sd_model.alphas_cumprod, device="cpu")
        den = lcm.LCMCompVisDenoiser(lcm_model)
        for steps in LCM_STEPS:
            sigmas = den.get_sigmas(steps)
            noise_holder.randn_like = CountingNoise((2,) + LATENT, 700 + steps).randn_like
            x = x_init(2, steps, False) * sigmas[0]
            out[f"lcm_{steps}"] = lcm.sample_lcm(den, x.clone(), sigmas, disable=True).numpy()
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    path = os.path.join(HERE, "timesteps_ref.npz")
    np.savez_compressed(path, **out)
    print(path, len(out), "arrays", os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
