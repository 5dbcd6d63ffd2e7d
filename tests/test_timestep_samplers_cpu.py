"""Host logic of the timestep samplers (DDIM, DDIM CFG++, PLMS, UniPC) and LCM against the reference's own code
(tests/golden/timesteps_ref.npz, written by tests/golden/make_golden_timesteps.py): the timestep tables, the LCM sigma
tables, UniPC's time grids, and the sampler registry."""
import os
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(HERE, "golden", "timesteps_ref.npz"))


class FakeModel:
    alphas_cumprod = None
    device = torch.device("cpu")
    parameterization = "eps"
    is_sdxl = False

    def __init__(self):
        from sdwebui_b200.samplers import make_alphas_cumprod

        self.alphas_cumprod = make_alphas_cumprod()


@pytest.mark.parametrize("discard", [False, True])
def test_get_timesteps_tables(gold, discard):
    from sdwebui_b200 import sd_samplers_timesteps as T

    smp = T.CompVisSampler("DDIM", FakeModel())
    smp.sched_opts.always_discard_next_to_last_sigma = discard
    for n in (1, 2, 3, 4, 5, 7, 10, 13, 20, 25, 30, 33, 50, 64, 100, 150):
        assert np.array_equal(smp.get_timesteps(None, n).numpy(), gold[f"timesteps_{n}{'_discard' if discard else ''}"]), n


def test_lcm_sigma_tables(gold):
    from sdwebui_b200 import sd_samplers_lcm as LC

    den = LC.LCMSampler("LCM", FakeModel()).model_wrap
    assert isinstance(den, LC.LCMCompVisDenoiser)
    assert np.allclose(den.sigmas.numpy(), gold["lcm_sigmas_table"], rtol=1e-6, atol=0)
    assert np.allclose(den.get_sigmas().numpy(), gold["lcm_sigmas_none"], rtol=1e-6, atol=0)
    for n in (1, 2, 3, 4, 5, 6, 8, 10, 20, 50):
        assert np.allclose(den.get_sigmas(n).numpy(), gold[f"lcm_sigmas_{n}"], rtol=1e-6, atol=0), n
    t = den.sigma_to_t(torch.from_numpy(gold["lcm_probe_sigmas"]))
    assert np.array_equal(t.numpy(), gold["lcm_sigma_to_t"])


def test_lcm_sampler_uses_lcm_schedule():
    from sdwebui_b200 import sd_samplers_lcm as LC

    smp = LC.LCMSampler("LCM", FakeModel())
    p = types.SimpleNamespace(scheduler="Automatic")
    sig = smp.get_sigmas(p, 4)
    assert np.allclose(sig.numpy(), smp.model_wrap.get_sigmas(4).numpy())
    assert smp.func is LC.sample_lcm and smp.label == "LCM"


@pytest.mark.parametrize("skip", ["time_uniform", "time_quadratic", "logSNR"])
def test_unipc_time_grids(gold, skip):
    from sdwebui_b200 import sd_samplers_timesteps as T

    ns = T.NoiseScheduleVP("discrete", alphas_cumprod=FakeModel().alphas_cumprod)
    for n in (3, 4, 10, 15, 20, 50):
        for t_T, tag in ((1.0, ""), (0.702, "_i2i")):
            got = T.get_time_steps(ns, skip, t_T, 1.0 / 1000, n)
            assert np.allclose(got, gold[f"unipc_grid_{skip}_{n}{tag}"], rtol=0, atol=1e-6), (n, tag)


def test_create_sampler_classes():
    from sdwebui_b200 import samplers as S
    from sdwebui_b200 import sd_samplers_lcm as LC
    from sdwebui_b200 import sd_samplers_timesteps as T

    m = FakeModel()
    expect = {"DDIM": T.CompVisSampler, "ddim": T.CompVisSampler, "DDIM CFG++": T.CompVisSampler, "ddim_cfgpp": T.CompVisSampler,
              "PLMS": T.CompVisSampler, "plms": T.CompVisSampler, "UniPC": T.CompVisSampler, "unipc": T.CompVisSampler,
              "LCM": LC.LCMSampler, "k_lcm": LC.LCMSampler, "Euler a": S.KDiffusionSampler, "k_euler_a": S.KDiffusionSampler,
              "DPM++ 2M": S.KDiffusionSampler, "Restart": S.KDiffusionSampler}
    funcs = {"DDIM": T.ddim, "DDIM CFG++": T.ddim_cfgpp, "PLMS": T.plms, "UniPC": T.unipc, "LCM": LC.sample_lcm}
    for name, cls in expect.items():
        smp = S.create_sampler(name, m)
        assert type(smp) is cls, name
        label, fn, _ = S.find_sampler_config(name)
        assert smp.label == label and smp.func is fn
        if label in funcs:
            assert fn is funcs[label]
    assert isinstance(S.create_sampler("DDIM", m).model_wrap_cfg, T.CFGDenoiserTimesteps)
    assert isinstance(S.create_sampler("LCM", m).model_wrap_cfg, LC.CFGDenoiserLCM)
    assert S.find_sampler_config("DPM++ SDE") is None
    with pytest.raises(Exception):
        S.create_sampler("DPM++ SDE", m)


def test_kdiffusion_table_unchanged():
    from sdwebui_b200 import samplers as S

    assert "ddim" not in S._sampler_map and "lcm" not in S._sampler_map and "unipc" not in S._sampler_map
    with pytest.raises(Exception):
        S.KDiffusionSampler("DDIM", FakeModel())


def test_eta_defaults():
    """eta: opts.eta_ddim (0) for the timestep samplers, opts.eta_ancestral (1) for k-diffusion, p.eta wins for both."""
    from sdwebui_b200 import samplers as S

    m = FakeModel()
    for name, want in (("DDIM", 0.0), ("Euler a", 1.0)):
        smp = S.create_sampler(name, m)
        kw = smp.initialize(types.SimpleNamespace(eta=None, rng=None))
        assert smp.eta == want and kw["eta"] == want
        smp.initialize(types.SimpleNamespace(eta=0.3, rng=None))
        assert smp.eta == 0.3


def test_unipc_options_reach_the_sampler():
    from sdwebui_b200 import samplers as S

    smp = S.create_sampler("UniPC", FakeModel())
    smp.unipc_opts.uni_pc_order = 2
    smp.unipc_opts.uni_pc_skip_type = "logSNR"
    kw = smp.initialize(types.SimpleNamespace(eta=None, rng=None))
    assert kw == {"variant": "bh1", "skip_type": "logSNR", "order": 2, "lower_order_final": True}


def test_v_prediction_rejected():
    from sdwebui_b200 import samplers as S
    from sdwebui_b200.lib import SdxeError

    m = FakeModel()
    m.parameterization = "v"
    with pytest.raises(SdxeError):
        S.create_sampler("DDIM", m)
