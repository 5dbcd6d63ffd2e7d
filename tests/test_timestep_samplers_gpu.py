"""DDIM, DDIM CFG++, PLMS, UniPC and LCM on the engine:
  (a) sdxe_cfg_combine_affine against its torch formula and against sdxe_cfg_combine_multi;
  (b) each sampler loop on a toy eps model against the REFERENCE's own output (tests/golden/timesteps_ref.npz);
  (c) process_images with the tiny UNet against the fp32 torch pipeline (tests/timestep_oracle.py): txt2img for all five,
      masked img2img (DDIM, UniPC), an AND-composed prompt with s_min_uncond (DDIM), a hires pass (UniPC), and the
      pred_x0 an interrupted DDIM job returns;
  (d) SD1.5 512x512 batch 8 fp16 for UniPC 10 and LCM 4 under DESIGN section 4's end-to-end rule."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from timestep_toys import (LATENT, LCM_STEPS, STEPS, UNIPC_ORDERS, UNIPC_SKIPS, UNIPC_VARIANTS, CountingNoise,  # noqa: E402
                           ToyTimestepModel, img2img_t_enc, lcm_toy_apply_model, x_init)


def rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


# ---------------------------------------------------------------------------------------------------------------- (a)
def _affine_ref(x, eps, conds_list, urows, cx, ce, x0_coef):
    B = x.shape[0]
    e = eps.float()
    out, x0, unc = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    for b in range(B):
        eu = e[urows[b]]
        acc = eu.clone()
        for r, w in conds_list[b]:
            acc += (e[r] - eu) * w
        out[b] = cx[b] * x[b] + ce[b] * acc
        x0[b] = x0_coef[2 * b] * x[b] + x0_coef[2 * b + 1] * e[conds_list[b][0][0]]
        unc[b] = eu
    return out, x0, unc


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("skip_uncond", [False, True])
def test_cfg_combine_affine(cuda, dtype, skip_uncond):
    from sdwebui_b200 import lib as L

    lib = L.load()
    B, elems = 3, 4 * 16 * 16
    conds_list = [[(0, 0.7), (1, 0.5)], [(2, 1.0)], [(3, 0.4), (4, -0.3), (5, 0.9)]]   # AND-composed, weighted
    n_cond = 6
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(B, 4, 16, 16, device=cuda, generator=g)
    eps = torch.randn(n_cond + (0 if skip_uncond else B), 4, 16, 16, device=cuda, generator=g).to(dtype)
    urows = [c[0][0] for c in conds_list] if skip_uncond else [n_cond + b for b in range(B)]
    ptr = torch.tensor([0, 2, 3, 6], device=cuda, dtype=torch.int32)
    rows = torch.tensor([r for c in conds_list for r, _ in c], device=cuda, dtype=torch.int32)
    w = torch.tensor([w for c in conds_list for _, w in c], device=cuda, dtype=torch.float32)
    ur = torch.tensor(urows, device=cuda, dtype=torch.int32)
    cx = torch.rand(B, device=cuda, generator=g)
    ce = torch.randn(B, device=cuda, generator=g)
    x0c = torch.randn(2 * B, device=cuda, generator=g)
    out, x0, unc = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    L.check(lib.sdxe_cfg_combine_affine(L.ptr(x), L.ptr(eps), L.ptr(ptr), L.ptr(rows), L.ptr(w), L.ptr(ur), L.ptr(cx), L.ptr(ce),
                                        L.ptr(out), L.ptr(x0c), L.ptr(x0), L.ptr(unc), B, elems, L.torch_dtype_code(dtype),
                                        L.current_stream()))
    r_out, r_x0, r_unc = _affine_ref(x, eps, conds_list, urows, cx.tolist(), ce.tolist(), x0c.tolist())
    assert rel(out, r_out) < 1e-6 and rel(x0, r_x0) < 1e-6 and torch.equal(unc, r_unc)
    # the optional outputs may be absent
    out2 = torch.empty_like(x)
    L.check(lib.sdxe_cfg_combine_affine(L.ptr(x), L.ptr(eps), L.ptr(ptr), L.ptr(rows), L.ptr(w), L.ptr(ur), L.ptr(cx), L.ptr(ce),
                                        L.ptr(out2), None, None, None, B, elems, L.torch_dtype_code(dtype), L.current_stream()))
    assert torch.equal(out, out2)
    # cx = 1, ce = -sigma is the k-diffusion combine
    sigma = torch.rand(B, device=cuda, generator=g) * 10 + 0.1
    multi = torch.empty_like(x)
    L.check(lib.sdxe_cfg_combine_multi(L.ptr(x), L.ptr(eps), L.ptr(sigma), L.ptr(ptr), L.ptr(rows), L.ptr(w), L.ptr(ur), L.ptr(multi),
                                       B, elems, L.torch_dtype_code(dtype), L.current_stream()))
    ones, neg = torch.ones(B, device=cuda), (-sigma).contiguous()
    L.check(lib.sdxe_cfg_combine_affine(L.ptr(x), L.ptr(eps), L.ptr(ptr), L.ptr(rows), L.ptr(w), L.ptr(ur), L.ptr(ones), L.ptr(neg),
                                        L.ptr(out2), None, None, None, B, elems, L.torch_dtype_code(dtype), L.current_stream()))
    err = rel(out2, multi)
    print(f"affine vs multi ({dtype}, skip={skip_uncond}): {err:.2e}")
    assert err < 1e-6


# ---------------------------------------------------------------------------------------------------------------- (b)
def _golden():
    return np.load(os.path.join(HERE, "golden", "timesteps_ref.npz"))


def _ac(cuda):
    from sdwebui_b200.samplers import make_alphas_cumprod

    return make_alphas_cumprod().to(cuda)


def _ts(steps, img2img):
    ts = torch.clip(torch.arange(0, 1000, 1000 // steps) + 1, 0, 999)
    return ts[:img2img_t_enc(steps)] if img2img else ts


@pytest.mark.parametrize("family", ["ddim", "ddim_eta07", "ddim_cfgpp", "plms"])
def test_ddim_plms_match_reference(cuda, family):
    from sdwebui_b200 import sd_samplers_timesteps as T

    g = _golden()
    for steps in STEPS:
        for i2i in (False, True):
            name = f"{family}_{steps}{'_i2i' if i2i else ''}"
            toy = ToyTimestepModel(_ac(cuda))
            x = x_init(2, steps, i2i).to(cuda)
            noise = CountingNoise((2,) + LATENT, 500 + steps, cuda)
            if family == "plms":
                got = T.plms(toy, x, _ts(steps, i2i))
            else:
                fn = T.ddim_cfgpp if family == "ddim_cfgpp" else T.ddim
                got = fn(toy, x, _ts(steps, i2i), eta=0.7 if family == "ddim_eta07" else 0.0, noise_sampler=noise)
            err = rel(got.cpu(), torch.from_numpy(g[name]))
            print(f"{name}: {len(toy.calls)} model calls, rel err vs reference {err:.2e}")
            assert np.allclose(toy.calls, g[name + "_calls"])
            assert err < 5e-6


@pytest.mark.parametrize("variant", UNIPC_VARIANTS)
def test_unipc_matches_reference(cuda, variant):
    from sdwebui_b200 import sd_samplers_timesteps as T

    g = _golden()
    worst = 0.0
    for steps in STEPS:
        for i2i in (False, True):
            for skip in UNIPC_SKIPS:
                for order in UNIPC_ORDERS:
                    for lof in (True, False):
                        name = f"unipc_{variant}_{skip}_o{order}_{'lof' if lof else 'nolof'}_{steps}{'_i2i' if i2i else ''}"
                        toy = ToyTimestepModel(_ac(cuda))
                        x = x_init(1 if variant == "vary_coeff" else 2, steps, i2i).to(cuda)
                        got = T.unipc(toy, x, _ts(steps, i2i), is_img2img=i2i, variant=variant, skip_type=skip, order=order,
                                      lower_order_final=lof)
                        err = rel(got.cpu(), torch.from_numpy(g[name]))
                        worst = max(worst, err)
                        assert np.allclose(toy.calls, g[name + "_calls"], rtol=1e-5), name
                        # order 3 without lower_order_final ends on steps whose coefficients amplify the reference's own
                        # fp32 rounding (its solver runs in fp32, these coefficients in fp64): 5.4e-6 at 10 steps
                        assert err < (1e-5 if order == 3 and not lof else 5e-6), (name, err)
    print(f"unipc {variant}: worst rel err vs reference {worst:.2e}")


def test_lcm_matches_reference(cuda):
    import types

    from sdwebui_b200 import sd_samplers_lcm as LC

    g = _golden()
    den = LC.LCMCompVisDenoiser(types.SimpleNamespace(alphas_cumprod=_ac(cuda), device=cuda, apply_model=lcm_toy_apply_model))
    for steps in LCM_STEPS:
        sig = den.get_sigmas(steps)
        x = (x_init(2, steps, False).to(cuda) * sig[0])
        got = LC.sample_lcm(den, x, sig.cpu(), noise_sampler=CountingNoise((2,) + LATENT, 700 + steps, cuda))
        err = rel(got.cpu(), torch.from_numpy(g[f"lcm_{steps}"]))
        print(f"lcm {steps}: rel err vs reference {err:.2e}")
        assert err < 5e-6


# ---------------------------------------------------------------------------------------------------------------- (c)
@pytest.fixture(scope="module")
def tiny(cuda):
    from oracle.synth import init_module_
    from oracle.unet import UNetModel, tiny_config
    from oracle.vae import AutoencoderKLDecode, AutoencoderKLEncode, tiny_vae_config
    from sdwebui_b200.engine import UNetSpec, VAEDecoderEngine, VAEEncoderEngine, VAESpec
    from sdwebui_b200.processing import SdModel
    from sdwebui_b200.sd_unet import SdxeUnet

    ucfg, vcfg = tiny_config(), tiny_vae_config()
    vcfg.ch_mult = [1, 2, 2, 2]  # f = 8 like the real VAE
    unet = init_module_(UNetModel(ucfg), 1).eval().to(cuda)
    dec = init_module_(AutoencoderKLDecode(vcfg), 2).eval().to(cuda)
    enc = init_module_(AutoencoderKLEncode(vcfg), 3).eval().to(cuda)
    su = SdxeUnet(unet.state_dict(), UNetSpec.from_any(ucfg), dtype=torch.float16, device=cuda)
    su.activate()
    vd = VAEDecoderEngine(VAESpec.from_any(vcfg), dtype=torch.float16, device=cuda)
    vd.load_state_dict(dec.state_dict()); vd.finalize()
    ve = VAEEncoderEngine(VAESpec.from_any(vcfg), dtype=torch.float16, device=cuda)
    ve.load_state_dict(enc.state_dict()); ve.finalize()
    model = SdModel(su, vd, is_sdxl=False, dtype_unet=torch.float16, device=cuda, vae_encoder=ve)
    yield ucfg, unet, dec, model
    su.deactivate()
    vd.close()


def _conds(ucfg, B, cuda):
    from oracle.synth import synthetic_context

    return synthetic_context(B, 77, ucfg.context_dim, 3, cuda), synthetic_context(B, 77, ucfg.context_dim, 4, cuda)


@pytest.mark.parametrize("sampler,steps", [("DDIM", 8), ("DDIM CFG++", 8), ("PLMS", 8), ("UniPC", 8), ("LCM", 4)])
def test_tiny_txt2img(cuda, tiny, sampler, steps):
    from oracle.pipeline import SamplingParams
    from sdwebui_b200.processing import StableDiffusionProcessingTxt2Img, process_images
    from timestep_oracle import SamplerOraclePipeline

    ucfg, unet, dec, model = tiny
    B, seeds = 2, (1000, 1001)
    cond, uncond = _conds(ucfg, B, cuda)
    sp = SamplingParams(sampler=sampler, steps=steps, width=128, height=128, seeds=seeds, randn_source="NV")
    lat32 = SamplerOraclePipeline(unet, dec, cuda).sample(sp, cond, uncond)
    p = StableDiffusionProcessingTxt2Img(sd_model=model, c=cond, uc=uncond, seeds=list(seeds), sampler_name=sampler, steps=steps,
                                         width=128, height=128, randn_source="NV", do_not_decode=True)
    err = rel(process_images(p).latents, lat32)
    print(f"tiny {sampler} {steps}: latent rel err vs fp32 oracle {err:.3e}")
    assert err < 1.5e-2


def test_tiny_ddim_eta(cuda, tiny):
    """eta > 0: every step draws from p.rng (the webui's randn_like), the oracle draws the same sequence."""
    from oracle.pipeline import SamplingParams
    from sdwebui_b200.processing import StableDiffusionProcessingTxt2Img, process_images
    from timestep_oracle import SamplerOraclePipeline

    ucfg, unet, dec, model = tiny
    cond, uncond = _conds(ucfg, 2, cuda)
    sp = SamplingParams(sampler="DDIM", steps=8, width=128, height=128, seeds=(5, 6), randn_source="NV")
    lat32 = SamplerOraclePipeline(unet, dec, cuda, eta=0.5).sample(sp, cond, uncond)
    p = StableDiffusionProcessingTxt2Img(sd_model=model, c=cond, uc=uncond, seeds=[5, 6], sampler_name="DDIM", steps=8, eta=0.5,
                                         width=128, height=128, randn_source="NV", do_not_decode=True)
    err = rel(process_images(p).latents, lat32)
    print(f"tiny DDIM eta 0.5: latent rel err vs fp32 oracle {err:.3e}")
    assert err < 1.5e-2


@pytest.mark.parametrize("sampler", ["DDIM", "UniPC"])
def test_tiny_masked_img2img(cuda, tiny, sampler):
    from oracle.pipeline import SamplingParams
    from sdwebui_b200.processing import StableDiffusionProcessingImg2Img, process_images
    from timestep_oracle import SamplerOraclePipeline

    ucfg, unet, dec, model = tiny
    B, H, W = 2, 128, 128
    g = torch.Generator(device="cuda").manual_seed(12)
    init = torch.rand(B, 3, H, W, device=cuda, generator=g)
    enoise = torch.randn(B, 4, H // 8, W // 8, device=cuda, generator=g)
    cond, uncond = _conds(ucfg, B, cuda)
    lmask = torch.zeros(1, 1, H // 8, W // 8, device=cuda)
    lmask[..., 4:12, 4:12] = 1.0
    seeds = [2000, 2001]
    p = StableDiffusionProcessingImg2Img(sd_model=model, c=cond, uc=uncond, seeds=seeds, sampler_name=sampler, steps=12, cfg_scale=6.0,
                                         width=W, height=H, randn_source="NV", denoising_strength=0.6, init_images=init,
                                         encode_noise=enoise, latent_mask=lmask, do_not_decode=True)
    res = process_images(p)
    sp = SamplingParams(sampler=sampler, steps=12, cfg_scale=6.0, width=W, height=H, seeds=tuple(seeds), randn_source="NV",
                        denoising_strength=0.6)
    lat32 = SamplerOraclePipeline(unet, dec, cuda).img2img_latent(sp, p.init_latent.float(), cond, uncond, latent_mask=lmask)
    err = rel(res.latents, lat32)
    print(f"tiny masked img2img {sampler}: latent rel err vs fp32 oracle {err:.3e}")
    assert err < 1.5e-2
    keep = (1 - lmask).expand_as(res.latents).bool()
    assert torch.equal(res.latents[keep], p.init_latent.float()[keep])


def test_tiny_and_prompt_s_min_uncond_ddim(cuda, tiny):
    """AND-composed weighted prompt, with s_min_uncond above every timestep: every other step skips the uncond pass."""
    from oracle.pipeline import SamplingParams
    from oracle.synth import synthetic_context
    from sdwebui_b200 import prompt_parser as P
    from sdwebui_b200.processing import StableDiffusionProcessingTxt2Img, process_images
    from timestep_oracle import SamplerOraclePipeline

    ucfg, unet, dec, model = tiny
    steps = 8
    ca, cb, cc = (synthetic_context(1, 77, ucfg.context_dim, s, cuda)[0] for s in (7, 8, 9))
    uncond = synthetic_context(2, 77, ucfg.context_dim, 4, cuda)
    parts = [[(ca, 1.0), (cb, 0.6)], [(cc, 1.0)]]
    multi = P.MulticondLearnedConditioning(shape=(2,), batch=[
        [P.ComposableScheduledPromptConditioning([P.ScheduledPromptConditioning(steps, c)], w) for c, w in img] for img in parts])
    sp = SamplingParams(sampler="DDIM", steps=steps, width=128, height=128, seeds=(3, 4), randn_source="NV")
    lat32 = SamplerOraclePipeline(unet, dec, cuda, s_min_uncond=1000.0).sample(sp, parts, uncond)
    p = StableDiffusionProcessingTxt2Img(sd_model=model, c=multi, uc=uncond, seeds=[3, 4], sampler_name="DDIM", steps=steps,
                                         s_min_uncond=1000.0, width=128, height=128, randn_source="NV", do_not_decode=True)
    err = rel(process_images(p).latents, lat32)
    print(f"tiny DDIM AND prompt + s_min_uncond: latent rel err vs fp32 oracle {err:.3e}")
    assert err < 1.5e-2


def test_tiny_hires_unipc(cuda, tiny):
    from oracle.pipeline import SamplingParams
    from sdwebui_b200.processing import StableDiffusionProcessingTxt2Img, process_images
    from timestep_oracle import SamplerOraclePipeline

    ucfg, unet, dec, model = tiny
    cond, uncond = _conds(ucfg, 2, cuda)
    kw = dict(steps=6, width=64, height=64, randn_source="NV", enable_hr=True, hr_scale=2.0, hr_second_pass_steps=6,
              denoising_strength=0.6)
    sp = SamplingParams(sampler="UniPC", seeds=(11, 12), **kw)
    lat32 = SamplerOraclePipeline(unet, dec, cuda).sample(sp, cond, uncond)
    p = StableDiffusionProcessingTxt2Img(sd_model=model, c=cond, uc=uncond, seeds=[11, 12], sampler_name="UniPC", do_not_decode=True, **kw)
    err = rel(process_images(p).latents, lat32)
    print(f"tiny UniPC hires: latent rel err vs fp32 oracle {err:.3e}")
    assert err < 1.5e-2


def test_interrupted_ddim_returns_pred_x0(cuda, tiny):
    """An interrupted job returns the sampler's last_latent: on the timestep path, pred_x0 of the first cond
    (x - sqrt(1 - a_t) eps_cond) / sqrt(a_t) of the last completed denoiser call."""
    from sdwebui_b200 import samplers as S
    from sdwebui_b200.processing import StableDiffusionProcessingTxt2Img, process_images

    ucfg, unet, dec, model = tiny
    cond, uncond = _conds(ucfg, 2, cuda)
    seen = {}
    p = StableDiffusionProcessingTxt2Img(sd_model=model, c=cond, uc=uncond, seeds=[1, 2], sampler_name="DDIM", steps=10,
                                         width=128, height=128, randn_source="NV", do_not_decode=True)
    orig = S.create_sampler

    def create(name, m):
        smp = orig(name, m)
        cfg = smp.model_wrap_cfg

        def capture(x, sigma_in, c):
            seen["x"], seen["t"] = x.clone(), sigma_in[0].item()

        def eps_cb(eps):
            seen["eps"] = eps[0:2].float().clone()
            if cfg.step == 3:
                S.state.interrupted = True   # the next denoiser call raises InterruptedException

        cfg.on_cfg_denoiser.append(capture)
        cfg.on_cfg_denoised.append(eps_cb)
        return smp

    S.create_sampler = create
    try:
        res = process_images(p)
    finally:
        S.create_sampler = orig
        S.state.interrupted = False
    a = model.alphas_cumprod[int(seen["t"])]
    want = (seen["x"] - (1 - a).sqrt() * seen["eps"]) / a.sqrt()
    err = rel(res.latents, want)
    print(f"interrupted DDIM: last_latent vs pred_x0 {err:.2e}")
    assert err < 1e-5


# ---------------------------------------------------------------------------------------------------------------- (d)
@pytest.mark.parametrize("sampler,steps", [("UniPC", 10), ("LCM", 4)])
def test_sd15_512_b8_fp16(cuda, sampler, steps):
    """SD1.5 512x512, batch 8, CFG 7, fp16 engine vs the fp32 torch pipeline; beside it the same torch pipeline under fp16
    autocast (the reference's GPU arithmetic). Rule (DESIGN section 4): rel-L2 <= max(3 x torch-fp16, 5e-3), PSNR >= 35 dB."""
    import gc

    from oracle.pipeline import SamplingParams, psnr_uint8
    from oracle.synth import synthetic_context
    from sdwebui_b200 import checkpoint as C
    from sdwebui_b200.engine import UNetSpec, VAEDecoderEngine, VAESpec
    from sdwebui_b200.processing import SdModel, StableDiffusionProcessingTxt2Img, process_images
    from sdwebui_b200.sd_unet import SdxeUnet
    from oracle.unet import UNetModel, sd15_config
    from oracle.vae import AutoencoderKLDecode, VAEConfig
    from timestep_oracle import SamplerOraclePipeline

    spec = UNetSpec.sd15()
    usd = C.synthetic_state_dict(C.unet_param_shapes(spec), seed=21, device=cuda, dtype=torch.float32)
    vsd = C.synthetic_state_dict(C.vae_decoder_param_shapes(VAESpec()), seed=22, device=cuda, dtype=torch.float32)
    B, seeds = 8, tuple(range(1000, 1008))
    cond, uncond = synthetic_context(B, 77, 768, 3, cuda), synthetic_context(B, 77, 768, 4, cuda)
    su = SdxeUnet(dict(usd), spec, dtype=torch.float16, device=cuda)
    su.activate()
    ve = VAEDecoderEngine(VAESpec(), dtype=torch.float16, device=cuda)
    ve.load_state_dict(vsd); ve.finalize()
    model = SdModel(su, ve, is_sdxl=False, dtype_unet=torch.float16, device=cuda)
    p = StableDiffusionProcessingTxt2Img(sd_model=model, c=cond, uc=uncond, seeds=list(seeds), sampler_name=sampler, steps=steps,
                                         width=512, height=512, randn_source="NV")
    out = process_images(p)
    lat_e, img_e = out.latents.float().cpu(), out.images.permute(0, 3, 1, 2).float() / 255.0
    su.deactivate(); ve.close()
    del model, out, su, ve
    gc.collect(); torch.cuda.empty_cache()
    with torch.device(cuda):
        unet, vae = UNetModel(sd15_config()).eval(), AutoencoderKLDecode(VAEConfig()).eval()
    unet.load_state_dict(usd); vae.load_state_dict(vsd)
    del usd, vsd
    sp = SamplingParams(sampler=sampler, steps=steps, width=512, height=512, seeds=seeds, randn_source="NV")
    o32 = SamplerOraclePipeline(unet, vae, cuda)
    lat32 = o32.sample(sp, cond, uncond)
    img32 = o32.decode(lat32, 0.18215).cpu()
    lat32 = lat32.cpu()
    o16 = SamplerOraclePipeline(copy.deepcopy(unet).half(), copy.deepcopy(vae).half(), cuda, dtype_unet=torch.float16,
                                dtype_vae=torch.float16, autocast=True)
    lat16 = o16.sample(sp, cond, uncond)
    img16 = o16.decode(lat16, 0.18215).cpu()
    e_eng, e_ref = rel(lat_e, lat32), rel(lat16.cpu(), lat32)
    ps_eng, ps_ref = psnr_uint8(img_e, img32), psnr_uint8(img16, img32)
    print(f"\nSD1.5 512 B=8 {sampler} {steps}: sdxe fp16 rel-L2 {e_eng:.3e} PSNR {ps_eng:.1f} dB | torch fp16 rel-L2 {e_ref:.3e} "
          f"PSNR {ps_ref:.1f} dB")
    assert e_eng < max(3 * e_ref, 5e-3) and ps_eng >= 35.0, (e_eng, e_ref, ps_eng)
