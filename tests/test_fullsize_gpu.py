"""Full-size parity on the configurations bench.py measures, in the dtypes it measures (BASELINE.json configs[1..3]):

  C2  SD1.5 512x512, 20 Euler-a steps, batch 8 — bf16 (the headline dtype) AND fp16 (the reference's own arithmetic)
  C3  SDXL-base 1024x1024: UNet forward at 128x128 latent, CFG batch 2B = 8; 30 DPM++ 2M Karras steps end to end
  VAE decode at 1024x1024 (attention N = 16384, d = 512)
  C4  SD1.5 512 -> 1024 hires fix, 20 + 20 Euler-a steps

Ground truth = the fp32 oracle on the same box (TF32 disabled, tests/conftest.py). Beside every engine error the test
prints the error of the reference's own GPU path restated in torch (fp16 autocast + SDPA, "ref16") and, for bf16, of the
same torch path under bf16 autocast ("refbf16" — the reference has no bf16 UNet mode, modules/shared_init.py:30-32, so
this is what its code would produce if it had).

STATED TOLERANCES (final latent, relative L2 vs the fp32 oracle; decoded pixels, PSNR on truncated uint8):
  fp16 engine : rel-L2 <= max(3 x ref16, 5e-3),  PSNR >= 35 dB
  bf16 engine : rel-L2 <= max(1.5 x refbf16, 4e-2), PSNR >= 28 dB   (bf16 has 3 fewer mantissa bits: 8x the fp16 ulp)
  single UNet forward / VAE decode: fp16 <= max(3 x ref16, 2e-3); bf16 <= max(1.5 x refbf16, 1.6e-2)
"""
import copy
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _mem(tag):
    free, total = torch.cuda.mem_get_info()
    print(f"  [mem {tag}] device free {free / 2**30:.1f} / {total / 2**30:.1f} GiB, torch allocated {torch.cuda.memory_allocated() / 2**30:.1f} "
          f"reserved {torch.cuda.memory_reserved() / 2**30:.1f} GiB")


def _state_dicts(cuda, config, seed_u, seed_v):
    """Seeded synthetic fp32 weights (sdwebui_b200.checkpoint), generated on the GPU."""
    from sdwebui_b200 import checkpoint as C
    from sdwebui_b200.engine import UNetSpec, VAESpec

    spec = UNetSpec.sd15() if config == "sd15" else UNetSpec.sdxl()
    usd = C.synthetic_state_dict(C.unet_param_shapes(spec), seed=seed_u, device=cuda, dtype=torch.float32)
    vsd = C.synthetic_state_dict(C.vae_decoder_param_shapes(VAESpec()), seed=seed_v, device=cuda, dtype=torch.float32)
    return spec, usd, vsd


def _oracle_from(cuda, config, usd, vsd):
    from oracle.unet import UNetModel, sd15_config, sdxl_config
    from oracle.vae import AutoencoderKLDecode, VAEConfig

    with torch.device(cuda):
        unet = UNetModel(sd15_config() if config == "sd15" else sdxl_config()).eval()
        vae = AutoencoderKLDecode(VAEConfig()).eval()
    unet.load_state_dict(usd)
    vae.load_state_dict(vsd)
    return unet, vae


def _oracle_models(cuda, config, seed_u, seed_v):
    spec, usd, vsd = _state_dicts(cuda, config, seed_u, seed_v)
    unet, vae = _oracle_from(cuda, config, usd, vsd)
    return spec, unet, vae, usd, vsd


def _engine_model(cuda, spec, usd, vsd, dtype, is_sdxl):
    from sdwebui_b200.engine import VAEDecoderEngine, VAESpec
    from sdwebui_b200.processing import SdModel
    from sdwebui_b200.sd_unet import SdxeUnet

    su = SdxeUnet(dict(usd), spec, dtype=dtype, device=cuda)
    su.activate()
    ve = VAEDecoderEngine(VAESpec(), dtype=dtype, device=cuda)
    ve.load_state_dict(vsd)
    ve.finalize()
    return SdModel(su, ve, is_sdxl=is_sdxl, dtype_unet=dtype, device=cuda)


def _torch16(unet, vae, cuda, dtype):
    from oracle.pipeline import OraclePipeline

    u, v = copy.deepcopy(unet).to(dtype), copy.deepcopy(vae).to(dtype)
    return OraclePipeline(u, v, cuda, dtype_unet=dtype, dtype_vae=dtype, autocast=True)


def _report(tag, lat, img, lat32, img32):
    from oracle.pipeline import psnr_uint8

    e = rel_err(lat, lat32)
    mx = (lat.float() - lat32).abs().max().item()
    rms = ((lat.float() - lat32).pow(2).mean().sqrt() / lat32.pow(2).mean().sqrt()).item()
    ps = psnr_uint8(img, img32)
    print(f"  {tag:14s} latent rel-L2 {e:.3e}  max-abs {mx:.3e}  rel-RMS {rms:.3e}  PSNR {ps:.1f} dB")
    return e, ps


def _txt2img_case(cuda, config, sp, B, dtypes, ctx_dim, adm, scale_factor):
    """The engines run FIRST: they take their memory from cudaMalloc, and after a full-size fp32 oracle run the PyTorch
    caching allocator keeps > 150 GB reserved (fragmented segments that empty_cache() cannot return)."""
    from oracle.pipeline import OraclePipeline
    from oracle.synth import synthetic_context, synthetic_vector
    from sdwebui_b200.processing import StableDiffusionProcessingTxt2Img, process_images

    spec, usd, vsd = _state_dicts(cuda, config, 21, 22)
    cond = synthetic_context(B, 77, ctx_dim, 3, cuda)
    uncond = synthetic_context(B, 77, ctx_dim, 4, cuda)
    yc = synthetic_vector(B, adm, 5, cuda) if adm else None
    yu = synthetic_vector(B, adm, 6, cuda) if adm else None
    eng_out = {}
    for dt in dtypes:
        model = _engine_model(cuda, spec, usd, vsd, dt, is_sdxl=bool(adm))
        c = {"crossattn": cond, "vector": yc} if adm else cond
        u = {"crossattn": uncond, "vector": yu} if adm else uncond
        p = StableDiffusionProcessingTxt2Img(sd_model=model, c=c, uc=u, seeds=list(sp.seeds), sampler_name=sp.sampler, steps=sp.steps,
                                             cfg_scale=sp.cfg_scale, width=sp.width, height=sp.height, randn_source=sp.randn_source,
                                             enable_hr=sp.enable_hr, hr_scale=sp.hr_scale, hr_second_pass_steps=sp.hr_second_pass_steps,
                                             denoising_strength=sp.denoising_strength)
        model.scale_factor = scale_factor
        out = process_images(p)
        eng_out[dt] = (out.latents.float().cpu(), out.images.permute(0, 3, 1, 2).float() / 255.0)
        model.unet.deactivate()
        model.vae.close()
        del model, out
        _free()
    unet, vae = _oracle_from(cuda, config, usd, vsd)
    del usd, vsd
    _free()
    lat32, img32 = OraclePipeline(unet, vae, cuda, dtype_unet=torch.float32).txt2img(sp, cond, uncond, yc, yu)
    lat32, img32 = lat32.cpu(), img32.cpu()
    res = {}
    for dt in dtypes:
        p16 = _torch16(unet, vae, cuda, dt)
        lat_r, img_r = p16.txt2img(sp, cond, uncond, yc, yu)
        res[("ref", dt)] = _report(f"torch {str(dt)[6:]}", lat_r.cpu(), img_r.cpu(), lat32, img32)
        del p16
        _free()
    del unet, vae
    _free()
    for dt in dtypes:
        res[("eng", dt)] = _report(f"sdxe {str(dt)[6:]}", eng_out[dt][0], eng_out[dt][1], lat32, img32)
    for dt in dtypes:
        e, ps = res[("eng", dt)]
        e_ref, _ = res[("ref", dt)]
        if dt == torch.float16:
            assert e < max(3 * e_ref, 5e-3) and ps > 35.0, (dt, e, e_ref, ps)
        else:
            assert e < max(1.5 * e_ref, 4e-2) and ps > 28.0, (dt, e, e_ref, ps)
    return res


def test_c2_sd15_b8_bf16_and_fp16(cuda):
    """BASELINE configs[1] exactly as benched: SD1.5 512x512, 20 Euler-a steps, batch 8, CFG 7; bf16 and fp16 engines."""
    from oracle.pipeline import SamplingParams

    print("\nC2 SD1.5 512x512 20 Euler-a steps B=8 (vs fp32 oracle):")
    sp = SamplingParams(sampler="Euler a", steps=20, width=512, height=512, seeds=tuple(range(1000, 1008)), randn_source="NV")
    _txt2img_case(cuda, "sd15", sp, 8, [torch.bfloat16, torch.float16], 768, 0, 0.18215)


def test_c3_sdxl_dpmpp2m_30_steps(cuda):
    """BASELINE configs[2] at B=2 (the fp32 oracle needs ~0.8 PFLOP at B=2 already): SDXL-base 1024x1024, 30 DPM++ 2M
    Karras steps, CFG 7, incl. the VAE decode at 1024x1024."""
    from oracle.pipeline import SamplingParams

    print("\nC3 SDXL 1024x1024 30 DPM++ 2M Karras steps B=2 (vs fp32 oracle):")
    sp = SamplingParams(sampler="DPM++ 2M", steps=30, width=1024, height=1024, seeds=(1000, 1001), randn_source="NV", scale_factor=0.13025)
    _txt2img_case(cuda, "sdxl", sp, 2, [torch.float16, torch.bfloat16], 2048, 2816, 0.13025)


def test_c4_sd15_hires_512_to_1024(cuda):
    """BASELINE configs[3] at B=2: SD1.5 512x512 20 steps + latent hires fix to 1024x1024, 20 more steps (Euler a)."""
    from oracle.pipeline import SamplingParams

    print("\nC4 SD1.5 512->1024 hires 20+20 Euler-a steps B=2 (vs fp32 oracle):")
    sp = SamplingParams(sampler="Euler a", steps=20, width=512, height=512, seeds=(1000, 1001), randn_source="NV", enable_hr=True,
                        hr_scale=2.0, hr_second_pass_steps=20, denoising_strength=0.7)
    _txt2img_case(cuda, "sd15", sp, 2, [torch.float16], 768, 0, 0.18215)


@pytest.mark.parametrize("config,n,h,w", [("sd15", 16, 64, 64), ("sdxl", 8, 128, 128), ("sdxl", 4, 104, 152), ("sd15", 8, 64, 96)])
def test_unet_forward_bench_shape(cuda, config, n, h, w):
    """One UNet forward at the CFG batch the bench runs: SD1.5 2B = 16 @ 64x64, SDXL 2B = 8 @ 128x128; and at sizes
    whose convolutions all go through im2col: SDXL's 1216x832 bucket (latent 104x152, ragged GEMM tiles, self-attention
    over 3952 and 988 tokens) and SD1.5 at 768x512 (latent 64x96). fp16 and bf16."""
    spec, unet, vae, usd, vsd = _oracle_models(cuda, config, 3, 4)
    from sdwebui_b200.engine import UNetEngine

    del vae, vsd
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn(n, 4, h, w, device=cuda, generator=g)
    t = torch.linspace(950.0, 20.5, n, device=cuda)
    ctx = torch.randn(n, 77, spec.context_dim, device=cuda, generator=g)
    y = torch.randn(n, spec.adm_in_channels, device=cuda, generator=g) if spec.adm_in_channels else None
    print(f"\n{config} UNet forward n={n} @ {h}x{w}:")
    refs, ref32 = {}, {}
    for dt in (torch.float16, torch.bfloat16):
        xq, tq, cq, yq = x.to(dt), t.to(dt), ctx.to(dt), (y.to(dt) if y is not None else None)
        outs = []
        with torch.no_grad():
            for a in range(0, n, 4):  # fp32 oracle in slices of 4 samples (activation memory)
                outs.append(unet(xq[a:a + 4].float(), tq[a:a + 4].float(), context=cq[a:a + 4].float(), y=None if yq is None else yq[a:a + 4].float()))
        ref32[dt] = torch.cat(outs)
        m16 = copy.deepcopy(unet).to(dt)
        with torch.no_grad(), torch.autocast("cuda", dtype=dt):
            refs[dt] = rel_err(torch.cat([m16(xq[a:a + 4], tq[a:a + 4], context=cq[a:a + 4], y=None if yq is None else yq[a:a + 4]) for a in range(0, n, 4)]), ref32[dt])
        del m16
        _free()
    del unet
    _free()
    for dt in (torch.float16, torch.bfloat16):
        eng = UNetEngine(spec, dtype=dt, device=cuda)
        eng.load_state_dict(usd)
        eng.finalize()
        out = eng.forward(x.to(dt), t.to(dt), ctx.to(dt), y.to(dt) if y is not None else None)
        e = rel_err(out, ref32[dt])
        print(f"  {str(dt)[6:]:9s} engine {e:.3e}   torch autocast {refs[dt]:.3e}")
        assert e < (max(3 * refs[dt], 2e-3) if dt == torch.float16 else max(1.5 * refs[dt], 1.6e-2))
        eng.close()
        del eng
        _free()


def _vae_decode_case(cuda, n, h, w, seed_w, seed_z):
    from oracle.vae import AutoencoderKLDecode, VAEConfig
    from sdwebui_b200 import checkpoint as C
    from sdwebui_b200.engine import VAEDecoderEngine, VAESpec

    vsd = C.synthetic_state_dict(C.vae_decoder_param_shapes(VAESpec()), seed=seed_w, device=cuda, dtype=torch.float32)
    with torch.device(cuda):
        vae = AutoencoderKLDecode(VAEConfig()).eval()
    vae.load_state_dict(vsd)
    g = torch.Generator(device="cuda").manual_seed(seed_z)
    z = torch.randn(n, 4, h, w, device=cuda, generator=g)
    print(f"\nVAE decode {n} x {h}x{w} -> {8 * h}x{8 * w}:")
    for dt in (torch.float16, torch.bfloat16):
        zq = z.to(dt)
        with torch.no_grad():
            ref32 = torch.cat([vae.decode(zq[i:i + 1].float()) for i in range(n)])
            v16 = copy.deepcopy(vae).to(dt)
            ref16 = torch.cat([v16.decode(zq[i:i + 1]) for i in range(n)])
        del v16
        eng = VAEDecoderEngine(VAESpec(), dtype=dt, device=cuda)
        eng.load_state_dict(vsd)
        eng.finalize()
        out = eng.decode(zq)
        e, e_ref = rel_err(out, ref32), rel_err(ref16, ref32)
        print(f"  {str(dt)[6:]:9s} engine {e:.3e}   torch {str(dt)[6:]} {e_ref:.3e}   max-abs {(out.float() - ref32).abs().max().item():.3e}")
        assert e < (max(3 * e_ref, 2e-3) if dt == torch.float16 else max(1.5 * e_ref, 1.6e-2))
        eng.close()
        del eng, ref32, ref16
        _free()


def test_vae_decode_1024(cuda):
    """KL-f8 decoder at 128x128 latent -> 1024x1024, B=2: mid-block attention over 16384 tokens at d = 512, convs with
    up to 2M output rows per image."""
    _vae_decode_case(cuda, 2, 128, 128, 8, 5)


def test_vae_decode_832x1216(cuda):
    """KL-f8 decoder at SDXL's 1216x832 bucket (latent 104x152), B=1: every conv through im2col, mid-block attention
    over 15808 tokens (a ragged last KV block) at d = 512."""
    _vae_decode_case(cuda, 1, 104, 152, 8, 6)
