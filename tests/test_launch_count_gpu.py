"""sdxe_launch_count (bench's `gpu_launches`) counts every kernel the library runs exactly once: for each C-ABI primitive and
one forward of each model kind, the counter's increase equals the number of kernels torch.profiler recorded on the device.
Inputs are prepared and synchronised first, so that a profiling window holds nothing but the library call. The models run
with engine profiling on, so their plans execute op by op rather than as a CUDA graph replay."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from sdwebui_b200 import lib as L

    return L, L.load()


def _counted_and_ran(call):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    L, lib = _lib()
    torch.cuda.synchronize()
    n0 = lib.sdxe_launch_count()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    counted = lib.sdxe_launch_count() - n0
    kernels = [e.name for e in prof.events()
               if e.device_type == DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset"))]
    return counted, kernels


def _check(call, expect_min=1):
    call()  # first call: module loading, plan build
    counted, kernels = _counted_and_ran(call)
    assert len(kernels) >= expect_min, kernels
    assert counted == len(kernels), (counted, kernels)


def _rand(*shape, dtype=torch.float16, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(dtype)


# ---- C-ABI primitives ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geglu", [False, True], ids=["plain", "geglu"])
def test_gemm(cuda, geglu):
    L, lib = _lib()
    M, N, K = (1000, 328, 200) if not geglu else (256, 640, 320)
    a, w = _rand(M, K), _rand(N, K, scale=K ** -0.5, seed=1)
    bias = _rand(N, dtype=torch.float32, seed=2)
    res = None if geglu else _rand(M, N, seed=3)
    out = torch.empty(M, N // 2 if geglu else N, dtype=torch.float16, device=cuda)
    code = L.torch_dtype_code(torch.float16)
    _check(lambda: L.check(lib.sdxe_gemm(L.ptr(a), L.ptr(w), L.ptr(out), M, N, K, L.ptr(bias), L.ptr(res), int(geglu), code,
                                         L.current_stream()), "sdxe_gemm"),
           expect_min=3 if geglu else 1)  # GEGLU: weight and bias interleave, then the GEMM


def test_conv3x3(cuda):
    L, lib = _lib()
    n, h, w, cin, cout = 2, 16, 16, 64, 128
    x, wp = _rand(n, h, w, cin), _rand(cout, 9 * cin, scale=(9 * cin) ** -0.5, seed=1)
    bias = _rand(cout, dtype=torch.float32, seed=2)
    out = torch.empty(n, h, w, cout, dtype=torch.float16, device=cuda)
    code = L.torch_dtype_code(torch.float16)
    _check(lambda: L.check(lib.sdxe_conv3x3_nhwc(L.ptr(x), L.ptr(wp), L.ptr(out), n, h, w, cin, cout, L.ptr(bias), code,
                                                 L.current_stream()), "sdxe_conv3x3_nhwc"))


@pytest.mark.parametrize("D", [64, 160])  # 160: two passes over the value columns
def test_attention(cuda, D):
    L, lib = _lib()
    B, H, Nq, Nk = 2, 2, 256, 200
    q, k, v = _rand(B, H, Nq, D), _rand(B, H, Nk, D, seed=1), _rand(B, H, Nk, D, seed=2)
    out = torch.empty(B, Nq, H * D, dtype=torch.float16, device=cuda)
    code = L.torch_dtype_code(torch.float16)
    _check(lambda: L.check(lib.sdxe_attention(L.ptr(q), L.ptr(k), L.ptr(v), L.ptr(out), B, H, Nq, Nk, D, D ** -0.5, code,
                                              L.current_stream()), "sdxe_attention"),
           expect_min=2 if D > 128 else 1)


# (n, h*w, C): a strip of h*w*C/32 16-bit values <= 48 KB takes the one-pass kernel, a larger one the streaming kernels
@pytest.mark.parametrize("n,hw,c", [(2, 256, 320), (2, 4096, 640)], ids=["one_pass", "streaming"])
def test_group_norm(cuda, n, hw, c):
    L, lib = _lib()
    x = _rand(n, hw, c)
    gamma, beta = _rand(c, dtype=torch.float32, seed=1), _rand(c, dtype=torch.float32, seed=2)
    out = torch.empty_like(x)
    code = L.torch_dtype_code(torch.float16)
    _check(lambda: L.check(lib.sdxe_group_norm_nhwc(L.ptr(x), L.ptr(gamma), L.ptr(beta), L.ptr(out), n, hw, c, 32, 1e-5, 1,
                                                    code, L.current_stream()), "sdxe_group_norm_nhwc"),
           expect_min=1 if hw * c // 32 * 2 <= 48 * 1024 else 3)


def test_sampler_steps(cuda):
    L, lib = _lib()
    B, elems = 2, 4 * 64 * 64
    x, den, old, noise = (_rand(B, elems, dtype=torch.float32, seed=s) for s in range(4))
    out = torch.empty_like(x)
    s = L.current_stream
    _check(lambda: L.check(lib.sdxe_lincomb(L.ptr(out), L.ptr(x), 0.5, L.ptr(den), 0.25, L.ptr(old), 0.125, L.ptr(noise),
                                            0.0625, x.numel(), s()), "sdxe_lincomb"))
    _check(lambda: L.check(lib.sdxe_euler_ancestral_step(L.ptr(x), L.ptr(den), L.ptr(noise), 2.0, 1.5, 0.5, x.numel(), s()),
                           "sdxe_euler_ancestral_step"))
    _check(lambda: L.check(lib.sdxe_dpmpp_2m_step(L.ptr(x), L.ptr(den), L.ptr(old), 0.9, -0.1, 1.5, -0.5, x.numel(), s()),
                           "sdxe_dpmpp_2m_step"))
    # CFG combine over 2B eps rows: image b has cond row b (weight 7) and uncond row B + b; with pred_x0 and the uncond copy
    eps = _rand(2 * B, elems, seed=5)
    i32 = dict(dtype=torch.int32, device=cuda)
    row_ptr, cond_rows, uncond_rows = torch.arange(B + 1, **i32), torch.arange(B, **i32), torch.arange(B, 2 * B, **i32)
    cond_w = torch.full((B,), 7.0, device=cuda)
    cx, ce, x0_coef = torch.rand(B, device=cuda), torch.rand(B, device=cuda), torch.rand(2 * B, device=cuda)
    x0_out, uncond_out = torch.empty_like(x), torch.empty_like(x)
    code = L.torch_dtype_code(eps.dtype)
    _check(lambda: L.check(lib.sdxe_cfg_combine_affine(L.ptr(x), L.ptr(eps), L.ptr(row_ptr), L.ptr(cond_rows), L.ptr(cond_w),
                                                       L.ptr(uncond_rows), L.ptr(cx), L.ptr(ce), L.ptr(out), L.ptr(x0_coef),
                                                       L.ptr(x0_out), L.ptr(uncond_out), B, elems, code, s()),
                           "sdxe_cfg_combine_affine"))


# ---- model forwards (plans run eagerly under engine profiling) ------------------------------------------------------
def _finalized(eng, sd):
    eng.load_state_dict(sd)
    eng.finalize()
    eng.profile(True)
    return eng


def test_unet_forward(cuda):
    from oracle.unet import tiny_config
    from sdwebui_b200.checkpoint import synthetic_state_dict, unet_param_shapes
    from sdwebui_b200.engine import UNetEngine, UNetSpec

    L, lib = _lib()
    spec = UNetSpec.from_any(tiny_config())
    eng = _finalized(UNetEngine(spec, dtype=torch.float16, device=cuda), synthetic_state_dict(unet_param_shapes(spec), 1))
    n, h, w, T = 2, 24, 40, 77
    x, ctx = _rand(n, 4, h, w), _rand(n, T, tiny_config().context_dim, seed=1)
    t = torch.tensor([500.0, 20.0], device=cuda, dtype=torch.float16)
    out = torch.empty_like(x)
    code = L.torch_dtype_code(torch.float16)
    _check(lambda: L.check(lib.sdxe_unet_forward(eng._h, L.ptr(x), L.ptr(t), L.ptr(ctx), None, L.ptr(out), n, h, w, T, code,
                                                 L.current_stream()), "sdxe_unet_forward"))
    eng.close()


@pytest.mark.parametrize("encoder", [False, True], ids=["decoder", "encoder"])
def test_vae(cuda, encoder):
    from oracle.vae import tiny_vae_config
    from sdwebui_b200.checkpoint import synthetic_state_dict, vae_decoder_param_shapes, vae_encoder_param_shapes
    from sdwebui_b200.engine import VAEDecoderEngine, VAEEncoderEngine, VAESpec

    L, lib = _lib()
    spec = VAESpec.from_any(tiny_vae_config())
    f = 2 ** (len(spec.ch_mult) - 1)
    code = L.torch_dtype_code(torch.float16)
    if encoder:
        eng = _finalized(VAEEncoderEngine(spec, dtype=torch.float16, device=cuda),
                         synthetic_state_dict(vae_encoder_param_shapes(spec), 2))
        n, h, w = 1, 64, 64
        x, out = _rand(n, 3, h, w), torch.empty(n, 2 * spec.z_channels, h // f, w // f, dtype=torch.float16, device=cuda)
        fn = lib.sdxe_vae_encode
    else:
        eng = _finalized(VAEDecoderEngine(spec, dtype=torch.float16, device=cuda),
                         synthetic_state_dict(vae_decoder_param_shapes(spec), 3))
        n, h, w = 1, 16, 16
        x, out = _rand(n, 4, h, w), torch.empty(n, spec.out_ch, h * f, w * f, dtype=torch.float16, device=cuda)
        fn = lib.sdxe_vae_decode
    _check(lambda: L.check(fn(eng._h, L.ptr(x), L.ptr(out), n, h, w, code, L.current_stream()), "sdxe_vae"))
    eng.close()


@pytest.mark.parametrize("fixes,out_dtype,final_norm", [(False, torch.float32, True), (True, torch.float16, False)],
                         ids=["fp32_out", "fixes_16bit_out"])
def test_clip_forward(cuda, fixes, out_dtype, final_norm):
    from oracle.clip import CLIPTextModel, tiny_clip_config
    from sdwebui_b200.engine import CLIPTextEngine, CLIPTextSpec

    L, lib = _lib()
    cfg = tiny_clip_config()
    torch.manual_seed(3)
    spec = CLIPTextSpec(vocab_size=cfg.vocab_size, hidden_size=cfg.hidden_size, intermediate_size=cfg.intermediate_size,
                        num_layers=cfg.num_layers, num_heads=cfg.num_heads, max_positions=cfg.max_positions, act="quick_gelu")
    eng = _finalized(CLIPTextEngine(spec, dtype=torch.float16, device=cuda), CLIPTextModel(cfg).state_dict())
    n, T = 2, 77
    ids = torch.randint(0, cfg.vocab_size, (n, T), dtype=torch.int32, device=cuda)
    out = torch.empty(n, T, cfg.hidden_size, dtype=out_dtype, device=cuda)
    rows = torch.tensor([5, 80, 81], dtype=torch.int32, device=cuda) if fixes else None
    vecs = _rand(3, cfg.hidden_size) if fixes else None
    n_fix = 3 if fixes else 0
    _check(lambda: L.check(lib.sdxe_clip_forward_fixes(eng._h, L.ptr(ids), L.ptr(out), n, T, cfg.num_layers, int(final_norm),
                                                       L.torch_dtype_code(out_dtype), L.ptr(rows), L.ptr(vecs), n_fix,
                                                       L.current_stream()), "sdxe_clip_forward_fixes"))
    eng.close()
