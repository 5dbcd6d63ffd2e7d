"""Hypertile on the engine: gather + segmented flash attention against torch, UNet forwards with fixed draws against the
fp32 oracle wrapped by tests/hypertile_oracle.py, the static-graph property (draws change per call, the plan and its
graph do not), and whole jobs against the oracle pipeline.

Tolerances as DESIGN §4: the primitive element by element within tests/prim_bounds.py's fp64 bound; a UNet forward's
below max(3 x the reference 16-bit path's error, 2e-3 fp16 / 1.6e-2 bf16); a job's latents below max(3 x torch fp16's,
5e-3) with PSNR >= 35 dB."""
import copy
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import hypertile_oracle as HO  # noqa: E402
import prim_bounds as PB  # noqa: E402

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


def rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def _floor(dtype):
    return 2e-3 if dtype == torch.float16 else 1.6e-2


# ---- primitive --------------------------------------------------------------------------------------------------
# (B, H, D, h', w', nh, nw, max_tiles): square, transposed grid (152 x 104 of a 1216 x 832 image), ragged T (19 x 52 =
# 988 tokens per tile), nh = 3, a single tile, and a draw below the grid's bound
PRIM_CASES = [
    (2, 8, 40, 64, 64, 2, 2, 4),
    (1, 5, 64, 152, 104, 8, 2, 16),
    (2, 4, 80, 96, 64, 3, 2, 6),
    (1, 2, 160, 48, 32, 3, 1, 9),
    (2, 8, 40, 32, 32, 1, 1, 4),
    (1, 10, 64, 64, 96, 2, 3, 9),
    # tiles of 6 x 10 = 60 tokens (less than one KV block), three per row; 13 x 10 = 130 (a ragged second Q tile);
    # 13 x 5 = 65 (a last KV block of one key, the next tile's first key right behind it)
    (2, 4, 40, 12, 30, 2, 3, 6),
    (1, 5, 64, 26, 20, 2, 2, 4),
    (1, 2, 80, 13, 10, 1, 2, 2),
]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", PRIM_CASES, ids=lambda c: "B{}H{}d{}_{}x{}_{}x{}".format(*c[:7]))
def test_hypertile_attention_primitive(cuda, dtype, case):
    """Element by element against the fp64 bound of tests/prim_bounds.py. Every tile's first token holds a dominant
    key (prim_bounds.hypertile_inputs): in tile-major order it sits in the previous tile's masked last KV block, so a
    mask that lets a key past T in moves that tile's rows by O(|v|). The input sits before a NaN tail of one KV block,
    the output before a sentinel tail, and a second call must give the same bits."""
    from sdwebui_b200 import lib as L

    lib = L.load()
    B, H, D, hp, wp, nh, nw, mt = case
    N = hp * wp
    th, tw = hp // nh, wp // nw
    qkv = PB.moat(PB.hypertile_inputs(B, H, D, hp, wp, nh, nw, dtype, 3).to(cuda), 64 * 3 * H * D)
    tiled = torch.empty_like(qkv)
    out, flat = PB.out_buffer((B, N, H * D), 128 * H * D, dtype, cuda)
    draw = torch.tensor([nh, nw], dtype=torch.int32, device=cuda)

    def call():
        L.check(lib.sdxe_hypertile_attention(L.ptr(qkv), L.ptr(tiled), L.ptr(draw), L.ptr(out), B, H, hp, wp, D, mt,
                                             D ** -0.5, L.torch_dtype_code(dtype), L.current_stream()),
                "sdxe_hypertile_attention")

    call()
    first = out.clone()
    call()
    torch.cuda.synchronize()
    assert PB.same_bits(first, out), "second call gave different bits"
    assert PB.sentinel_intact(flat, out.numel()), "store past the end of the output"
    q, k, v = (HO.regroup(t, hp, wp, nh, nw) for t in qkv.split(H * D, dim=-1))
    bt, T, _ = q.shape
    ref, bound = PB.attention_ref(*(t.reshape(bt, T, H, D).transpose(1, 2) for t in (q, k, v)))
    ref, bound = HO.ungroup(ref, hp, wp, nh, nw), HO.ungroup(bound, hp, wp, nh, nw)

    def where(i):
        r, c = divmod(i[1], wp)
        tile, t = (r // th) * nw + c // tw, (r % th) * tw + c % tw
        return (f"batch {i[0]} head {i[2] // D}, tile {tile} of {nh}x{nw} ({th}x{tw} = {T} tokens), tile-major row {t} "
                f"(Q tile {t // 128}), {(T + 63) // 64} KV blocks, the last holding {T - 64 * ((T - 1) // 64)} keys")

    PB.check(f"hypertile attention {'fp16' if dtype == torch.float16 else 'bf16'} {case}", first, ref, bound, where)
    assert torch.equal(tiled, HO.regroup(qkv, hp, wp, nh, nw).reshape(B, N, -1))


# ---- UNet forward -----------------------------------------------------------------------------------------------
def _model(cfg, seed, device):
    from oracle.synth import init_module_
    from oracle.unet import UNetModel

    return init_module_(UNetModel(cfg), seed).eval().to(device)


def _engine(model, cfg, dtype, device):
    from sdwebui_b200.engine import UNetEngine, UNetSpec

    eng = UNetEngine(UNetSpec.from_any(cfg), dtype=dtype, device=device)
    eng.load_state_dict(model.state_dict())
    eng.finalize()
    return eng


def _fixed_rows(spec, h, w, draws_by_level, max_tiles=16):
    """Rows with the grid of a square image (h' = h_l, w' = w_l) and a fixed draw per level (None: untiled)."""
    from sdwebui_b200.hypertile import attn1_layers

    rows = []
    for _, level in attn1_layers(spec):
        d = draws_by_level.get(level)
        hl, wl = (h + 2 ** level - 1) // 2 ** level, (w + 2 ** level - 1) // 2 ** level
        rows.append((hl, wl, d[0], d[1], max_tiles) if d else (0, 0, 1, 1, 0))
    return rows


def _inputs(cfg, n, h, w, device, seed=5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, 4, h, w, device=device, generator=g)
    t = torch.rand(n, device=device, generator=g) * 999
    ctx = torch.randn(n, 77, cfg.context_dim, device=device, generator=g)
    y = torch.randn(n, cfg.adm_in_channels, device=device, generator=g) if cfg.adm_in_channels else None
    return x, t, ctx, y


def _check_forward(tag, model, eng, spec, cfg, dtype, x, t, ctx, y, rows):
    with torch.no_grad(), HO.hypertile_unet(model, spec, lambda _x: rows):
        ref32 = model(x, t.to(dtype).float(), context=ctx.to(dtype).float(), y=None if y is None else y.to(dtype).float())
        m16 = copy.deepcopy(model).to(dtype)
    with torch.no_grad(), HO.hypertile_unet(m16, spec, lambda _x: rows), torch.autocast("cuda", dtype=dtype):
        ref16 = m16(x.to(dtype), t.to(dtype), context=ctx.to(dtype), y=None if y is None else y.to(dtype))
    del m16
    out = eng.forward(x.to(dtype), t.to(dtype), ctx.to(dtype), None if y is None else y.to(dtype), hypertile=rows)
    e_eng, e_ref = rel_err(out, ref32), rel_err(ref16, ref32)
    print(f"{tag} {dtype}: engine {e_eng:.3e}  ref16 {e_ref:.3e}")
    assert e_eng < max(3 * e_ref, _floor(dtype)), (e_eng, e_ref)
    return out


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("variant", ["conv", "linear_adm"])
def test_tiny_unet_hypertile(cuda, dtype, variant):
    from oracle.unet import tiny_config
    from sdwebui_b200.engine import UNetSpec

    cfg = tiny_config(linear=(variant == "linear_adm"), adm=(96 if variant == "linear_adm" else 0))
    spec = UNetSpec.from_any(cfg)
    model = _model(cfg, 11, cuda)
    eng = _engine(model, cfg, dtype, cuda)
    # square 32 x 32 (level 0 in 2 x 4 tiles), and 24 x 40 with 3 x 5 tiles of 8 x 8 tokens at level 0
    for n, h, w, draws in [(2, 32, 32, {0: (2, 4), 1: (2, 2)}), (3, 24, 40, {0: (3, 5), 1: (1, 2)})]:
        x, t, ctx, y = _inputs(cfg, n, h, w, cuda)
        rows = _fixed_rows(spec, h, w, draws)
        _check_forward(f"tiny {variant} {n}x{h}x{w} {draws}", model, eng, spec, cfg, dtype, x, t, ctx, y, rows)
    eng.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_unit_draws_and_off_change_nothing(cuda, dtype):
    """All draws (1, 1) give the bits of Hypertile off; off leaves the op list as it is without Hypertile."""
    from oracle.unet import tiny_config
    from sdwebui_b200.engine import UNetSpec

    cfg = tiny_config()
    spec = UNetSpec.from_any(cfg)
    model = _model(cfg, 11, cuda)
    eng = _engine(model, cfg, dtype, cuda)
    x, t, ctx, y = _inputs(cfg, 2, 32, 24, cuda)
    args = (x.to(dtype), t.to(dtype), ctx.to(dtype))
    off = eng.forward(*args)
    ones = eng.forward(*args, hypertile=_fixed_rows(spec, 32, 24, {0: (1, 1), 1: (1, 1)}))
    assert torch.equal(off, ones)
    off2 = eng.forward(*args)  # the table applies to one call: the next call without it is off again
    assert torch.equal(off, off2)
    eng.close()


def _profiled_ops(eng, call, tmp_path, name):
    dump = tmp_path / name
    os.environ["SDXE_PROFILE_DUMP"] = str(dump)
    try:
        eng.profile(True)
        out = call()
        torch.cuda.synchronize()
        eng.profile(False)
    finally:
        del os.environ["SDXE_PROFILE_DUMP"]
    return out, [line.split(",")[2] for line in dump.read_text().splitlines()]


def test_static_graph_with_changing_draws(cuda, tmp_path):
    """Calls on one plan with different draws: each matches the eager profiled run of the same draws bit for bit, the
    launch count is the same for every call and for the eager run, and the plan cache does not grow. That the count
    equals the kernels torch.profiler sees is checked in test_launch_count_hypertile_gpu.py."""
    from oracle.unet import tiny_config
    from sdwebui_b200 import lib as L
    from sdwebui_b200.engine import UNetSpec

    lib = L.load()
    dtype = torch.float16
    cfg = tiny_config()
    spec = UNetSpec.from_any(cfg)
    model = _model(cfg, 11, cuda)
    eng = _engine(model, cfg, dtype, cuda)
    x, t, ctx, y = _inputs(cfg, 2, 32, 32, cuda)
    args = (x.to(dtype), t.to(dtype), ctx.to(dtype))
    rows_a = _fixed_rows(spec, 32, 32, {0: (4, 2), 1: (2, 2)})
    rows_b = _fixed_rows(spec, 32, 32, {0: (1, 4), 1: (1, 1)})
    eng.forward(*args, hypertile=rows_a)  # build + capture
    _, n_plans = eng.pool_stats()
    results, counts = [], []
    for rows in (rows_a, rows_b, rows_a):
        torch.cuda.synchronize()
        n0 = lib.sdxe_launch_count()
        out = eng.forward(*args, hypertile=rows)
        torch.cuda.synchronize()
        counts.append(lib.sdxe_launch_count() - n0)
        results.append(out.clone())
    assert counts[0] == counts[1] == counts[2]
    assert eng.pool_stats()[1] == n_plans
    assert torch.equal(results[0], results[2]) and not torch.equal(results[0], results[1])
    for rows, res, name in ((rows_a, results[0], "a"), (rows_b, results[1], "b")):
        eager, ops = _profiled_ops(eng, lambda: eng.forward(*args, hypertile=rows), tmp_path, name)
        assert torch.equal(eager, res)
        assert sum(1 for d in ops if d.startswith("ht_gather")) == sum(1 for r in rows if r[4])
        eng.profile(True)
        torch.cuda.synchronize()
        n0 = lib.sdxe_launch_count()
        eng.forward(*args, hypertile=rows)
        torch.cuda.synchronize()
        eng.profile(False)
        assert lib.sdxe_launch_count() - n0 == counts[0]  # eager and graph replay run the same kernels
    eng.close()


# ---- full size ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model_name", ["sd15", "sdxl"])
def test_fullsize_hypertile(cuda, model_name):
    """SD1.5 at 1024^2 (2B = 8, level 0 in 4 x 4 tiles) and SDXL at 1024^2 (2B = 4), reference default settings'
    largest draws, random-init weights, fp16."""
    from oracle.unet import sd15_config, sdxl_config
    from sdwebui_b200.engine import UNetSpec
    from sdwebui_b200 import hypertile as HT

    dtype = torch.float16
    cfg, n, is_sdxl = (sd15_config(), 8, False) if model_name == "sd15" else (sdxl_config(), 4, True)
    spec = UNetSpec.from_any(cfg)
    model = _model(cfg, 21, cuda)
    eng = _engine(model, cfg, dtype, cuda)
    st = HT.configure(spec, 1024, 1024, HT.HypertileOptions(enable_unet=True), True, is_sdxl)
    rows = [(hp, wp, mt and HT.get_divisors(hp, max(128, l.tile_size) // 8 * 2 ** l.depth, 3)[0],
             mt and HT.get_divisors(wp, max(128, l.tile_size) // 8 * 2 ** l.depth, 3)[0], mt) if mt else r
            for r, l in zip(st.draw_rows(128, 128), st.layers) for hp, wp, _, _, mt in [r]]
    if model_name == "sd15":
        assert rows[0][2:4] == (4, 4)
    x, t, ctx, y = _inputs(cfg, n, 128, 128, cuda)
    _check_forward(f"{model_name} 1024^2 n={n}", model, eng, spec, cfg, dtype, x, t, ctx, y, rows)
    eng.close()


# ---- end to end -------------------------------------------------------------------------------------------------
def _job(cuda, hires):
    from oracle.pipeline import OraclePipeline, SamplingParams
    from oracle.synth import init_module_, synthetic_context
    from oracle.unet import UNetModel, tiny_config
    from oracle.vae import AutoencoderKLDecode, tiny_vae_config
    from sdwebui_b200 import hypertile as HT
    from sdwebui_b200.engine import UNetSpec, VAEDecoderEngine, VAESpec
    from sdwebui_b200.processing import SdModel, StableDiffusionProcessingTxt2Img, process_images
    from sdwebui_b200.sd_unet import SdxeUnet

    ucfg, vcfg = tiny_config(), tiny_vae_config()
    spec = UNetSpec.from_any(ucfg)
    unet = init_module_(UNetModel(ucfg), 1).eval().to(cuda)
    vae = init_module_(AutoencoderKLDecode(vcfg), 2).eval().to(cuda)
    B, steps, W, H = 2, 4, 256, 256
    cond = synthetic_context(B, 77, ucfg.context_dim, 3, cuda)
    uncond = synthetic_context(B, 77, ucfg.context_dim, 4, cuda)
    seeds = (1000, 1001)
    # small tiles so that the tiny UNet's 32 x 32 level 0 has real choices: max tile 128 -> 16-token tiles
    opts = HT.HypertileOptions(enable_unet=not hires, enable_unet_secondpass=hires, max_tile_unet=128, swap_size_unet=3)
    su = SdxeUnet(unet.state_dict(), spec, dtype=torch.float16, device=cuda)
    su.activate()
    ve = VAEDecoderEngine(VAESpec.from_any(vcfg), dtype=torch.float16, device=cuda)
    ve.load_state_dict(vae.state_dict())
    ve.finalize()
    model = SdModel(su, ve, is_sdxl=False, dtype_unet=torch.float16, device=cuda)
    kw = dict(enable_hr=True, hr_scale=1.5, denoising_strength=0.6) if hires else {}
    p = StableDiffusionProcessingTxt2Img(sd_model=model, c=cond, uc=uncond, seeds=list(seeds), sampler_name="Euler",
                                         steps=steps, width=W, height=H, randn_source="NV", hypertile=opts, **kw)
    res = process_images(p)
    assert su.hypertile is None
    eng_lat = res.latents.float()

    # the oracle with the same draws: seeded and configured as the job does, one draw set per UNet forward
    state = {}

    def rows_fn(x):
        if state["hr_pending"] and state["calls"] == steps:  # the first pass made `steps` UNet calls (Euler, batched CFG)
            state["st"] = HT.begin_hr_pass(p, int(W * 1.5), int(H * 1.5))
            state["hr_pending"] = False
        state["calls"] += 1
        st = state["st"]
        return st.draw_rows(x.shape[-2], x.shape[-1]) if st is not None else [(0, 0, 1, 1, 0)] * len(HT.attn1_layers(spec))

    sp = SamplingParams(sampler="Euler", steps=steps, width=W, height=H, seeds=seeds, randn_source="NV", **kw)

    def run(pipe):
        state.update(calls=0, hr_pending=hires, st=HT.begin_job(p))  # seeds the draws as the job did
        with torch.no_grad(), HO.hypertile_unet(unet, spec, rows_fn):
            return pipe.txt2img(sp, cond, uncond)[0].float()

    lat32 = run(OraclePipeline(unet, vae, cuda, dtype_unet=torch.float32))
    lat16 = run(OraclePipeline(unet, vae, cuda, dtype_unet=torch.float16, dtype_vae=torch.float32, autocast=True))
    su.deactivate()
    return eng_lat, lat32, lat16


@pytest.mark.parametrize("hires", [False, True], ids=["txt2img_enable_unet", "hires_secondpass_only"])
def test_job_against_oracle(cuda, hires):
    eng, ref32, ref16 = _job(cuda, hires)
    e_eng, e_ref = rel_err(eng, ref32), rel_err(ref16, ref32)
    peak = ref32.abs().max().item()
    psnr = 10 * torch.log10(torch.tensor(peak ** 2 / ((eng - ref32) ** 2).mean().item())).item()
    print(f"hypertile job hires={hires}: engine {e_eng:.3e} (PSNR {psnr:.1f} dB)  torch fp16 {e_ref:.3e}")
    assert e_eng < max(3 * e_ref, 5e-3), (e_eng, e_ref)
    assert psnr >= 35.0
