"""The engine at latent sizes whose sides are not powers of two (SD1.5 512x768, SDXL's aspect buckets and the like).

Which kernel a 3x3 convolution runs depends on its geometry (conv_tile_shape, csrc/gemm.cu): the implicit TMA convolution
("T") takes an H x W plane only when W is a multiple of 128, or W divides 128 and the rows tile evenly; every other plane
goes through im2col3x3 + a plain GEMM over the column buffer ("I"). The cases below are chosen so that the tiny models take
every branch, and each asserts from the profiled op descriptors which one it took, so a change of the dispatch cannot
turn a case into a duplicate of another without a failure.

Yardstick as in test_engine_gpu.py: relative L2 error vs the fp32 oracle below max(3 x the reference 16-bit path's
error, 2e-3 fp16 / 1.6e-2 bf16). It is applied to the whole output, to each image on its own (a bad last tile cannot hide
in the batch average) and to the band of the outer 2 latent rows and columns (where the padding taps are), with the
reference's error measured on the same region.

Run as a script, this file is the child process of test_conv_s2_implicit_matches_im2col.
"""
import copy
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


def rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def _floor(dtype):
    return 2e-3 if dtype == torch.float16 else 1.6e-2


def _check_regions(tag, out, ref32, ref16, band, dtype):
    """Engine vs ref16 error (both against ref32) on the whole output, on each image and on the border band."""
    H, W = out.shape[-2:]
    border = torch.ones(H, W, dtype=torch.bool, device=out.device)
    border[band:H - band, band:W - band] = False
    regions = [("all", lambda t: t)]
    regions += [(f"image {i}", lambda t, i=i: t[i]) for i in range(out.shape[0])]
    regions += [("border", lambda t: t[..., border])]
    bad = []
    for name, sel in regions:
        e_eng, e_ref = rel_err(sel(out), sel(ref32)), rel_err(sel(ref16), sel(ref32))
        print(f"{tag} {name:8s}: engine {e_eng:.3e}  ref16 {e_ref:.3e}")
        if not e_eng < max(3 * e_ref, _floor(dtype)):
            bad.append((name, e_eng, e_ref))
    assert not bad, bad


def _ops(path):
    """(op, {field: value}) per line of an SDXE_PROFILE_DUMP file (index,kind,descriptor,us,flops,bytes)."""
    ops = []
    for line in path.read_text().splitlines():
        words = line.split(",")[2].split()
        if words:
            ops.append((words[0], dict(w.split("=", 1) for w in words[1:] if "=" in w)))
    return ops


def _im2col_gemms(ops, M):
    """GEMMs over an im2col column buffer of M output pixels. Their K is 9 x Cin with Cin a multiple of 64; no other
    GEMM of the tiny models has such a K (theirs are C, 4C, a channel concat or a padded 4-channel input)."""
    return [f for op, f in ops if op == "gemm" and int(f["M"]) == M and int(f["K"]) % 576 == 0]


def _path(what, implicit, im2col):
    assert bool(implicit) != bool(im2col), f"{what}: implicit convs {implicit}, im2col GEMMs {im2col}"
    return "T" if implicit else "I"


def _unet_paths(ops, n, h, w):
    """Path of the tiny UNet's level-0 convs, its Downsample and its level-1 convs, as a string such as "TII"."""
    h1, w1 = h // 2, w // 2
    m1 = n * h1 * w1
    level0 = _path("level 0", [f for op, f in ops if op == "conv3" and f["HxW"] == f"{h}x{w}"], _im2col_gemms(ops, n * h * w))
    # the Downsample keeps the 64 level-0 channels; every level-1 conv writes 128
    down = _path("Downsample", [f for op, f in ops if op == "conv3s2" and f["HoxWo"] == f"{h1}x{w1}"],
                 [f for f in _im2col_gemms(ops, m1) if f["N"] == "64" and f["K"] == "576"])
    level1 = _path("level 1", [f for op, f in ops if op == "conv3" and f["HxW"] == f"{h1}x{w1}"],
                   [f for f in _im2col_gemms(ops, m1) if f["N"] == "128"])
    return level0 + down + level1


def _all_im2col(ops, n, sizes):
    """Every conv, stride 1 or 2, went through im2col, and each plane in `sizes` had im2col GEMMs."""
    assert not [f for op, f in ops if op in ("conv3", "conv3s2")]
    for h, w in sizes:
        assert _im2col_gemms(ops, n * h * w), (h, w)


def _profiled(eng, monkeypatch, path, fn):
    """One extra call with per-op profiling, its op descriptors dumped to `path`."""
    monkeypatch.setenv("SDXE_PROFILE_DUMP", str(path))
    eng.profile(True)
    try:
        out = fn()
    finally:
        eng.profile(False)
        monkeypatch.delenv("SDXE_PROFILE_DUMP")
    return out, _ops(path)


# latent (n, h, w) -> path of the level-0 convs, the Downsample and the level-1 convs
UNET_GEOMETRY = [
    ((2, 24, 40), "III"),
    ((3, 12, 8), "III"),   # ragged M tiles at every level
    ((2, 48, 16), "TII"),  # both paths in one plan
    ((5, 8, 8), "TTT"),    # several images per tile, an odd count, a partial last tile
    ((1, 8, 136), "III"),  # W > 128 but not a multiple of 128
    ((2, 10, 6), "III"),   # 60 pixels per image
]


@pytest.mark.parametrize("shape,paths", UNET_GEOMETRY, ids=[f"{n}x{h}x{w}" for (n, h, w), _ in UNET_GEOMETRY])
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("variant", ["conv", "linear_adm"])
def test_tiny_unet_geometry(cuda, monkeypatch, tmp_path, variant, dtype, shape, paths):
    from oracle.synth import init_module_
    from oracle.unet import UNetModel, tiny_config
    from sdwebui_b200.engine import UNetEngine, UNetSpec

    cfg = tiny_config(linear=(variant == "linear_adm"), adm=(96 if variant == "linear_adm" else 0))
    model = init_module_(UNetModel(cfg), 11).eval().to(cuda)
    eng = UNetEngine(UNetSpec.from_any(cfg), dtype=dtype, device=cuda)
    eng.load_state_dict(model.state_dict())
    eng.finalize()
    n, h, w = shape
    g = torch.Generator(device="cuda").manual_seed(1000 * n + 10 * h + w)
    x = torch.randn(n, 4, h, w, device=cuda, generator=g).to(dtype)
    t = (torch.rand(n, device=cuda, generator=g) * 999).to(dtype)
    ctx = torch.randn(n, 77, cfg.context_dim, device=cuda, generator=g).to(dtype)
    y = torch.randn(n, cfg.adm_in_channels, device=cuda, generator=g).to(dtype) if cfg.adm_in_channels else None
    with torch.no_grad():
        ref32 = model(x.float(), t.float(), context=ctx.float(), y=None if y is None else y.float())
        with torch.autocast("cuda", dtype=dtype):  # the reference's GPU path: 16-bit weights and inputs under autocast
            ref16 = copy.deepcopy(model).to(dtype)(x, t, context=ctx, y=y)
    out = eng.forward(x, t, ctx, y)
    assert out.shape == x.shape and out.dtype == dtype
    _check_regions(f"tiny unet {variant} {str(dtype)[6:]} {n}x{h}x{w}", out, ref32, ref16, 2, dtype)
    # graph replay, and the eager per-op profiled run, give the same bits as the first call
    assert torch.equal(eng.forward(x, t, ctx, y), out)
    out_p, ops = _profiled(eng, monkeypatch, tmp_path / "ops.csv", lambda: eng.forward(x, t, ctx, y))
    assert torch.equal(out_p, out)
    assert _unet_paths(ops, n, h, w) == paths
    eng.close()


@pytest.mark.parametrize("n,h,w", [(1, 12, 20), (2, 20, 12)])
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
def test_tiny_vae_decoder_geometry(cuda, monkeypatch, tmp_path, dtype, n, h, w):
    from oracle.synth import init_module_
    from oracle.vae import AutoencoderKLDecode, tiny_vae_config
    from sdwebui_b200.engine import VAEDecoderEngine, VAESpec

    cfg = tiny_vae_config()
    vae = init_module_(AutoencoderKLDecode(cfg), 31).eval().to(cuda)
    eng = VAEDecoderEngine(VAESpec.from_any(cfg), dtype=dtype, device=cuda)
    eng.load_state_dict(vae.state_dict())
    eng.finalize()
    g = torch.Generator(device="cuda").manual_seed(1000 * n + 10 * h + w)
    z = (torch.randn(n, 4, h, w, device=cuda, generator=g) * 3).to(dtype)
    with torch.no_grad():
        ref32 = vae.decode(z.float())
        ref16 = copy.deepcopy(vae).to(dtype).decode(z)
    out = eng.decode(z)
    levels = len(cfg.ch_mult)
    up = 2 ** (levels - 1)
    assert out.shape == (n, 3, h * up, w * up)
    _check_regions(f"tiny vae decoder {str(dtype)[6:]} {n}x{h}x{w}", out, ref32, ref16, 2 * up, dtype)
    _, ops = _profiled(eng, monkeypatch, tmp_path / "ops.csv", lambda: eng.decode(z))
    _all_im2col(ops, n, [(h << l, w << l) for l in range(levels)])
    eng.close()


@pytest.mark.parametrize("ch_mult,n,h,w", [((1, 2), 2, 48, 80),
                                           ((1, 2, 2, 2), 1, 96, 160)])  # three stride-2 im2col convs with pad_lo = 0
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
def test_tiny_vae_encoder_geometry(cuda, monkeypatch, tmp_path, dtype, ch_mult, n, h, w):
    from oracle.synth import init_module_
    from oracle.vae import AutoencoderKLEncode, tiny_vae_config
    from sdwebui_b200.engine import VAEEncoderEngine, VAESpec

    cfg = tiny_vae_config()
    cfg.ch_mult = list(ch_mult)
    enc = init_module_(AutoencoderKLEncode(cfg), 33).eval().to(cuda)
    eng = VAEEncoderEngine(VAESpec.from_any(cfg), dtype=dtype, device=cuda)
    eng.load_state_dict(enc.state_dict())
    eng.finalize()
    g = torch.Generator(device="cuda").manual_seed(1000 * n + 10 * h + w)
    x = (torch.rand(n, 3, h, w, device=cuda, generator=g) * 2 - 1).to(dtype)
    with torch.no_grad():
        ref32 = enc.encode_moments(x.float())
        ref16 = copy.deepcopy(enc).to(dtype).encode_moments(x)
    out = eng.encode_moments(x)
    levels = len(cfg.ch_mult)
    f = 2 ** (levels - 1)
    assert out.shape == (n, 2 * cfg.z_channels, h // f, w // f)
    _check_regions(f"tiny vae encoder {list(ch_mult)} {str(dtype)[6:]} {n}x{h}x{w}", out, ref32, ref16, 2, dtype)
    _, ops = _profiled(eng, monkeypatch, tmp_path / "ops.csv", lambda: eng.encode_moments(x))
    _all_im2col(ops, n, [(h >> l, w >> l) for l in range(levels)])
    eng.close()


# ---- stride-2 conv: implicit TMA path vs im2col on the same operands ------------------------------------------------
# Where a stride-2 conv3 can run implicitly, SDXE_CONV_S2_IMPLICIT=0 sends it through im2col instead. Both feed the GEMM the
# same 16-bit operands (TMA's out-of-bounds zero fill is im2col's zero padding, and K runs tap-major, tap * C + c, in
# both) with the same K = 9C, hence the same tile width and epilogue: the outputs must be bit-identical.
# The switch is read once per process, so each setting runs in a child process (this file run as a script).

S2_DOWNSAMPLES = {"unet-fp16": 1, "unet-bf16": 1, "vae_encoder": 1, "vae_encoder_f8": 3}


def _s2_child(out_dir):
    """Every stride-2 case once, weights and inputs seeded on the CPU so that both processes see the same bits; the
    outputs go to out_dir/out.pt, one profiled call per case to out_dir/<case>.csv."""
    from oracle.synth import init_module_
    from oracle.unet import UNetModel, tiny_config
    from oracle.vae import AutoencoderKLEncode, tiny_vae_config
    from sdwebui_b200.engine import UNetEngine, UNetSpec, VAEEncoderEngine, VAESpec

    dev = torch.device("cuda:0")
    outs = {}

    def run(case, eng, fn):
        outs[case] = fn().cpu()
        os.environ["SDXE_PROFILE_DUMP"] = os.path.join(out_dir, case + ".csv")
        eng.profile(True)
        fn()
        eng.profile(False)
        del os.environ["SDXE_PROFILE_DUMP"]
        eng.close()

    cfg = tiny_config()
    unet = init_module_(UNetModel(cfg), 11).eval()
    for name, dtype in (("fp16", torch.float16), ("bf16", torch.bfloat16)):
        eng = UNetEngine(UNetSpec.from_any(cfg), dtype=dtype, device=dev)
        eng.load_state_dict({k: v.to(dev) for k, v in unet.state_dict().items()})
        eng.finalize()
        g = torch.Generator().manual_seed(5)
        x = torch.randn(2, 4, 32, 32, generator=g).to(dev, dtype)
        t = torch.tensor([801.0, 37.5]).to(dev, dtype)
        ctx = torch.randn(2, 77, cfg.context_dim, generator=g).to(dev, dtype)
        run(f"unet-{name}", eng, lambda: eng.forward(x, t, ctx))
    for case, ch_mult, hw in (("vae_encoder", [1, 2], 64), ("vae_encoder_f8", [1, 2, 2, 2], 128)):
        vcfg = tiny_vae_config()
        vcfg.ch_mult = ch_mult
        enc = init_module_(AutoencoderKLEncode(vcfg), 33).eval()
        eng = VAEEncoderEngine(VAESpec.from_any(vcfg), dtype=torch.float16, device=dev)
        eng.load_state_dict({k: v.to(dev) for k, v in enc.state_dict().items()})
        eng.finalize()
        g = torch.Generator().manual_seed(9)
        x = (torch.rand(1, 3, hw, hw, generator=g) * 2 - 1).to(dev, torch.float16)
        run(case, eng, lambda: eng.encode_moments(x))
    torch.save(outs, os.path.join(out_dir, "out.pt"))


@pytest.fixture(scope="module")
def s2_runs(cuda, tmp_path_factory):
    """{implicit (1 / 0): (outputs by case, directory of the op dumps)}"""
    runs = {}
    for implicit in (1, 0):
        d = tmp_path_factory.mktemp(f"conv_s2_implicit{implicit}")
        env = dict(os.environ, SDXE_CONV_S2_IMPLICIT=str(implicit))
        env.pop("SDXE_PROFILE_DUMP", None)
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), str(d)]
        r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
        runs[implicit] = (torch.load(d / "out.pt"), d)
    return runs


@pytest.mark.parametrize("case", list(S2_DOWNSAMPLES))
def test_conv_s2_implicit_matches_im2col(s2_runs, case):
    (out_t, dir_t), (out_i, dir_i) = s2_runs[1], s2_runs[0]
    implicit_t = [f for op, f in _ops(dir_t / f"{case}.csv") if op == "conv3s2"]
    implicit_i = [f for op, f in _ops(dir_i / f"{case}.csv") if op == "conv3s2"]
    assert len(implicit_t) == S2_DOWNSAMPLES[case] and not implicit_i
    a, b = out_t[case], out_i[case]
    assert torch.isfinite(a.float()).all()
    print(f"{case}: implicit vs im2col max |diff| {(a.float() - b.float()).abs().max().item():.3e}")
    assert torch.equal(a, b)


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    _s2_child(sys.argv[1])
