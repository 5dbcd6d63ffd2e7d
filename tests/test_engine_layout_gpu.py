"""The engine's host-side layout pinned exactly: for small seeded UNet, VAE and CLIP engines, the packed weight blob (size
and SHA-256), the activation-pool bytes after one forward (sdxe_pool_bytes), the launches of a replayed call, and the
profiled op list (kind, descriptor, FLOPs, bytes) against tests/golden/engine_layout_ref.json. The blob is what
parallel.broadcast_weight_blob ships to other ranks, so its bytes are part of the engine's interface; the pool bytes and
the op list follow the order in which a plan allocates and emits. Also pins the missing-weight report of
sdxe_finalize.

tests/golden/make_golden_engine_layout.py writes the golden file from these same cases."""
import hashlib
import json
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "engine_layout_ref.json")
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}


def _profiled_ops(eng, path, call):
    """(kind, descriptor, flops, bytes) of every op an eager profiled call runs (SDXE_PROFILE_DUMP)."""
    os.environ["SDXE_PROFILE_DUMP"] = str(path)
    eng.profile(True)
    try:
        call()
        torch.cuda.synchronize()
    finally:
        eng.profile(False)
        del os.environ["SDXE_PROFILE_DUMP"]
    ops = []
    for line in open(path).read().splitlines():
        _, kind, desc, _us, flops, by = line.split(",")
        ops.append([int(kind), desc, flops, by])
    os.remove(path)
    return ops


def _record(eng, call, tmp):
    from sdwebui_b200 import lib

    blob = eng.weight_blob().cpu().numpy().tobytes()
    call()  # builds the plan
    torch.cuda.synchronize()
    pool = eng.pool_stats()
    n0 = lib.load().sdxe_launch_count()
    call()  # graph replay
    torch.cuda.synchronize()
    launches = lib.load().sdxe_launch_count() - n0
    return {"blob_bytes": len(blob), "blob_sha256": hashlib.sha256(blob).hexdigest(), "pool_bytes": pool[0],
            "plans": pool[1], "launches": launches, "ops": _profiled_ops(eng, os.path.join(tmp, "ops.csv"), call)}


def _unet_spec(variant):
    from oracle.unet import tiny_config
    from sdwebui_b200.engine import UNetSpec

    # sd15: conv proj, heads by count; sdxl: linear proj, num_head_channels, adm_in_channels. Both have transformers at
    # both levels, a Downsample, an Upsample and skip-conv ResBlocks (64 -> 128 channels and the decoder's concats).
    return UNetSpec.from_any(tiny_config(linear=variant == "sdxl", adm=96 if variant == "sdxl" else 0))


def _unet_state_dict(spec, drop=()):
    from sdwebui_b200 import checkpoint as C

    sd = C.synthetic_state_dict(C.unet_param_shapes(spec), seed=21)
    return {k: v for k, v in sd.items() if k not in drop}


def _unet_engine(cuda, spec, dtype, drop=()):
    from sdwebui_b200.engine import UNetEngine

    eng = UNetEngine(spec, dtype=dtype, device=cuda)
    eng.load_state_dict(_unet_state_dict(spec, drop))
    return eng


def _hypertile_rows(spec, h, w):
    """One row per attn1 layer: level 0 (16 x 32 tokens) drawn 2 x 4 of at most 8 tiles, level 1 (8 x 16) 2 x 2 of 4."""
    from sdwebui_b200.hypertile import attn1_layers

    draws = {0: (2, 4, 8), 1: (2, 2, 4)}
    return [(h >> level, w >> level) + draws[level] for _, level in attn1_layers(spec)]


def _unet_case(cuda, tmp, variant, dtype, mode):
    spec = _unet_spec(variant)
    eng = _unet_engine(cuda, spec, dtype)
    eng.finalize()
    n, h, w = 2, 16, 32  # implicit-GEMM convs at both levels and in the Downsample
    g = torch.Generator().manual_seed(5)
    x = torch.randn(n, 4, h, w, generator=g).to(cuda, dtype)
    t = (torch.rand(n, generator=g) * 999).to(cuda, dtype)
    ctx = torch.randn(n, 77, spec.context_dim, generator=g).to(cuda, dtype)
    y = torch.randn(n, spec.adm_in_channels, generator=g).to(cuda, dtype) if spec.adm_in_channels else None
    rows = _hypertile_rows(spec, h, w) if mode == "hypertile" else None
    eng.set_circular(mode == "tiling")
    rec = _record(eng, lambda: eng.forward(x, t, ctx, y, hypertile=rows), tmp)
    eng.close()
    return rec


def _vae_engine(cuda, side, dtype, drop=()):
    from oracle.vae import tiny_vae_config
    from sdwebui_b200 import checkpoint as C
    from sdwebui_b200.engine import VAEDecoderEngine, VAEEncoderEngine, VAESpec

    spec = VAESpec.from_any(tiny_vae_config())
    if side == "decoder":
        E, shapes, seed = VAEDecoderEngine, C.vae_decoder_param_shapes(spec), 22
    else:
        E, shapes, seed = VAEEncoderEngine, C.vae_encoder_param_shapes(spec), 23
    eng = E(spec, dtype=dtype, device=cuda)
    eng.load_state_dict({k: v for k, v in C.synthetic_state_dict(shapes, seed=seed).items() if k not in drop})
    return eng


def _vae_case(cuda, tmp, side, dtype, tiling):
    eng = _vae_engine(cuda, side, dtype)
    eng.finalize()
    eng.set_circular(tiling)
    g = torch.Generator().manual_seed(6)
    if side == "decoder":
        z = torch.randn(1, 4, 12, 20, generator=g).to(cuda, dtype)  # im2col convs
        call = lambda: eng.decode(z)  # noqa: E731
    else:
        x = (torch.rand(2, 3, 64, 64, generator=g) * 2 - 1).to(cuda, dtype)
        call = lambda: eng.encode_moments(x)  # noqa: E731
    rec = _record(eng, call, tmp)
    eng.close()
    return rec


def _clip_case(cuda, tmp, dtype, final_norm):
    from oracle.clip import tiny_clip_config
    from test_clip_gpu import _models

    cfg = tiny_clip_config()
    _, eng = _models(cuda, cfg, dtype)
    g = torch.Generator().manual_seed(7)
    ids = torch.randint(0, cfg.vocab_size - 2, (3, 77), generator=g)
    rec = _record(eng, lambda: eng.forward(ids, final_norm=final_norm), tmp)
    eng.close()
    return rec


CASES = {
    "unet_sd15": lambda cuda, tmp, dt: _unet_case(cuda, tmp, "sd15", dt, None),
    "unet_sdxl": lambda cuda, tmp, dt: _unet_case(cuda, tmp, "sdxl", dt, None),
    "unet_sdxl_hypertile": lambda cuda, tmp, dt: _unet_case(cuda, tmp, "sdxl", dt, "hypertile"),
    "unet_sdxl_tiling": lambda cuda, tmp, dt: _unet_case(cuda, tmp, "sdxl", dt, "tiling"),
    "vae_decoder": lambda cuda, tmp, dt: _vae_case(cuda, tmp, "decoder", dt, False),
    "vae_decoder_tiling": lambda cuda, tmp, dt: _vae_case(cuda, tmp, "decoder", dt, True),
    "vae_encoder": lambda cuda, tmp, dt: _vae_case(cuda, tmp, "encoder", dt, False),
    "vae_encoder_tiling": lambda cuda, tmp, dt: _vae_case(cuda, tmp, "encoder", dt, True),
    "clip": lambda cuda, tmp, dt: _clip_case(cuda, tmp, dt, True),
    "clip_no_final_norm": lambda cuda, tmp, dt: _clip_case(cuda, tmp, dt, False),
}

# weights left out of a state dict, in the order sdxe_finalize reports them
DROPPED = {
    "unet": ["input_blocks.3.0.op.weight", "middle_block.1.transformer_blocks.0.attn2.to_k.weight"],
    "vae_decoder": ["decoder.mid.attn_1.k.weight", "decoder.up.1.upsample.conv.bias"],
    "vae_encoder": ["encoder.down.0.downsample.conv.weight", "encoder.mid.attn_1.proj_out.bias"],
}


def _missing_report(cuda, model):
    """The tail of sdxe_finalize's error (from "missing") when DROPPED[model] are left out."""
    from sdwebui_b200 import lib

    drop = DROPPED[model]
    if model == "unet":
        eng = _unet_engine(cuda, _unet_spec("sdxl"), torch.float16, drop)
    else:
        eng = _vae_engine(cuda, model[4:], torch.float16, drop)
    try:
        with pytest.raises(lib.SdxeError) as ei:
            eng.finalize()
    finally:
        eng.close()
    msg = str(ei.value)
    return msg[msg.index("missing"):]


def records(cuda, tmp):
    out = {}
    for name, case in CASES.items():
        for dn, dt in DTYPES.items():
            out[f"{name}/{dn}"] = case(cuda, tmp, dt)
    out["missing"] = {model: _missing_report(cuda, model) for model in DROPPED}
    return out


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("case", list(CASES))
def test_layout_matches_golden(cuda, tmp_path, case, dtype):
    want = _golden()[f"{case}/{dtype}"]
    got = CASES[case](cuda, str(tmp_path), DTYPES[dtype])
    for k in ("blob_bytes", "blob_sha256", "pool_bytes", "plans", "launches"):
        assert got[k] == want[k], (k, got[k], want[k])
    assert len(got["ops"]) == len(want["ops"])
    for i, (g, w) in enumerate(zip(got["ops"], want["ops"])):
        assert g == w, (i, g, w)


@pytest.mark.parametrize("model", list(DROPPED))
def test_finalize_names_missing_weights(cuda, model):
    report = _missing_report(cuda, model)
    assert report == _golden()["missing"][model]
    assert report.startswith("missing / mis-shaped weights: ")
    for key in DROPPED[model]:
        assert key in report
