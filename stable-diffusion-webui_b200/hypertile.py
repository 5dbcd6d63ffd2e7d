"""Hypertile for the engine UNet: the reference's built-in extension (extensions-builtin/hypertile/) re-implemented
against the engine's attn1 layers.

With Hypertile on, every hooked self-attention layer (`attn1`) of the UNet cuts its token sequence into nh x nw tiles and
attends inside each tile only; (nh, nw) is drawn per layer and per UNet call from one seeded `random.Random`. The
behaviour follows the reference exactly, including its quirks:
  * the token grid (h', w') is recovered from the token count and the image's W / H (`find_hw_candidates`), which
    transposes it for non-square images: the tiles are strided chunks of the row-major token sequence;
  * candidate tile counts need not be powers of two, and tiles need not be multiples of the kernels' row blocks;
  * every enabled layer draws on every UNet call (second-order sampler calls, cond / uncond sub-batches included), even
    when it has a single candidate; disabled layers draw nothing.

This module owns the host side: the layer / depth tables, the draw functions, the per-job configuration
(`HypertileOptions`, `configure`) and the per-call table of rows (h', w', nh, nw, max_tiles) that
`sdxe_unet_set_hypertile` takes. The tiling itself runs in the engine (gather + segmented attention, attention.cu).
"""
from __future__ import annotations

import math
import random
from dataclasses import dataclass
from functools import lru_cache
from typing import Dict, List, Optional, Tuple

# the draws of every Hypertile layer come from this one generator, seeded per job (extension script: process / before_hr)
RNG = random.Random()


def set_seed(seed: int) -> None:
    RNG.seed(seed)


@dataclass
class HypertileOptions:
    """The UNet settings of the Hypertile extension (scripts/hypertile_script.py:90-98), with their defaults."""

    enable_unet: bool = False             # hypertile_enable_unet
    enable_unet_secondpass: bool = False  # hypertile_enable_unet_secondpass
    max_depth_unet: int = 3               # hypertile_max_depth_unet
    max_tile_unet: int = 256              # hypertile_max_tile_unet
    swap_size_unet: int = 3               # hypertile_swap_size_unet


def _sd15_depths() -> Dict[str, int]:
    """SD1.5 (ldm names): the attn1 of both input and all three output transformer blocks of level l at depth l, the
    middle block at depth 3."""
    d = {}
    for level in range(3):
        for i in (3 * level + 1, 3 * level + 2):
            d[f"input_blocks.{i}.1.transformer_blocks.0.attn1"] = level
        for j in range(3 * (3 - level), 3 * (3 - level) + 3):
            d[f"output_blocks.{j}.1.transformer_blocks.0.attn1"] = level
    d["middle_block.1.transformer_blocks.0.attn1"] = 3
    return d


def _sdxl_depths() -> Dict[str, int]:
    """SDXL (ldm names): level 1's first transformer blocks at depth 0, its second ones and all of level 2 at depth 1,
    the middle block at depth 2; nothing at depth 3."""
    d = {}
    for k in range(2):
        for blk in ("input_blocks.4", "input_blocks.5", "output_blocks.3", "output_blocks.4", "output_blocks.5"):
            d[f"{blk}.1.transformer_blocks.{k}.attn1"] = k
    for k in range(10):
        for blk in ("input_blocks.7", "input_blocks.8", "output_blocks.0", "output_blocks.1", "output_blocks.2"):
            d[f"{blk}.1.transformer_blocks.{k}.attn1"] = 1
        d[f"middle_block.1.transformer_blocks.{k}.attn1"] = 2
    return d


DEPTHS_SD15 = _sd15_depths()
DEPTHS_SDXL = _sdxl_depths()


def layer_depth(name: str, is_sdxl: bool) -> Optional[int]:
    """Depth of the layer whose module name ends with a table entry (the reference matches with `endswith`), else None."""
    for entry, depth in (DEPTHS_SDXL if is_sdxl else DEPTHS_SD15).items():
        if name.endswith(entry):
            return depth
    return None


@lru_cache(maxsize=None)
def get_divisors(value: int, min_value: int, max_options: int = 1) -> List[int]:
    """Tile counts n = value / d for the divisors d >= min(min_value, value) of value, smallest d (largest n) first, at
    most max(1, max_options) of them."""
    lo = min(min_value, value)
    counts = [value // d for d in range(lo, value + 1) if value % d == 0]
    return counts[:max(1, max_options)]


def random_divisor(value: int, min_value: int, max_options: int = 1) -> int:
    """One of get_divisors(...), drawn from RNG (a draw happens even when there is a single candidate)."""
    counts = get_divisors(value, min_value, max_options)
    return counts[RNG.randint(0, len(counts) - 1)]


@lru_cache(maxsize=None)
def largest_tile_size_available(width: int, height: int) -> int:
    """Largest power of two dividing both image sides."""
    g = math.gcd(width, height)
    return g & -g if g else 1


def _closest_divisor_pair(hw: int, aspect_ratio: float) -> Tuple[int, int]:
    best = None
    for a in range(2, hw + 1):
        if hw % a == 0:
            err = abs((hw // a) / a - aspect_ratio)
            if best is None or err < best[0]:
                best = (err, a, hw // a)
    return best[1], best[2]


@lru_cache(maxsize=None)
def find_hw_candidates(hw: int, aspect_ratio: float) -> Tuple[int, int]:
    """(h', w') with h' * w' = hw from the token count and the image's W / H (note: h' follows W, w' follows H)."""
    h, w = round(math.sqrt(hw * aspect_ratio)), round(math.sqrt(hw / aspect_ratio))
    if h * w == hw:
        return h, w
    if (hw / h).is_integer():
        return h, hw // h
    if (hw / w).is_integer():
        return hw // w, w
    return _closest_divisor_pair(hw, aspect_ratio)


def attn1_layers(spec) -> List[Tuple[str, int]]:
    """(ldm module name, UNet level) of every attn1 layer of an engine UNet (engine.UNetSpec), in execution order: the
    order of the engine's table rows and of the stock modules' calls."""
    out = []
    nl, td = len(spec.channel_mult), spec.transformer_depth
    idx = 1
    for level in range(nl):
        for _ in range(spec.num_res_blocks):
            out += [(f"input_blocks.{idx}.1.transformer_blocks.{k}.attn1", level) for k in range(td[level])]
            idx += 1
        idx += level != nl - 1
    out += [(f"middle_block.1.transformer_blocks.{k}.attn1", nl - 1) for k in range(max(1, spec.middle_depth))]
    idx = 0
    for level in reversed(range(nl)):
        for _ in range(spec.num_res_blocks + 1):
            out += [(f"output_blocks.{idx}.1.transformer_blocks.{k}.attn1", level) for k in range(td[level])]
            idx += 1
    return out


def level_tokens(h: int, w: int, levels: int) -> List[int]:
    """Token count of each UNet level for an h x w latent (each Downsample halves a side, rounding up)."""
    out = []
    for _ in range(levels):
        out.append(h * w)
        h, w = (h + 1) // 2, (w + 1) // 2
    return out


@dataclass
class LayerState:
    """What the reference's hook keeps per layer (HypertileParams), for one job configuration."""

    name: str
    level: int
    depth: Optional[int]  # None: not in the table, never tiled
    enabled: bool
    tile_size: int
    swap_size: int
    aspect_ratio: float


class HypertileState:
    """Hypertile configured for one image size (hypertile_hook_model): per layer its depth and settings; per call the
    table for sdxe_unet_set_hypertile."""

    def __init__(self, levels: int, layers: List[LayerState]):
        self.levels = levels
        self.layers = layers
        self.enabled = any(l.enabled for l in layers)

    def structure(self, h: int, w: int) -> List[Tuple[int, int, Optional[int], bool]]:
        """(h', w', depth, enabled) per attn1 layer for an h x w latent."""
        tokens = level_tokens(h, w, self.levels)
        return [find_hw_candidates(tokens[l.level], l.aspect_ratio) + (l.depth, l.enabled) for l in self.layers]

    def draw_rows(self, h: int, w: int, divisor=None, candidates=None) -> List[Tuple[int, int, int, int, int]]:
        """Rows (h', w', nh, nw, max_tiles) of one UNet call, drawing (nh, nw) for the enabled layers in execution order;
        disabled layers are (0, 0, 1, 1, 0) and draw nothing. `divisor` / `candidates` default to this module's
        random_divisor / find_hw_candidates (the webui passes its own hypertile module's)."""
        divisor = divisor or random_divisor
        candidates = candidates or find_hw_candidates
        tokens = level_tokens(h, w, self.levels)
        rows = []
        for l in self.layers:
            if not l.enabled:
                rows.append((0, 0, 1, 1, 0))
                continue
            hp, wp = candidates(tokens[l.level], l.aspect_ratio)
            if hp * wp != tokens[l.level]:
                raise ValueError(f"Hypertile: no {hp} x {wp} grid for {tokens[l.level]} tokens")
            lo = max(128, l.tile_size) // 8 * 2 ** l.depth
            nh = divisor(hp, lo, l.swap_size)
            nw = divisor(wp, lo, l.swap_size)
            rows.append((hp, wp, nh, nw, get_divisors(hp, lo, l.swap_size)[0] * get_divisors(wp, lo, l.swap_size)[0]))
        return rows


def configure(spec, width: int, height: int, opts: HypertileOptions, enable: bool, is_sdxl: bool) -> Optional[HypertileState]:
    """hypertile_hook_model for the UNet: None when no layer is enabled (the reference's hooks then draw nothing)."""
    tile_size = min(largest_tile_size_available(width, height), opts.max_tile_unet)
    layers = []
    for name, level in attn1_layers(spec):
        depth = layer_depth(name, is_sdxl)
        layers.append(LayerState(name, level, depth, bool(enable and depth is not None and depth <= opts.max_depth_unet),
                                 tile_size, opts.swap_size_unet, width / height))
    st = HypertileState(len(spec.channel_mult), layers)
    return st if st.enabled else None


def _unet_spec(p):
    unet = p.sd_model.unet
    return unet.spec if unet.spec is not None else unet.engine.spec


def begin_job(p) -> Optional[HypertileState]:
    """The extension's process(): seed with the job's first seed, configure for (width, height) with enable_unet."""
    set_seed(p.seeds[0])
    return configure(_unet_spec(p), p.width, p.height, p.hypertile, p.hypertile.enable_unet, p.sd_model.is_sdxl)


def begin_hr_pass(p, width: int, height: int) -> Optional[HypertileState]:
    """The extension's before_hr(): enable = secondpass or enable_unet; re-seed only when enabled."""
    o = p.hypertile
    enable = o.enable_unet_secondpass or o.enable_unet
    if enable:
        set_seed(p.seeds[0])
    return configure(_unet_spec(p), width, height, o, enable, p.sd_model.is_sdxl)


def webui_state(spec, model, cache: dict) -> Optional[HypertileState]:
    """Inside the webui: the state the Hypertile extension's hooks left on the stock UNet `model`
    (shared.sd_model.model, still present on the CPU while the engine runs): `__webui_hypertile_layers` on the model
    and `__webui_hypertile_params` on each hooked module. None when the hooks are absent or no layer is enabled.
    `cache` keeps the layer -> params mapping between calls (the hooks mutate the params objects in place)."""
    hooked = getattr(model, "__webui_hypertile_layers", None)
    if not hooked:
        return None
    key = (id(model), id(hooked), len(hooked))
    if cache.get("key") != key:
        params = {}
        for name in hooked:
            try:
                params[name] = getattr(model.get_submodule(name), "__webui_hypertile_params")
            except AttributeError:
                continue
        per_layer = []
        for ldm, level in attn1_layers(spec):
            prm = next((v for n, v in params.items() if n == ldm or n.endswith("." + ldm)), None)
            per_layer.append((ldm, level, prm))
        cache.clear()
        cache.update(key=key, layers=per_layer)
    layers = [LayerState(ldm, level, prm.depth if prm is not None else None, bool(prm is not None and prm.enabled),
                         prm.tile_size if prm is not None else 0, prm.swap_size if prm is not None else 0,
                         prm.aspect_ratio if prm is not None else 1.0) for ldm, level, prm in cache["layers"]]
    st = HypertileState(len(spec.channel_mult), layers)
    return st if st.enabled else None
