"""Test-side Hypertile for the fp32 oracle UNet: the reference's regrouping (`b (nh h nw w) c -> (b nh nw) (h w) c` and
back, extensions-builtin/hypertile/hypertile.py:302-311) in torch reshape / permute, wrapped around the oracle's attn1
modules. The permutation is pinned to the reference by tests/test_hypertile_cpu.py; oracle/ itself stays unchanged."""
import contextlib

import torch
import torch.nn.functional as F


def regroup(x, hp, wp, nh, nw):
    """[b, hp*wp, c] -> [b*nh*nw, (hp/nh)*(wp/nw), c], tiles in (nh, nw) order."""
    b, n, c = x.shape
    th, tw = hp // nh, wp // nw
    return x.reshape(b, nh, th, nw, tw, c).permute(0, 1, 3, 2, 4, 5).reshape(b * nh * nw, th * tw, c)


def ungroup(y, hp, wp, nh, nw):
    bt, t, c = y.shape
    b, th, tw = bt // (nh * nw), hp // nh, wp // nw
    return y.reshape(b, nh, nw, th, tw, c).permute(0, 1, 3, 2, 4, 5).reshape(b, hp * wp, c)


def tiled_attention_ref(qkv, H, D, hp, wp, nh, nw):
    """fp32 reference of sdxe_hypertile_attention: qkv [B, N, 3*H*D] -> [B, N, H*D]."""
    q, k, v = (regroup(t.float(), hp, wp, nh, nw) for t in qkv.split(H * D, dim=-1))
    bt, T, _ = q.shape
    q, k, v = (t.reshape(bt, T, H, D).transpose(1, 2) for t in (q, k, v))
    o = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(bt, T, H * D)
    return ungroup(o, hp, wp, nh, nw)


@contextlib.contextmanager
def hypertile_unet(unet, spec, rows_fn):
    """Tile the oracle UNet's attn1 layers while active. rows_fn(x) is called once per UNet forward (x: its input) and
    returns the rows
    (h', w', nh, nw, max_tiles) of every attn1 layer in execution order (hypertile.attn1_layers(spec)); a row with
    max_tiles == 0 is not tiled."""
    from sdwebui_b200.hypertile import attn1_layers

    mods = [unet.get_submodule(name) for name, _ in attn1_layers(spec)]
    state = {"rows": None, "i": 0}
    orig_unet_forward = unet.forward

    def unet_forward(*a, **k):
        state["rows"], state["i"] = rows_fn(a[0] if a else k["x"]), 0
        return orig_unet_forward(*a, **k)

    def wrap(mod):
        orig = mod.forward

        def fwd(x, context=None):
            hp, wp, nh, nw, mt = state["rows"][state["i"]]
            state["i"] += 1
            if mt == 0 or nh * nw == 1:
                return orig(x, context)
            return ungroup(orig(regroup(x, hp, wp, nh, nw), context), hp, wp, nh, nw)

        return orig, fwd

    saved = []
    for m in mods:
        orig, fwd = wrap(m)
        saved.append((m, orig))
        m.forward = fwd
    unet.forward = unet_forward
    try:
        yield
    finally:
        unet.forward = orig_unet_forward
        for m, orig in saved:
            m.forward = orig
