"""Test-side Tiling for the fp32 oracle models: a restatement of StableDiffusionModelHijack.apply_circular
(modules/sd_hijack.py:311-318) over the module tree that hijack() flattens (:254-261). Every nn.Conv2d gets
padding_mode 'circular' or 'zeros'; a padding-0 conv (the VAE encoder's Downsample after its constant pad) is unaffected by
the mode, as in the reference. Pinned to the reference's own code by tests/golden/tiling_ref.npz
(tests/golden/make_golden_tiling.py, checked in tests/test_tiling_cpu.py); oracle/ itself stays unchanged."""
import torch


def apply_circular(model: torch.nn.Module, enable: bool) -> None:
    for layer in model.modules():
        if type(layer) == torch.nn.Conv2d:  # noqa: E721  the reference's exact-type test: subclasses keep their mode
            layer.padding_mode = "circular" if enable else "zeros"


# seeded cases shared by the generator and the tests: (name, build(), inputs(generator) -> args, run(model, args))
def cases():
    from oracle.synth import init_module_
    from oracle.unet import UNetModel, tiny_config
    from oracle.vae import AutoencoderKLDecode, AutoencoderKLEncode, tiny_vae_config

    def unet(linear):
        cfg = tiny_config(linear=linear, adm=96 if linear else 0)
        return init_module_(UNetModel(cfg), 11).eval(), cfg

    def unet_case(linear, n, h, w, seed):
        def build():
            return unet(linear)[0]

        def inputs():
            cfg = unet(linear)[1]
            g = torch.Generator().manual_seed(seed)
            x = torch.randn(n, 4, h, w, generator=g)
            t = torch.rand(n, generator=g) * 999
            ctx = torch.randn(n, 77, cfg.context_dim, generator=g)
            y = torch.randn(n, cfg.adm_in_channels, generator=g) if cfg.adm_in_channels else None
            return x, t, ctx, y

        return build, inputs, lambda m, a: m(a[0], a[1], context=a[2], y=a[3])

    def dec_case(n, h, w, seed):
        def inputs():
            return (torch.randn(n, 4, h, w, generator=torch.Generator().manual_seed(seed)) * 3,)

        return (lambda: init_module_(AutoencoderKLDecode(tiny_vae_config()), 31).eval(), inputs, lambda m, a: m.decode(a[0]))

    def enc_case(n, h, w, seed):
        def inputs():
            return (torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(seed)) * 2 - 1,)

        return (lambda: init_module_(AutoencoderKLEncode(tiny_vae_config()), 33).eval(), inputs, lambda m, a: m.encode_moments(a[0]))

    return {
        "unet_conv": unet_case(False, 2, 8, 12, 1),
        "unet_linear_adm": unet_case(True, 1, 6, 10, 2),   # 3 x 5 after the Downsample: odd sides wrap through im2col
        "vae_decoder": dec_case(1, 6, 10, 3),
        "vae_encoder": enc_case(1, 12, 20, 4),
    }
