"""The layer list of tests/vqgan_layers.py covers every convolution the default-config VQGAN runs: the model is traversed
on the CPU with an Ops stand-in that records each call instead of launching it. If the config, the module wiring or the
mixed-precision policy changes, this test fails until the GPU layer tests follow."""
import torch

from vqgan_layers import LAYERS, images_for, layer_id, out_hw, tiles_per_image


def _recording_ops():
    from lwm_b200 import vqgan as V

    class RecordingOps(V.Ops):
        """Ops with the C calls replaced: prep returns a description of its planes, conv / conv_cin3 record the call
        (with the scheme conv_gn chose) and return zeros of the output's shape."""

        def __init__(self):
            super().__init__("fp16x2")
            self.calls = []

        def gn_stats(self, x):
            raise AssertionError("fp16x2 traversal asked for statistics of a tensor: covered by the recorded convs")

        def prep(self, x, gn=None, upsample=False, cpad=None, n_pass=None):
            return ("planes", tuple(x.shape), gn is not None, upsample, n_pass or self.n_pass)

        def conv(self, planes, pc, stride=1, residual=None, clip=False, want_stats=False):
            _, (N, H, W, C), gn, up, n_pass = planes
            assert C == pc.cin
            self.calls.append(("gn_conv" if gn else "conv", C, pc.cout, pc.k, stride, up, H, W, residual is not None,
                               clip, want_stats, {1: "bf16", 2: "fp16x2", 3: "bf16x3"}[n_pass]))
            Ho, Wo = out_hw(H, W, stride, up)
            return torch.zeros(N, Ho, Wo, pc.cout)

        def conv_cin3(self, x, pc):
            N, H, W, C = x.shape
            self.calls.append(("cin3", C, pc.cout, pc.k, 1, False, H, W, False, False, False, "fp32"))
            return torch.zeros(N, H, W, pc.cout)

    return RecordingOps()


def test_layer_list_covers_every_conv_of_the_default_model():
    from lwm_b200.vqgan import VQGANConfig, VQGANModel, init_params
    cfg = VQGANConfig()
    model = VQGANModel(cfg, init_params(cfg), device="cpu")
    model.ops = ops = _recording_ops()
    g = torch.Generator().manual_seed(0)
    x = torch.rand(1, cfg.resolution, cfg.resolution, cfg.num_channels, generator=g) * 2 - 1
    h = ops.conv_gn(model.encoder(x), model.p["quant_conv"])
    assert tuple(h.shape) == (1, 16, 16, cfg.quantized_embed_dim)
    y = model.decoder(ops.conv_gn(torch.zeros(1, 16, 16, cfg.quantized_embed_dim), model.p["post_quant_conv"]))
    assert tuple(y.shape) == (1, cfg.resolution, cfg.resolution, cfg.num_channels)
    assert len(ops.calls) == 78
    missing = sorted({c for c in ops.calls if c not in LAYERS})
    assert not missing, "convs of the default model missing from tests/vqgan_layers.py: %s" % missing
    assert set(LAYERS) == set(ops.calls), "stale entries: %s" % sorted(set(LAYERS) - set(ops.calls))
    assert len(set(LAYERS)) == len(LAYERS) == len({layer_id(s) for s in LAYERS})


def test_layer_cases_cover_every_n_tile_and_fill_the_persistent_grid():
    """the GPU layer tests launch at least 2 x 132 tiles over at least two images, and their Cout values include every
    N-tile regime of the kernel"""
    couts = set()
    for kind, cin, cout, k, stride, up, H, W, res, clip, stats, scheme in LAYERS:
        if kind == "cin3":
            continue
        Ho, Wo = out_hw(H, W, stride, up)
        for sch in {scheme, "bf16x3"}:
            n = images_for(Ho, Wo, cout, sch)
            assert n >= 2 and n * tiles_per_image(Ho, Wo, cout, sch) >= 264
        couts.add(cout)
    assert {3, 64, 256, 512, 768} <= couts
