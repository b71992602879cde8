"""Host side of the H100 VQGAN tokenizer — mirrors the reference's public surface
(lwm/vqgan.py): `VQGAN(vqgan_checkpoint, replicate=False).encode(pixel_values)` ->
(quantized_states, codebook_indices), `.decode(encoding)` -> pixels in [-1, 1], `VQGANConfig`
defaults (vqgan.py:62-77), and the sub-modules north_star names (`ResnetBlock`, `Downsample`,
`Upsample`, `VectorQuantizer`) as functions over flax-named parameter sub-trees.

NHWC fp32 activations and the flax parameter tree ({'encoder': {'Conv_0': {'kernel' HWIO, 'bias'},
'DownsamplingBlock_i': {'ResnetBlock_j': {'GroupNorm_0','Conv_0','GroupNorm_1','Conv_1',['Conv_2']},
'Downsample_0': {'Conv_0'}}, ...}, 'quantize': {'embeddings'}, 'quant_conv', 'post_quant_conv'}) are kept;
weights are re-packed once into the conv kernel's layout ([tap][Cout_pad][Cin_pad] bf16 hi/lo).

All arithmetic happens in liblwm_b200.so (include/lwm_b200.h: lwm_vq_*). torch only owns memory.
precision (the reference computes these convs in fp32):
  'fp16x2' (default)  activation = one fp16 plane, weights split hi + lo (two fp16) stacked along Cout so that one wide
                      wgmma does both halves; GroupNorm statistics come out of the producing conv's epilogue. Within
                      1e-3 end-to-end relative error on the encoder latents, 2x the algorithmic tensor work.
  'bf16x3'            both operands split into two bf16, three MMAs: fp32-class accuracy (1e-5), 3x the tensor work.
  'bf16'              single pass (≈1e-2 end-to-end relative error, 99.6 % code agreement on synthetic weights).

Under torch.use_deterministic_algorithms(True), every mode runs the ordered entry points (lwm_vq_*_ordered): GroupNorm
statistics summed in a fixed order and one fp16 plane scale per image, so that a frame's latents, codes and pixels are
the same bits on every run and whatever batch or video it is encoded in.
"""
import contextlib
import pickle

import numpy as np
import torch

from . import _lib

GN_GROUPS, GN_EPS = 32, 1e-6   # flax nn.GroupNorm() defaults
# 'fp16x2' is a MIXED mode: convs with at least this many output pixels per frame (the 64x64 .. 256x256 levels: 85 % of
# the encoder's FLOPs and bytes) run the 2-MMA fp16 scheme, the small deep layers keep the 3-MMA split-bf16 scheme.
# Measured with the oracle's operand-rounding emulation (DESIGN.md §4): 6.7e-4 (encode) / 5.9e-4 (decode) end-to-end
# relative error, against 8.9e-4 / 8.8e-4 with every layer on the 2-MMA scheme — margin under the 1e-3 bound.
MIXED_MIN_PIXELS = 64 * 64


class VQGANConfig:
    """Defaults of lwm/vqgan.py:62-77."""

    def __init__(self, resolution=256, num_channels=3, hidden_channels=128, channel_mult=(1, 2, 2, 4, 6),
                 num_res_blocks=2, attn_resolutions=(), no_attn_mid_block=True, z_channels=64, num_embeddings=8192,
                 quantized_embed_dim=64, dropout=0.0, resample_with_conv=True, commitment_cost=0.25):
        self.resolution = resolution
        self.num_channels = num_channels
        self.hidden_channels = hidden_channels
        self.channel_mult = tuple(channel_mult)
        self.num_res_blocks = num_res_blocks
        self.attn_resolutions = tuple(attn_resolutions)
        self.no_attn_mid_block = no_attn_mid_block
        self.z_channels = z_channels
        self.num_embeddings = num_embeddings
        self.quantized_embed_dim = quantized_embed_dim
        self.dropout = dropout
        self.resample_with_conv = resample_with_conv
        self.commitment_cost = commitment_cost
        self.num_resolutions = len(self.channel_mult)
        if self.attn_resolutions or not self.no_attn_mid_block:
            raise NotImplementedError("AttnBlock is disabled in every LWM VQGAN config (vqgan.py:69-70)")
        if not self.resample_with_conv:
            raise NotImplementedError("resample_with_conv=False (avg-pool) is unused by LWM")

    @classmethod
    def get_default_config(cls, updates=None):
        return cls(**(updates or {}))


def init_params(config=None, seed=0, codebook="normal"):
    """Random parameters in the flax tree layout of lwm/vqgan.py (for synthetic benchmarks; real use loads the
    pickled checkpoint). Conv kernels HWIO ~ N(0, 1/(k^2 Cin)), GroupNorm scale 1 / bias 0 perturbed by N(0, 0.02),
    codebook N(0,1) or the reference initialiser U(-1/n_e, 1/n_e) (vqgan.py:198-200)."""
    cfg = config or VQGANConfig.get_default_config()
    g = torch.Generator().manual_seed(seed)

    def conv(k, cin, cout):
        return {"kernel": torch.randn(k, k, cin, cout, generator=g) * (1.0 / (k * k * cin) ** 0.5),
                "bias": torch.randn(cout, generator=g) * 0.02}

    def gn(c):
        return {"scale": 1.0 + 0.02 * torch.randn(c, generator=g), "bias": 0.02 * torch.randn(c, generator=g)}

    def resnet(cin, cout):
        p = {"GroupNorm_0": gn(cin), "Conv_0": conv(3, cin, cout), "GroupNorm_1": gn(cout), "Conv_1": conv(3, cout, cout)}
        if cin != cout:
            p["Conv_2"] = conv(1, cin, cout)
        return p

    hc, mult, nres, nlev = cfg.hidden_channels, cfg.channel_mult, cfg.num_res_blocks, cfg.num_resolutions
    enc = {"Conv_0": conv(3, cfg.num_channels, hc)}
    cin = hc
    for i in range(nlev):
        blk = {}
        for j in range(nres):
            blk["ResnetBlock_%d" % j] = resnet(cin, hc * mult[i])
            cin = hc * mult[i]
        if i != nlev - 1:
            blk["Downsample_0"] = {"Conv_0": conv(3, cin, cin)}
        enc["DownsamplingBlock_%d" % i] = blk
    enc["MidBlock_0"] = {"ResnetBlock_0": resnet(cin, cin), "ResnetBlock_1": resnet(cin, cin)}
    enc["GroupNorm_0"] = gn(cin)
    enc["Conv_1"] = conv(3, cin, cfg.z_channels)
    ctop = hc * mult[-1]
    dec = {"Conv_0": conv(3, cfg.z_channels, ctop),
           "MidBlock_0": {"ResnetBlock_0": resnet(ctop, ctop), "ResnetBlock_1": resnet(ctop, ctop)}}
    cin = ctop
    for n, i in enumerate(reversed(range(nlev))):      # UpsamplingBlock_0 <=> block_idx nlev-1 (vqgan.py:179-180)
        blk = {}
        for j in range(nres + 1):
            blk["ResnetBlock_%d" % j] = resnet(cin, hc * mult[i])
            cin = hc * mult[i]
        if i != 0:
            blk["Upsample_0"] = {"Conv_0": conv(3, cin, cin)}
        dec["UpsamplingBlock_%d" % n] = blk
    dec["GroupNorm_0"] = gn(cin)
    dec["Conv_1"] = conv(3, cin, cfg.num_channels)
    n_e, e_dim = cfg.num_embeddings, cfg.quantized_embed_dim
    emb = torch.randn(n_e, e_dim, generator=g) if codebook == "normal" else (torch.rand(n_e, e_dim, generator=g) * 2 - 1) / n_e
    return {"encoder": enc, "decoder": dec, "quantize": {"embeddings": emb},
            "quant_conv": conv(1, cfg.z_channels, e_dim), "post_quant_conv": conv(1, e_dim, cfg.z_channels)}


def _pad_to(n, m):
    return (n + m - 1) // m * m


def _f32(t, dev):
    return torch.as_tensor(np.asarray(t), dtype=torch.float32).to(dev).contiguous()


class PackedConv:
    """One flax nn.Conv re-packed for lwm_vq_conv2d (done once at load time)."""

    def __init__(self, p, dev):
        w = _f32(p["kernel"], dev)                      # HWIO
        self.k, _, self.cin, self.cout = w.shape
        self.bias = _f32(p["bias"], dev)
        self.cpad = _pad_to(self.cin, 64)
        self.cout_pad = _pad_to(self.cout, 16)
        if self.cout_pad > 256:
            self.cout_pad = _pad_to(self.cout, 128)
        wt = w.permute(0, 1, 3, 2).reshape(self.k * self.k, self.cout, self.cin)   # [tap][Cout][Cin]
        full = torch.zeros(self.k * self.k, self.cout_pad, self.cpad, dtype=torch.float32, device=dev)
        full[:, :self.cout, :self.cin] = wt
        self.w_hi = full.to(torch.bfloat16).contiguous()
        self.w_lo = (full - self.w_hi.float()).to(torch.bfloat16).contiguous()
        self.w_hwio = w                                  # kept for the Cin=3 CUDA-core path
        # fp16x2 mode: w * 2^k = hi + lo (two fp16; k puts |w|max in [2^12, 2^13) so that lo stays a normal fp16),
        # stacked per N tile of BN output channels: [taps][Cout_pad/BN][hi rows | lo rows][Cpad]
        wmax = float(full.abs().max())
        k = 12 - int(np.floor(np.log2(wmax))) if wmax > 0 else 0
        self.w_scale_inv = float(2.0 ** -k)
        sc = full * float(2.0 ** k)
        hi16 = sc.to(torch.float16)
        lo16 = (sc - hi16.float()).to(torch.float16)
        self.bn = max(d for d in range(16, 129, 16) if self.cout_pad % d == 0)   # same rule as lwm_vq_conv2d_f16
        taps, nt = self.k * self.k, self.cout_pad // self.bn
        self.w_stack = torch.cat([hi16.view(taps, nt, self.bn, self.cpad), lo16.view(taps, nt, self.bn, self.cpad)],
                                 dim=2).contiguous()


class Ops:
    """Thin typed wrappers over the C ABI (every method allocates its outputs with torch)."""

    def __init__(self, precision="fp16x2"):
        if precision not in ("fp16x2", "bf16x3", "bf16"):
            raise ValueError("precision must be 'fp16x2', 'bf16x3' or 'bf16'")
        self.n_pass = {"fp16x2": 2, "bf16x3": 3, "bf16": 1}[precision]
        # None: follow torch.are_deterministic_algorithms_enabled() at each call; VQGANModel pins it for one
        # encode / decode, so that a producer conv and its consumer prep agree on the statistics and scale formats
        self.ordered = None

    def _ordered(self):
        return torch.are_deterministic_algorithms_enabled() if self.ordered is None else self.ordered

    def gn_stats(self, x):
        N, H, W, C = x.shape
        st = torch.empty(N, GN_GROUPS, 2, dtype=torch.float64, device=x.device)
        if self._ordered():
            ws = torch.empty(N * -(-H * W // 128) * GN_GROUPS * 2, dtype=torch.float32, device=x.device)
            _lib.call("lwm_vq_gn_stats_ordered", _lib.ptr(x), _lib.ptr(st), _lib.ptr(ws), ws.numel() * 4, N, H, W, C,
                      GN_GROUPS, _lib.stream_ptr())
            return st
        _lib.call("lwm_vq_gn_stats", _lib.ptr(x), _lib.ptr(st), N, H, W, C, GN_GROUPS, _lib.stream_ptr())
        return st

    def passes_for(self, out_pixels):
        """MMA scheme of one conv: 1 bf16, 2 fp16 activation x stacked fp16 hi|lo weights, 3 split-bf16"""
        if self.n_pass != 2:
            return self.n_pass
        return 2 if out_pixels >= MIXED_MIN_PIXELS else 3

    def conv_gn(self, x, pc, gn=None, upsample=False, stride=1, residual=None, clip=False, want_stats=False):
        """[GroupNorm + SiLU ->] [nearest 2x ->] conv: operand preparation and conv with the scheme the mode assigns to
        this layer."""
        s = 2 if upsample else 1
        n_pass = self.passes_for((x.shape[1] * s // stride) * (x.shape[2] * s // stride))
        return self.conv(self.prep(x, gn, upsample, n_pass=n_pass), pc, stride=stride, residual=residual, clip=clip,
                         want_stats=want_stats)

    def prep(self, x, gn=None, upsample=False, cpad=None, n_pass=None):
        """-> (hi, lo) operand planes [N,H',W',Cpad]: bf16 hi (+ bf16 lo), or one fp16 plane (n_pass 2);
        gn = flax GroupNorm params or None."""
        n_pass = n_pass or self.n_pass
        N, H, W, C = x.shape
        cpad = cpad or _pad_to(C, 64)
        s = 2 if upsample else 1
        st = g = b = None
        if gn is not None:
            # the producing conv's epilogue may already have accumulated this tensor's statistics (fp16x2 mode)
            st = getattr(x, "_gn_stats", None)
            if st is None:
                st = self.gn_stats(x)
            g, b = gn["scale"], gn["bias"]
        if n_pass == 2:
            # the plane holds y / s for a power of two s (device float, hi._plane_scale) that keeps it finite and normal
            # without GroupNorm, |x|max comes from the producing conv's epilogue when it computed one
            hi = torch.empty(N, H * s, W * s, cpad, dtype=torch.float16, device=x.device)
            amax = getattr(x, "_absmax_bits", None) if gn is None else None
            if self._ordered():       # one scale per image: hi._plane_scale [N]
                sc = torch.empty(2, N, dtype=torch.float32, device=x.device)   # [s, |x|max workspace] per image
                if amax is not None and amax.numel() != N:
                    amax = None
                _lib.call("lwm_vq_prep_f16_ordered", _lib.ptr(x), _lib.ptr(st), _lib.ptr(g), _lib.ptr(b), _lib.ptr(hi),
                          _lib.ptr(sc[0]), _lib.ptr(sc[1] if amax is None else amax), int(amax is not None), N, H, W, C,
                          cpad, GN_GROUPS, int(upsample), GN_EPS, _lib.stream_ptr())
                hi._plane_scale = sc[0]
                return hi, None
            if amax is not None and amax.numel() != 1:
                amax = None
            sc = torch.empty(2, dtype=torch.float32, device=x.device)        # [s, |x|max workspace]
            _lib.call("lwm_vq_prep_f16", _lib.ptr(x), _lib.ptr(st), _lib.ptr(g), _lib.ptr(b), _lib.ptr(hi), _lib.ptr(sc),
                      _lib.ptr(sc[1:] if amax is None else amax), int(amax is not None), N, H, W, C, cpad, GN_GROUPS,
                      int(upsample), GN_EPS, _lib.stream_ptr())
            hi._plane_scale = sc[:1]
            return hi, None
        hi = torch.empty(N, H * s, W * s, cpad, dtype=torch.bfloat16, device=x.device)
        lo = torch.empty_like(hi) if n_pass == 3 else None
        _lib.call("lwm_vq_prep", _lib.ptr(x), _lib.ptr(st), _lib.ptr(g), _lib.ptr(b), _lib.ptr(hi), _lib.ptr(lo),
                  N, H, W, C, cpad, GN_GROUPS, int(upsample), GN_EPS, _lib.stream_ptr())
        return hi, lo

    def conv(self, planes, pc, stride=1, residual=None, clip=False, want_stats=False):
        """want_stats: the output feeds a GroupNorm (or a raw fp16 plane) — have the epilogue accumulate its statistics
        and its |max| (fp16x2 mode)."""
        hi, lo = planes
        N, Hin, Win, cpad = hi.shape
        assert cpad == pc.cpad, (cpad, pc.cpad)
        Ho, Wo = Hin // stride, Win // stride
        pad = (pc.k // 2) if stride == 1 else 0
        out = torch.empty(N, Ho, Wo, pc.cout, dtype=torch.float32, device=hi.device)
        n_pass = 2 if hi.dtype == torch.float16 else (3 if lo is not None else 1)
        if n_pass == 2 and self._ordered():
            return self._conv_f16_ordered(hi, pc, stride, pad, residual, out, clip, want_stats)
        if n_pass == 2:
            a_scale = getattr(hi, "_plane_scale", None)
            if a_scale is not None and a_scale.numel() != 1:
                raise ValueError("this fp16 plane has one scale per image (prepared under "
                                 "torch.use_deterministic_algorithms): it needs the ordered conv")
            st = amax = None
            if want_stats:         # |out|max too: the scale of a raw fp16 plane of this tensor (Downsample, shortcut)
                # one zero-filled buffer: [N, groups, 2] float64 statistics, then the |max| bit pattern
                buf = torch.zeros(N * GN_GROUPS * 2 + 1, dtype=torch.float64, device=hi.device)
                amax = buf[-1:].view(torch.int32)[:1]
                if pc.cout % 16 == 0 and pc.cout % GN_GROUPS == 0 and (pc.cout // GN_GROUPS) % 4 == 0:
                    st = buf[:-1].view(N, GN_GROUPS, 2)
            _lib.call("lwm_vq_conv2d_f16", _lib.ptr(hi), _lib.ptr(a_scale),
                      _lib.ptr(pc.w_stack), _lib.ptr(pc.bias), _lib.ptr(residual), _lib.ptr(out), _lib.ptr(st),
                      _lib.ptr(amax), N, Hin, Win, cpad, Ho, Wo, pc.cout, pc.cout_pad, pc.k, stride, pad,
                      pc.w_scale_inv, GN_GROUPS, int(clip), _lib.stream_ptr())
            if st is not None:
                out._gn_stats = st
            if amax is not None:
                out._absmax_bits = amax
            return out
        _lib.call("lwm_vq_conv2d", _lib.ptr(hi), _lib.ptr(lo), _lib.ptr(pc.w_hi),
                  _lib.ptr(pc.w_lo if n_pass == 3 else None), _lib.ptr(pc.bias), _lib.ptr(residual),
                  _lib.ptr(out), N, Hin, Win, cpad, Ho, Wo, pc.cout, pc.cout_pad, pc.k, stride, pad, n_pass,
                  int(clip), _lib.stream_ptr())
        return out

    def _conv_f16_ordered(self, hi, pc, stride, pad, residual, out, clip, want_stats):
        """the fp16x2 conv with a scale per image and GroupNorm statistics summed in a fixed order"""
        N, Hin, Win, cpad = hi.shape
        _, Ho, Wo, _ = out.shape
        a_scale = getattr(hi, "_plane_scale", None)
        if a_scale is not None and a_scale.numel() != N:      # one scale for the whole batch is one per image too
            a_scale = a_scale.expand(N).contiguous()
        st = ws = amax = None
        if want_stats:
            amax = torch.empty(N, dtype=torch.int32, device=hi.device)      # zeroed by the call
            cpg = pc.cout // GN_GROUPS
            if pc.cout % 16 == 0 and pc.cout % GN_GROUPS == 0 and (cpg == 4 or (cpg % 8 == 0 and pc.bn % cpg == 0)):
                st = torch.empty(N, GN_GROUPS, 2, dtype=torch.float64, device=hi.device)
                ws = torch.empty(N * (Ho // 8) * (Wo // 16) * 8 * GN_GROUPS * 2, dtype=torch.float32, device=hi.device)
        _lib.call("lwm_vq_conv2d_f16_ordered", _lib.ptr(hi), _lib.ptr(a_scale), _lib.ptr(pc.w_stack), _lib.ptr(pc.bias),
                  _lib.ptr(residual), _lib.ptr(out), _lib.ptr(st), _lib.ptr(ws), 0 if ws is None else ws.numel() * 4,
                  _lib.ptr(amax), N, Hin, Win, cpad, Ho, Wo, pc.cout, pc.cout_pad, pc.k, stride, pad, pc.w_scale_inv,
                  GN_GROUPS, int(clip), _lib.stream_ptr())
        if st is not None:
            out._gn_stats = st
        if amax is not None:
            out._absmax_bits = amax
        return out

    def conv_cin3(self, x, pc):
        N, H, W, C = x.shape
        assert C == 3 and pc.k == 3
        out = torch.empty(N, H, W, pc.cout, dtype=torch.float32, device=x.device)
        _lib.call("lwm_vq_conv_cin3", _lib.ptr(x), _lib.ptr(pc.w_hwio), _lib.ptr(pc.bias), _lib.ptr(out), N, H, W,
                  pc.cout, _lib.stream_ptr())
        return out

    def vq_argmin(self, z_flat, emb, want_zq=True):
        N, D = z_flat.shape
        idx = torch.empty(N, dtype=torch.int32, device=z_flat.device)
        zq = torch.empty_like(z_flat) if want_zq else None
        ws = torch.empty(8 * N * 2, dtype=torch.float32, device=z_flat.device)
        _lib.call("lwm_vq_argmin", _lib.ptr(z_flat), _lib.ptr(emb), _lib.ptr(idx), _lib.ptr(zq), _lib.ptr(ws), N,
                  emb.shape[0], D, _lib.stream_ptr())
        return zq, idx

    def vq_gather(self, idx_flat, emb):
        out = torch.empty(idx_flat.numel(), emb.shape[1], dtype=torch.float32, device=emb.device)
        _lib.call("lwm_vq_gather", _lib.ptr(idx_flat), _lib.ptr(emb), _lib.ptr(out), idx_flat.numel(), emb.shape[0],
                  emb.shape[1], _lib.stream_ptr())
        return out


def _pack_tree(p, dev):
    """flax param tree -> same tree with PackedConv / fp32 GroupNorm leaves."""
    if "kernel" in p:
        return PackedConv(p, dev)
    if "scale" in p and "bias" in p and len(p) == 2:
        return {"scale": _f32(p["scale"], dev), "bias": _f32(p["bias"], dev)}
    if "embeddings" in p:
        return {"embeddings": _f32(p["embeddings"], dev)}
    return {k: _pack_tree(v, dev) for k, v in p.items()}


# ---- the reference's modules, as functions over packed parameter sub-trees -------------------------
def ResnetBlock(ops, x, p):
    """lwm/vqgan.py:242-263: GN -> SiLU -> Conv3x3 -> GN -> SiLU -> Conv3x3 (+ 1x1 shortcut) + residual."""
    h = ops.conv_gn(x, p["Conv_0"], gn=p["GroupNorm_0"], want_stats=True)
    res = ops.conv_gn(x, p["Conv_2"]) if "Conv_2" in p else x
    return ops.conv_gn(h, p["Conv_1"], gn=p["GroupNorm_1"], residual=res, want_stats=True)


def Downsample(ops, x, p):
    """lwm/vqgan.py:286-303: zero-pad bottom/right, 3x3 stride-2 VALID conv."""
    return ops.conv_gn(x, p["Conv_0"], stride=2, want_stats=True)


def Upsample(ops, x, p):
    """lwm/vqgan.py:306-319: nearest 2x then 3x3 SAME conv (the resize is fused into the operand prep)."""
    return ops.conv_gn(x, p["Conv_0"], upsample=True, want_stats=True)


def VectorQuantizer(ops, z, p, encoding_indices=None):
    """lwm/vqgan.py:187-221. z [..., 64] fp32 -> (z + sg(z_q - z), indices int32); or a lookup."""
    emb = p["embeddings"]
    if encoding_indices is not None:
        idx = encoding_indices.to(torch.int32).contiguous()
        return ops.vq_gather(idx.reshape(-1), emb).reshape(tuple(idx.shape) + (emb.shape[1],))
    flat = z.reshape(-1, z.shape[-1]).contiguous()
    zq, idx = ops.vq_argmin(flat, emb)
    return zq.reshape(z.shape), idx.reshape(z.shape[:-1])


class VQGANModel:
    """lwm/vqgan.py:105-146 on packed parameters."""

    def __init__(self, config, params, device="cuda", precision="fp16x2"):
        self.config = config
        self.device = torch.device(device)
        self.ops = Ops(precision)
        self.p = _pack_tree(params, self.device)

    def encoder(self, x):
        cfg, p, ops = self.config, self.p["encoder"], self.ops
        assert x.shape[1] == x.shape[2] == cfg.resolution, tuple(x.shape)   # vqgan.py:154
        h = ops.conv_cin3(x, p["Conv_0"]) if x.shape[-1] == 3 else ops.conv_gn(x, p["Conv_0"], want_stats=True)
        for i in range(cfg.num_resolutions):
            blk = p["DownsamplingBlock_%d" % i]
            for j in range(cfg.num_res_blocks):
                h = ResnetBlock(ops, h, blk["ResnetBlock_%d" % j])
            if i != cfg.num_resolutions - 1:
                h = Downsample(ops, h, blk["Downsample_0"])
        h = ResnetBlock(ops, h, p["MidBlock_0"]["ResnetBlock_0"])
        h = ResnetBlock(ops, h, p["MidBlock_0"]["ResnetBlock_1"])
        return ops.conv_gn(h, p["Conv_1"], gn=p["GroupNorm_0"])

    def decoder(self, z):
        cfg, p, ops = self.config, self.p["decoder"], self.ops
        h = ops.conv_gn(z, p["Conv_0"], want_stats=True)
        h = ResnetBlock(ops, h, p["MidBlock_0"]["ResnetBlock_0"])
        h = ResnetBlock(ops, h, p["MidBlock_0"]["ResnetBlock_1"])
        for n, i in enumerate(reversed(range(cfg.num_resolutions))):
            blk = p["UpsamplingBlock_%d" % n]
            for j in range(cfg.num_res_blocks + 1):
                h = ResnetBlock(ops, h, blk["ResnetBlock_%d" % j])
            if i != 0:
                h = Upsample(ops, h, blk["Upsample_0"])
        return ops.conv_gn(h, p["Conv_1"], gn=p["GroupNorm_0"], clip=True)   # clip(-1,1): vqgan.py:141

    @contextlib.contextmanager
    def _order_pinned(self):
        """reads torch.are_deterministic_algorithms_enabled() once for the whole call (the ordered path: DESIGN.md §4)"""
        prev = getattr(self.ops, "ordered", None)
        self.ops.ordered = torch.are_deterministic_algorithms_enabled()
        try:
            yield
        finally:
            self.ops.ordered = prev

    def encode(self, pixel_values):
        with self._order_pinned():
            return self._encode(pixel_values)

    def decode(self, encoding, is_codebook_indices=True):
        with self._order_pinned():
            return self._decode(encoding, is_codebook_indices)

    def _encode(self, pixel_values):
        x = self._to_dev(pixel_values)
        T = None
        if x.dim() == 5:   # video [B,T,H,W,C] (vqgan.py:118-121)
            T = x.shape[1]
            x = x.reshape((-1,) + tuple(x.shape[2:]))
        h = self.encoder(x.contiguous())
        h = self.ops.conv_gn(h, self.p["quant_conv"])
        zq, idx = VectorQuantizer(self.ops, h, self.p["quantize"])
        if T is not None:
            zq = zq.reshape((-1, T) + tuple(zq.shape[1:]))
            idx = idx.reshape((-1, T) + tuple(idx.shape[1:]))
        return zq, idx

    def _decode(self, encoding, is_codebook_indices):
        enc = torch.as_tensor(encoding).to(self.device)
        z = VectorQuantizer(self.ops, None, self.p["quantize"], enc) if is_codebook_indices else enc.float()
        T = None
        if z.dim() == 5:
            T = z.shape[1]
            z = z.reshape((-1,) + tuple(z.shape[2:]))
        h = self.ops.conv_gn(z.contiguous(), self.p["post_quant_conv"])
        y = self.decoder(h)
        if T is not None:
            y = y.reshape((-1, T) + tuple(y.shape[1:]))
        return y

    def _to_dev(self, x):
        if not torch.cuda.is_available():
            raise _lib.LwmError("VQGAN needs an sm_90 GPU: lwm_b200 has no CPU fallback")
        return torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).to(self.device, torch.float32)


class VQGAN:
    """Drop-in for lwm/vqgan.py:14-56. `vqgan_checkpoint` is a path to the pickled flax params (as in the reference) or
    an already loaded param tree. replicate=True is the reference's `jax.pmap` branch (vqgan.py:20-28) in the
    process-per-GPU model: the LEADING axis of the argument is mapped over the ranks of `group` (default WORLD) —
    rank r computes slice [r] with its replicated weights and the per-rank results are all-gathered, so every rank
    returns the full [n_ranks, ...] result, like pmap's output. Frames are independent: no other collective."""

    def __init__(self, vqgan_checkpoint, replicate=False, precision="fp16x2", device=None, group=None):
        assert vqgan_checkpoint != '' and vqgan_checkpoint is not None
        self.replicate = replicate
        self.group = group
        self.config = VQGANConfig.get_default_config()
        if isinstance(vqgan_checkpoint, (str, bytes)):
            with open(vqgan_checkpoint, "rb") as f:
                self.params = pickle.load(f)
        else:
            self.params = vqgan_checkpoint
        if device is None:
            device = "cuda:%d" % torch.cuda.current_device() if torch.cuda.is_available() else "cuda"
        self.model = VQGANModel(self.config, self.params, device, precision)

    def _pmap(self, fn, x):
        import torch.distributed as dist
        world, rank = 1, 0
        if dist.is_available() and dist.is_initialized():
            world, rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        x = torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x)
        if x.shape[0] != world:
            raise ValueError("replicate=True maps the leading axis over the %d rank(s) of the group (jax.pmap semantics, "
                             "lwm/vqgan.py:27-28): got leading axis %d" % (world, x.shape[0]))
        outs = fn(x[rank])
        single = not isinstance(outs, tuple)
        outs = (outs,) if single else outs
        full = []
        for o in outs:
            o = o.contiguous()
            if world == 1:
                full.append(o[None])
                continue
            g = torch.empty((world * o.shape[0],) + tuple(o.shape[1:]), dtype=o.dtype, device=o.device)
            dist.all_gather_into_tensor(g, o, group=self.group)      # concatenated along dim 0 (gloo and NCCL agree)
            full.append(g.view((world,) + tuple(o.shape)))
        return full[0] if single else tuple(full)

    def encode(self, pixel_values):
        if self.replicate:
            return self._pmap(self.model.encode, pixel_values)
        return self.model.encode(pixel_values)

    def decode(self, encoding):
        if self.replicate:
            return self._pmap(self.model.decode, encoding)
        return self.model.decode(encoding)
