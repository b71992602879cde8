"""Every distinct convolution call of the default-config VQGAN encoder and decoder (lwm_b200/vqgan.py with
VQGANConfig() defaults), and the float64 helpers the layer tests compare the kernels with.

A call is identified by (kind, Cin, Cout, k, stride, upsample, H, W, residual, clip, want_stats, scheme):
  kind    'cin3' (lwm_vq_conv_cin3, the 3-channel conv_in), 'gn_conv' (silu(groupnorm(x)) -> conv) or 'conv' (the conv
          reads the raw activation: Downsample, Upsample, the 1x1 shortcuts, quant/post_quant, the decoder's conv_in)
  H, W    the INPUT resolution; scheme is the one the default mixed 'fp16x2' mode assigns ('fp32' for conv_in).
tests/test_vqgan_layer_shapes_cpu.py checks that this list is complete; tests/test_vqgan_layers_gpu.py runs every entry
at production size."""
import math

import torch
import torch.nn.functional as F

LAYERS = [
    ("cin3", 3, 128, 3, 1, False, 256, 256, False, False, False, "fp32"),
    ("gn_conv", 128, 128, 3, 1, False, 256, 256, False, False, True, "fp16x2"),
    ("gn_conv", 128, 128, 3, 1, False, 256, 256, True, False, True, "fp16x2"),
    ("conv", 128, 128, 3, 2, False, 256, 256, False, False, True, "fp16x2"),
    ("gn_conv", 128, 256, 3, 1, False, 128, 128, False, False, True, "fp16x2"),
    ("conv", 128, 256, 1, 1, False, 128, 128, False, False, False, "fp16x2"),
    ("gn_conv", 256, 256, 3, 1, False, 128, 128, True, False, True, "fp16x2"),
    ("gn_conv", 256, 256, 3, 1, False, 128, 128, False, False, True, "fp16x2"),
    ("conv", 256, 256, 3, 2, False, 128, 128, False, False, True, "fp16x2"),
    ("gn_conv", 256, 256, 3, 1, False, 64, 64, False, False, True, "fp16x2"),
    ("gn_conv", 256, 256, 3, 1, False, 64, 64, True, False, True, "fp16x2"),
    ("conv", 256, 256, 3, 2, False, 64, 64, False, False, True, "bf16x3"),
    ("gn_conv", 256, 512, 3, 1, False, 32, 32, False, False, True, "bf16x3"),
    ("conv", 256, 512, 1, 1, False, 32, 32, False, False, False, "bf16x3"),
    ("gn_conv", 512, 512, 3, 1, False, 32, 32, True, False, True, "bf16x3"),
    ("gn_conv", 512, 512, 3, 1, False, 32, 32, False, False, True, "bf16x3"),
    ("conv", 512, 512, 3, 2, False, 32, 32, False, False, True, "bf16x3"),
    ("gn_conv", 512, 768, 3, 1, False, 16, 16, False, False, True, "bf16x3"),
    ("conv", 512, 768, 1, 1, False, 16, 16, False, False, False, "bf16x3"),
    ("gn_conv", 768, 768, 3, 1, False, 16, 16, True, False, True, "bf16x3"),
    ("gn_conv", 768, 768, 3, 1, False, 16, 16, False, False, True, "bf16x3"),
    ("gn_conv", 768, 64, 3, 1, False, 16, 16, False, False, False, "bf16x3"),
    ("conv", 64, 64, 1, 1, False, 16, 16, False, False, False, "bf16x3"),
    ("conv", 64, 768, 3, 1, False, 16, 16, False, False, True, "bf16x3"),
    ("conv", 768, 768, 3, 1, True, 16, 16, False, False, True, "bf16x3"),
    ("gn_conv", 768, 512, 3, 1, False, 32, 32, False, False, True, "bf16x3"),
    ("conv", 768, 512, 1, 1, False, 32, 32, False, False, False, "bf16x3"),
    ("conv", 512, 512, 3, 1, True, 32, 32, False, False, True, "fp16x2"),
    ("gn_conv", 512, 256, 3, 1, False, 64, 64, False, False, True, "fp16x2"),
    ("conv", 512, 256, 1, 1, False, 64, 64, False, False, False, "fp16x2"),
    ("conv", 256, 256, 3, 1, True, 64, 64, False, False, True, "fp16x2"),
    ("conv", 256, 256, 3, 1, True, 128, 128, False, False, True, "fp16x2"),
    ("gn_conv", 256, 128, 3, 1, False, 256, 256, False, False, True, "fp16x2"),
    ("conv", 256, 128, 1, 1, False, 256, 256, False, False, False, "fp16x2"),
    ("gn_conv", 128, 3, 3, 1, False, 256, 256, False, True, False, "fp16x2"),
]

H100_SMS = 132


def layer_id(sig):
    kind, cin, cout, k, stride, up, H, W, res, clip, stats, scheme = sig
    return "%s-%d-%d-k%d%s%s-%dx%d%s%s%s-%s" % (kind, cin, cout, k, "-s2" if stride == 2 else "", "-up" if up else "",
                                               H, W, "-res" if res else "", "-clip" if clip else "",
                                               "-stats" if stats else "", scheme)


def out_hw(H, W, stride, up):
    s = 2 if up else 1
    return H * s // stride, W * s // stride


def n_tile_width(cout, scheme):
    """the conv kernel's N tile (lwm_vq_conv2d[_f16]): fp16x2 the largest multiple of 16 <= 128 dividing Cout_pad,
    the bf16 schemes the widest power of two <= 256 dividing it (PackedConv's padding rule)"""
    cout_pad = -(-cout // 16) * 16
    if cout_pad > 256:
        cout_pad = -(-cout // 128) * 128
    if scheme == "fp16x2":
        return cout_pad, max(d for d in range(16, 129, 16) if cout_pad % d == 0)
    return cout_pad, max(d for d in (16, 32, 64, 128, 256) if cout_pad % d == 0)


def tiles_per_image(Ho, Wo, cout, scheme):
    cout_pad, bn = n_tile_width(cout, scheme)
    return (Ho // 8) * (Wo // 16) * (cout_pad // bn)


def images_for(Ho, Wo, cout, scheme, min_tiles=2 * H100_SMS):
    """enough images that the persistent grid (one CTA per SM) gives every CTA at least two tiles, and at least two
    images, so that some CTA's contiguous tile range crosses an image boundary (and an N-tile boundary when there is
    more than one N tile)"""
    return max(2, math.ceil(min_tiles / tiles_per_image(Ho, Wo, cout, scheme)))


def conv_ref(x, kernel, bias, stride=1):
    """flax nn.Conv in float64, x [N,H,W,Cin], kernel HWIO: SAME padding for stride 1, the Downsample's bottom/right pad
    + VALID for stride 2. Evaluated tap by tap as shifted 1x1 products, one image at a time, so that a 256x256x256 conv
    needs a few hundred MB rather than a full im2col."""
    x = x.double()
    w = kernel.double()
    k = w.shape[0]
    N, H, W, cin = x.shape
    cout = w.shape[3]
    if stride == 1:
        p = k // 2
        xp = F.pad(x, (0, 0, p, p, p, p))
        Ho, Wo = H, W
    else:
        xp = F.pad(x, (0, 0, 0, 1, 0, 1))
        Ho, Wo = H // 2, W // 2
    out = bias.double().expand(N, Ho, Wo, cout).clone()
    for n in range(N):
        for kh in range(k):
            for kw in range(k):
                xs = xp[n, kh:kh + stride * Ho:stride, kw:kw + stride * Wo:stride, :]
                out[n] += (xs.reshape(-1, cin) @ w[kh, kw]).reshape(Ho, Wo, cout)
    return out


def plane_scale(x):
    """power-of-two scale of an fp16 operand plane read without GroupNorm: 2^(e-12), e the exponent of |x|max"""
    m = float(x.abs().max())
    return 2.0 ** (math.frexp(m)[1] - 1 - 12) if m > 0 else 1.0


def round_f16_scaled(x, s=1.0):
    """x rounded like the fp16 plane that holds x / s"""
    return (x.double() / s).to(torch.float16).double() * s


def stats_of(y, groups=32):
    """float64 (sum, sum of squares) per (image, group) of y [N,H,W,C]"""
    N, H, W, C = y.shape
    yg = y.double().reshape(N, H * W, groups, C // groups)
    return torch.stack([yg.sum(dim=(1, 3)), (yg * yg).sum(dim=(1, 3))], dim=-1)
