"""The fp16x2 convs at extreme activation magnitudes: input x 2^k, k in {-24, -16, -12, 0, 12, 16, 20}.

The convs that read the raw residual stream (Downsample, Upsample, the 1x1 shortcuts) put the activation into ONE fp16
plane. Without a scale such a plane overflows to inf above 65504 and goes subnormal (or to zero) below 2^-14, where the
reference's fp32 conv has neither limit. The plane is written in units of a power of two taken from |x|max, so the
result must stay finite and within the usual tolerance at every k (the bias is scaled with the input, so that it
does not hide the activation's rounding), and, with zero bias and no residual, scaling the input by 2^k must scale the
output by exactly 2^k, bit for bit (bf16x3 has fp32's exponent range and must too).
A ResnetBlock reads the raw input through its shortcut and silu(groupnorm(x)) through Conv_0. At k = -24 the group
variance (~2^-48) is far below eps = 1e-6, so GroupNorm no longer normalises: with beta = 0 the prepped values shrink to
about 3e-5, fp16's subnormal range, so that plane needs a scale as well. Inside the block the conv biases dominate
Conv_0's output, so the GroupNorm-prepped conv is also checked on its own, with zero conv bias."""
import zlib

import pytest
import torch

from helpers import rel_fro, to_np
from vqgan_layers import conv_ref

pytestmark = pytest.mark.gpu

KS = [-24, -16, -12, 0, 12, 16, 20]
# production raw-input convs that the default mode runs in the fp16x2 scheme: (Cin, Cout, k, stride, upsample, H)
RAW = {
    "downsample-128-at-256": (128, 128, 3, 2, False, 256),
    "upsample-512-at-32": (512, 512, 3, 1, True, 32),
    "shortcut-256-128-at-256": (256, 128, 1, 1, False, 256),
}
TOL = {"fp16x2": 6e-4, "bf16x3": 1e-4}


@pytest.fixture(scope="module")
def vr():
    from oracle import vqgan_ref
    return vqgan_ref


def _gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def _raw_case(vr, name, bias_scale=1.0):
    from lwm_b200.vqgan import PackedConv
    cin, cout, k, stride, up, H = RAW[name]
    g = _gen(name)
    x = torch.randn(2, H, H, cin, generator=g)
    p = vr._conv_p(g, k, cin, cout)
    p["bias"] *= bias_scale
    return x, p, PackedConv(p, torch.device("cuda")), stride, up


def _run(ops, x, pc, stride, up):
    y = ops.conv_gn(x.cuda(), pc, upsample=up, stride=stride)
    torch.cuda.synchronize()
    return y


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("name", list(RAW))
def test_raw_input_conv_at_magnitude(vr, name, k):
    from lwm_b200.vqgan import Ops
    x, p, pc, stride, up = _raw_case(vr, name, bias_scale=2.0 ** k)
    ops = Ops("fp16x2")
    s = 2 if up else 1
    assert ops.passes_for((x.shape[1] * s // stride) ** 2) == 2
    xk = x * 2.0 ** k
    y = _run(ops, xk, pc, stride, up)
    assert bool(torch.isfinite(y).all())
    xin = xk.double().repeat_interleave(2, dim=1).repeat_interleave(2, dim=2) if up else xk.double()
    err = rel_fro(to_np(y), conv_ref(xin, p["kernel"], p["bias"], stride).numpy())
    print("%s k=%d: rel err %.2e" % (name, k, err))
    assert err < TOL["fp16x2"]


@pytest.mark.parametrize("k", [k for k in KS if k != 0])
@pytest.mark.parametrize("mode", ["fp16x2", "bf16x3"])
@pytest.mark.parametrize("name", list(RAW))
def test_raw_input_conv_scales_exactly(vr, name, mode, k):
    """conv(2^k x) == 2^k conv(x) bit for bit (zero bias, no residual)"""
    from lwm_b200.vqgan import Ops
    x, p, pc, stride, up = _raw_case(vr, name, bias_scale=0.0)
    ops = Ops(mode)
    y0 = _run(ops, x, pc, stride, up)
    yk = _run(ops, x * 2.0 ** k, pc, stride, up)
    assert bool(torch.isfinite(yk).all())
    want = y0 * 2.0 ** k
    assert torch.equal(yk, want), "%d of %d elements differ" % (int((yk != want).sum()), yk.numel())


def _resnet_ref(vr, x, p):
    """ResnetBlock (oracle/vqgan_ref.py::resnet_block) in float64 with the tap-by-tap conv"""
    d = {k: {kk: vv.double() for kk, vv in v.items()} for k, v in p.items()}
    h = conv_ref(vr.silu(vr.group_norm(x.double(), d["GroupNorm_0"])), d["Conv_0"]["kernel"], d["Conv_0"]["bias"])
    h = conv_ref(vr.silu(vr.group_norm(h, d["GroupNorm_1"])), d["Conv_1"]["kernel"], d["Conv_1"]["bias"])
    return h + conv_ref(x.double(), d["Conv_2"]["kernel"], d["Conv_2"]["bias"])


@pytest.mark.parametrize("beta", ["random_beta", "zero_beta"])
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("mode", ["fp16x2", "bf16x3"])
def test_resnet_block_at_magnitude(vr, mode, k, beta):
    """ResnetBlock 128 -> 256 at 128x128 (the encoder's DownsamplingBlock_1.ResnetBlock_0)"""
    from lwm_b200 import vqgan as V
    g = _gen("resnet-128-256")
    x = torch.randn(2, 128, 128, 128, generator=g)
    p = vr._resnet_p(g, 128, 256)
    if beta == "zero_beta":
        p["GroupNorm_0"]["bias"].zero_()
        p["GroupNorm_1"]["bias"].zero_()
    xk = x * 2.0 ** k
    ops = V.Ops(mode)
    y = V.ResnetBlock(ops, xk.cuda(), V._pack_tree(p, torch.device("cuda")))
    torch.cuda.synchronize()
    assert bool(torch.isfinite(y).all())
    err = rel_fro(to_np(y), _resnet_ref(vr, xk, p).numpy())
    print("ResnetBlock %s %s k=%d: rel err %.2e" % (mode, beta, k, err))
    assert err < TOL[mode]


@pytest.mark.parametrize("beta", ["random_beta", "zero_beta"])
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("mode", ["fp16x2", "bf16x3"])
def test_groupnorm_conv_at_magnitude(vr, mode, k, beta):
    """silu(groupnorm(x 2^k)) -> conv 128 -> 256 at 128x128 (that ResnetBlock's Conv_0), zero conv bias"""
    from lwm_b200.vqgan import Ops, PackedConv
    g = _gen("gn-conv-128-256")
    x = torch.randn(2, 128, 128, 128, generator=g)
    gn = vr._gn_p(g, 128)
    if beta == "zero_beta":
        gn["bias"].zero_()
    p = vr._conv_p(g, 3, 128, 256)
    p["bias"].zero_()
    xk = x * 2.0 ** k
    y = Ops(mode).conv_gn(xk.cuda(), PackedConv(p, torch.device("cuda")),
                          gn={"scale": gn["scale"].cuda(), "bias": gn["bias"].cuda()})
    torch.cuda.synchronize()
    assert bool(torch.isfinite(y).all())
    a = vr.silu(vr.group_norm(xk.double(), {"scale": gn["scale"].double(), "bias": gn["bias"].double()}))
    err = rel_fro(to_np(y), conv_ref(a, p["kernel"], p["bias"]).numpy())
    print("GroupNorm conv %s %s k=%d: rel err %.2e" % (mode, beta, k, err))
    assert err < TOL[mode]
