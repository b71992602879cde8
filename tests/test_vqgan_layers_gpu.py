"""Every convolution of the default-config VQGAN at production size, against float64 (tests/vqgan_layers.py).

Each case goes through Ops.conv_gn as VQGANModel dispatches it, with enough images that every CTA of the persistent
conv kernel runs several tiles and some CTA's tile range crosses an image (and N-tile) boundary: the stage ring, the
accumulator reset and the GroupNorm-statistics flush are exercised across tiles, which the small op tests of
test_vqgan_gpu.py never do. Non-square images pin the H/W bookkeeping; the standalone statistics and operand-prep
kernels run at the channel counts and resolutions where the model uses them.

Tolerances (relative Frobenius): fp16x2 <= 2e-5 against the same fp16 operand rounding in float64 and <= 6e-4 against
the unrounded result; bf16x3 <= 1e-4; epilogue statistics <= 1e-5 of their max against float64 sums of the output."""
import zlib

import pytest
import torch

from helpers import rel_fro, to_np
from vqgan_layers import (LAYERS, conv_ref, images_for, layer_id, out_hw, plane_scale, round_f16_scaled, stats_of)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vr():
    from oracle import vqgan_ref
    return vqgan_ref


def _pc(p):
    from lwm_b200.vqgan import PackedConv
    return PackedConv(p, torch.device("cuda"))


def _gn(p):
    return None if p is None else {"scale": p["scale"].cuda(), "bias": p["bias"].cuda()}


def _gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def _silu_gn64(vr, x, p):
    return vr.silu(vr.group_norm(x.double(), {"scale": p["scale"].double(), "bias": p["bias"].double()}))


def _up(a):
    return a.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)


def _check_stats(y):
    # |y|max from the same epilogue: the scale of a raw fp16 plane read from y
    assert y._absmax_bits.view(torch.float32).item() == y.abs().max().item()
    st = y._gn_stats.cpu()
    ref = stats_of(y.cpu())
    err = float((st - ref).abs().max() / ref.abs().max())
    assert err < 1e-5, err
    return err


CASES = [(s, "fp16x2") for s in LAYERS] + [(s, "bf16x3") for s in LAYERS if s[-1] == "fp16x2"]


@pytest.mark.parametrize("sig,mode", CASES, ids=["%s-mode_%s" % (layer_id(s), m) for s, m in CASES])
def test_production_layer(vr, sig, mode):
    from lwm_b200.vqgan import Ops
    kind, cin, cout, k, stride, up, H, W, res, clip, want_stats, scheme = sig
    ops = Ops(mode)
    g = _gen(layer_id(sig) + mode)
    p = vr._conv_p(g, k, cin, cout)
    pc = _pc(p)
    Ho, Wo = out_hw(H, W, stride, up)
    if kind == "cin3":
        x = torch.rand(2, H, W, cin, generator=g) * 2 - 1
        y = ops.conv_cin3(x.cuda(), pc)
        err = rel_fro(to_np(y), conv_ref(x, p["kernel"], p["bias"]).numpy())
        print("%s: rel err %.2e" % (layer_id(sig), err))
        assert err < 1e-5
        return
    used = scheme if mode == "fp16x2" else "bf16x3"
    assert {2: "fp16x2", 3: "bf16x3"}[ops.passes_for(Ho * Wo)] == used
    N = images_for(Ho, Wo, cout, used)
    x = torch.randn(N, H, W, cin, generator=g) * 1.3
    gnp = vr._gn_p(g, cin) if kind == "gn_conv" else None
    r = torch.randn(N, Ho, Wo, cout, generator=g) if res else None
    y = ops.conv_gn(x.cuda(), pc, gn=_gn(gnp), upsample=up, stride=stride, residual=None if r is None else r.cuda(),
                    clip=clip, want_stats=want_stats)
    torch.cuda.synchronize()
    assert tuple(y.shape) == (N, Ho, Wo, cout)
    a = _silu_gn64(vr, x, gnp) if gnp is not None else x.double()

    def conv64(a_in):
        out = conv_ref(_up(a_in) if up else a_in, p["kernel"], p["bias"], stride)
        if r is not None:
            out += r.double()
        return out.clamp(-1.0, 1.0) if clip else out

    got = to_np(y)
    err = rel_fro(got, conv64(a).numpy())
    msg = "%s mode %s, %d images: rel err %.2e" % (layer_id(sig), mode, N, err)
    if used == "fp16x2":
        # the plane of a raw activation is scaled by a power of two, a GroupNorm-prepped one is not (ordinary range)
        err16 = rel_fro(got, conv64(round_f16_scaled(a, 1.0 if gnp is not None else plane_scale(x))).numpy())
        msg += ", vs the same fp16 operand rounding %.2e" % err16
        assert err16 < 2e-5, msg
        assert err < 6e-4, msg
    else:
        assert err < 1e-4, msg
    if want_stats and used == "fp16x2":
        msg += ", statistics %.2e" % _check_stats(y)
    else:
        assert not hasattr(y, "_gn_stats")
    print(msg)


# ---- non-square images: the tile grid's H/W order, the TMA box dimensions and the stride-2 / upsample coordinates
@pytest.mark.parametrize("want_stats", [False, True], ids=["plain", "stats"])
@pytest.mark.parametrize("stride,up", [(1, False), (2, False), (1, True)], ids=["s1", "s2", "up"])
@pytest.mark.parametrize("H,W", [(64, 128), (128, 64)], ids=["64x128", "128x64"])
@pytest.mark.parametrize("mode", ["fp16x2", "bf16x3"])
def test_conv_non_square(vr, mode, H, W, stride, up, want_stats):
    from lwm_b200.vqgan import Ops
    g = _gen("nonsq%s%d%d%d%d" % (mode, H, W, stride, up))
    x = torch.randn(2, H, W, 128, generator=g) * 1.3
    p = vr._conv_p(g, 3, 128, 256)
    ops = Ops(mode)
    n_pass = 2 if mode == "fp16x2" else 3
    y = ops.conv(ops.prep(x.cuda(), upsample=up, n_pass=n_pass), _pc(p), stride=stride, want_stats=want_stats)
    torch.cuda.synchronize()
    Ho, Wo = out_hw(H, W, stride, up)
    assert tuple(y.shape) == (2, Ho, Wo, 256)
    xin = _up(x.double()) if up else x.double()
    got = to_np(y)
    err = rel_fro(got, conv_ref(xin, p["kernel"], p["bias"], stride).numpy())
    if n_pass == 2:
        err16 = rel_fro(got, conv_ref(round_f16_scaled(xin, plane_scale(x)), p["kernel"], p["bias"], stride).numpy())
        assert err16 < 2e-5 and err < 6e-4, (err16, err)
    else:
        assert err < 1e-4, err
    if want_stats and n_pass == 2:
        _check_stats(y)
        # a raw plane of y takes its scale from the epilogue's |y|max instead of another pass over y
        hi, _ = ops.prep(y, n_pass=2)
        s = plane_scale(y.cpu())
        assert float(hi._plane_scale) == s
        assert torch.equal(hi.cpu(), (y.cpu().double() / s).to(torch.float16))
    else:
        assert not hasattr(y, "_gn_stats")


@pytest.mark.parametrize("H,W", [(64, 128), (128, 64)], ids=["64x128", "128x64"])
def test_stats_and_prep_non_square(vr, H, W):
    from lwm_b200.vqgan import Ops
    g = _gen("prepnonsq%d%d" % (H, W))
    x = torch.randn(2, H, W, 256, generator=g) * 1.7 + 0.3
    p = vr._gn_p(g, 256)
    xd = x.cuda()
    st = Ops("bf16x3").gn_stats(xd)
    ref_st = stats_of(x)
    assert float((st.cpu() - ref_st).abs().max() / ref_st.abs().max()) < 1e-5
    ref = _silu_gn64(vr, x, p)
    hi, lo = Ops("bf16x3").prep(xd, _gn(p))
    assert rel_fro(to_np(hi) + to_np(lo), ref.numpy()) < 2e-5
    ops16 = Ops("fp16x2")
    for up in (False, True):
        hi, lo = ops16.prep(xd, _gn(p), upsample=up)
        assert lo is None and tuple(hi.shape) == (2, H << up, W << up, 256)
        assert float(hi._plane_scale) == 1.0
        assert rel_fro(to_np(hi), (_up(ref) if up else ref).numpy()) < 3e-4
        # without GroupNorm the plane is exactly fp16(x / s), s = 2^(e-12), e the exponent of |x|max
        hi, _ = ops16.prep(xd, upsample=up)
        s = plane_scale(x)
        assert float(hi._plane_scale) == s
        want = (x.double() / s).to(torch.float16)
        assert torch.equal(hi.cpu(), _up(want) if up else want)


# ---- standalone GroupNorm statistics and operand prep at the model's channel counts and resolutions
@pytest.mark.parametrize("C,H", [(128, 256), (128, 128), (256, 128), (256, 64), (256, 32), (512, 64), (512, 32),
                                 (512, 16), (768, 16)])
def test_stats_and_prep_production(vr, C, H):
    """inputs with a mean offset of 3 sigma (the fp32 fast variance E[x^2] - E[x]^2 stays accurate there)"""
    from lwm_b200.vqgan import Ops
    g = _gen("prep%d%d" % (C, H))
    sigma = 1.7
    x = torch.randn(2, H, H, C, generator=g) * sigma + 3 * sigma
    p = vr._gn_p(g, C)
    xd = x.cuda()
    st = Ops("bf16x3").gn_stats(xd)
    ref_st = stats_of(x)
    e_st = float((st.cpu() - ref_st).abs().max() / ref_st.abs().max())
    assert e_st < 1e-5, e_st
    ref = _silu_gn64(vr, x, p)
    hi, lo = Ops("bf16x3").prep(xd, _gn(p))
    e_hl = rel_fro(to_np(hi) + to_np(lo), ref.numpy())
    assert e_hl < 2e-5, e_hl
    ops16 = Ops("fp16x2")
    for up in (False, True):
        hi, _ = ops16.prep(xd, _gn(p), upsample=up)
        assert float(hi._plane_scale) == 1.0
        e16 = rel_fro(to_np(hi), (_up(ref) if up else ref).numpy())
        assert e16 < 3e-4, (up, e16)
    print("C %d @%d: stats %.2e, bf16 hi+lo %.2e, fp16 plane %.2e" % (C, H, e_st, e_hl, e16))
