"""The VQGAN tokenizer under torch.use_deterministic_algorithms(True): GroupNorm statistics summed in a fixed order and
one fp16 plane scale per image (lwm_vq_*_ordered, DESIGN.md §4), default VQGANConfig, synthetic weights
(oracle/vqgan_ref.init_params), 256x256 frames.

  * repeatability: three encodes of a 16-frame clip give the same bits of the pre-quantisation latent, zq and codes,
    in fp16x2, bf16x3 and bf16; three decodes of 16 frames of codes give the same pixels (how many codes the flag-off
    path changed between runs is printed, not asserted);
  * batch invariance: every frame's latent and codes are the same bits encoded alone, in a 16-frame clip, in a
    shuffled clip and in a [2, 8, ...] video, with frames of widely different magnitudes, a constant frame and a NaN
    frame in the batch; likewise decode; and the raw-plane convs (Downsample, 1x1 shortcut) on images 2^20 apart;
  * the statistics: within fp32 resolution of a float64 sum, and the same bits for an image at N = 1 and N = 7, from
    the stand-alone pass and from the conv epilogue;
  * frames to codes: process_frames_cuda and the host process_frames give the same codes on a 1280x720 clip;
  * accuracy: the end-to-end parity bounds of tests/test_vqgan_gpu.py hold under the flag;
  * plumbing: with the flag off only the existing entry points run, with it on none of the three unordered ones."""
import numpy as np
import pytest
import torch

from helpers import rel_fro, to_np

pytestmark = pytest.mark.gpu
MODES = ["fp16x2", "bf16x3", "bf16"]
T = 16


@pytest.fixture
def deterministic():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


@pytest.fixture(scope="module")
def vr():
    from oracle import vqgan_ref
    return vqgan_ref


@pytest.fixture(scope="module")
def params(vr):
    return vr.init_params(seed=0, codebook="normal")


_MODELS = {}


def _model(params, mode):
    from lwm_b200.vqgan import VQGAN
    if mode not in _MODELS:
        _MODELS[mode] = VQGAN(params, precision=mode).model
    return _MODELS[mode]


def _clip(seed=11, nan=False):
    """16 frames in [-1, 1] of different kinds; with `nan`, frames of widely different magnitudes and one NaN pixel"""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(T, 256, 256, 3, generator=g) * 2 - 1
    x[1] = 0.3                                                         # constant frame
    x[2] = torch.linspace(-1, 1, 256)[None, :, None].expand(256, 256, 3)   # smooth ramp
    if nan:
        x[3] *= 2.0 ** -12
        x[4] *= 2.0 ** 8
        x[5] *= 2.0 ** -20
        x[6, 100, 37, 1] = float("nan")
    return x


def _encode(model, x):
    """(pre-quantisation latent, zq, codes) of frames x [n, 256, 256, 3] or a video [B, T, 256, 256, 3]"""
    x = x.cuda()
    zq, idx = model.encode(x)
    flat = x.reshape((-1,) + tuple(x.shape[-3:]))
    h = model.ops.conv_gn(model.encoder(flat.contiguous()), model.p["quant_conv"])
    torch.cuda.synchronize()
    n = flat.shape[0]
    return h.reshape(n, -1).cpu(), zq.reshape(n, -1).cpu(), idx.reshape(n, -1).cpu()


def _bits(t):
    return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t


def _same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


def _codes(seed):
    return torch.randint(0, 8192, (T, 16, 16), generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("mode", MODES)
def test_three_encodes_are_bit_identical(params, deterministic, mode):
    model = _model(params, mode)
    x = _clip()
    runs = [_encode(model, x) for _ in range(3)]
    for r in runs[1:]:
        for name, a, b in zip(("latent", "zq", "codes"), runs[0], r):
            assert _same_bits(a, b), "%s: %d of %d elements differ" % (name, int((_bits(a) != _bits(b)).sum()), a.numel())
    torch.use_deterministic_algorithms(False)
    free = [_encode(model, x)[2] for _ in range(3)]
    torch.use_deterministic_algorithms(True)
    print("%s, flag off: %d and %d of %d codes changed between runs; flag on: 0" % (
        mode, int((free[0] != free[1]).sum()), int((free[0] != free[2]).sum()), free[0].numel()))


@pytest.mark.parametrize("mode", MODES)
def test_three_decodes_are_bit_identical(params, deterministic, mode):
    model = _model(params, mode)
    codes = _codes(12)
    runs = [model.decode(codes).cpu() for _ in range(3)]
    for r in runs[1:]:
        assert _same_bits(runs[0], r), "%d of %d pixels differ" % (int((_bits(runs[0]) != _bits(r)).sum()), r.numel())


@pytest.mark.parametrize("mode", MODES)
def test_encode_is_batch_invariant(params, deterministic, mode):
    model = _model(params, mode)
    x = _clip(seed=13, nan=True)
    clip = _encode(model, x)
    perm = torch.randperm(T, generator=torch.Generator().manual_seed(1))
    shuffled = _encode(model, x[perm])
    video = _encode(model, x.reshape(2, T // 2, 256, 256, 3))
    for t in range(T):
        alone = _encode(model, x[t:t + 1])
        j = int((perm == t).nonzero())
        for name, k in (("latent", 0), ("codes", 2)) + ((("zq", 1),) if t != 6 else ()):
            want = alone[k][0]
            for way, got in (("clip", clip[k][t]), ("shuffled clip", shuffled[k][j]), ("video", video[k][t])):
                if t == 6 and name == "latent":      # the NaN frame: NaN bit patterns are not compared
                    assert torch.equal(torch.isnan(want), torch.isnan(got))
                    continue
                assert _same_bits(want, got), "frame %d %s: alone vs %s: %d elements differ" % (
                    t, name, way, int((_bits(want) != _bits(got)).sum()))
    assert all(bool(torch.isfinite(clip[0][t]).all()) for t in range(T) if t != 6)


@pytest.mark.parametrize("mode", MODES)
def test_decode_is_batch_invariant(params, deterministic, mode):
    model = _model(params, mode)
    codes = _codes(14)
    clip = model.decode(codes).cpu()
    perm = torch.randperm(T, generator=torch.Generator().manual_seed(2))
    shuffled = model.decode(codes[perm]).cpu()
    video = model.decode(codes.reshape(2, T // 2, 16, 16)).cpu().reshape(T, 256, 256, 3)
    for t in range(T):
        alone = model.decode(codes[t:t + 1]).cpu()[0]
        j = int((perm == t).nonzero())
        for way, got in (("clip", clip[t]), ("shuffled clip", shuffled[j]), ("video", video[t])):
            assert _same_bits(alone, got), "frame %d: alone vs %s" % (t, way)


RAW = {   # (Cin, Cout, k, stride, H): the raw-input convs of the encoder that run the fp16x2 scheme
    "downsample-128-at-256": (128, 128, 3, 2, 256),
    "shortcut-128-256-at-128": (128, 256, 1, 1, 128),
}


@pytest.mark.parametrize("name", list(RAW))
def test_raw_plane_conv_is_batch_invariant_across_magnitudes(vr, deterministic, name):
    """images 2^20 apart in scale in one batch: each image's output (and |max|) is the single-image result, bit for
    bit; the plane carries one scale per image"""
    from lwm_b200.vqgan import Ops, PackedConv
    cin, cout, k, stride, H = RAW[name]
    g = torch.Generator().manual_seed(len(name))
    x = torch.randn(3, H, H, cin, generator=g)
    x[1] *= 2.0 ** 20
    x[2] *= 2.0 ** -20
    pc = PackedConv(vr._conv_p(g, k, cin, cout), torch.device("cuda"))
    ops = Ops("fp16x2")
    assert ops.passes_for((H // stride) ** 2) == 2
    plane = ops.prep(x.cuda(), n_pass=2)
    assert tuple(plane[0]._plane_scale.shape) == (3,)
    y = ops.conv(plane, pc, stride=stride, want_stats=True)
    for i in range(3):
        yi = ops.conv(ops.prep(x[i:i + 1].cuda(), n_pass=2), pc, stride=stride, want_stats=True)
        assert _same_bits(yi[0].cpu(), y[i].cpu()), "image %d" % i
        assert int(yi._absmax_bits[0]) == int(y._absmax_bits[i])
        assert _same_bits(yi._gn_stats[0].cpu().view(torch.int64), y._gn_stats[i].cpu().view(torch.int64))
    assert bool(torch.isfinite(y).all())


def _stats_f64(y, groups=32):
    N, H, W, C = y.shape
    yg = y.double().reshape(N, H * W, groups, C // groups)
    ref = torch.stack([yg.sum(dim=(1, 3)), (yg * yg).sum(dim=(1, 3))], dim=-1)
    mag = torch.stack([yg.abs().sum(dim=(1, 3)), (yg * yg).sum(dim=(1, 3))], dim=-1)
    return ref, mag


def _check_stats(st, y):
    ref, mag = _stats_f64(y.cpu())
    err = float(((st.cpu() - ref).abs() / mag).max())
    print("ordered statistics vs float64: %.1e of the magnitude sum" % err)
    assert err < 1e-5


@pytest.mark.parametrize("C,H", [(128, 64), (512, 32), (768, 16)])
def test_standalone_statistics_are_exact_and_batch_invariant(deterministic, C, H):
    from lwm_b200.vqgan import Ops
    g = torch.Generator().manual_seed(C + H)
    x = (torch.randn(7, H, H, C, generator=g) + 0.5) * (2.0 ** torch.arange(-9, 12, 3.0))[:, None, None, None]
    ops = Ops("bf16x3")
    st = ops.gn_stats(x.cuda())
    _check_stats(st, x)
    for i in range(7):
        si = ops.gn_stats(x[i:i + 1].cuda())
        assert torch.equal(si[0].cpu().view(torch.int64), st[i].cpu().view(torch.int64)), i


@pytest.mark.parametrize("cin,cout,H", [(128, 128, 64), (128, 256, 64), (256, 512, 32)])
def test_epilogue_statistics_are_exact_and_batch_invariant(vr, deterministic, cin, cout, H):
    from lwm_b200.vqgan import Ops, PackedConv
    g = torch.Generator().manual_seed(cin + cout)
    x = torch.randn(7, H, H, cin, generator=g) * (2.0 ** torch.arange(-6, 8, 2.0))[:, None, None, None]
    pc = PackedConv(vr._conv_p(g, 3, cin, cout), torch.device("cuda"))
    ops = Ops("fp16x2")
    y = ops.conv(ops.prep(x.cuda(), n_pass=2), pc, want_stats=True)
    _check_stats(y._gn_stats, y)
    for i in range(7):
        yi = ops.conv(ops.prep(x[i:i + 1].cuda(), n_pass=2), pc, want_stats=True)
        assert _same_bits(yi[0].cpu(), y[i].cpu())
        assert torch.equal(yi._gn_stats[0].cpu().view(torch.int64), y._gn_stats[i].cpu().view(torch.int64)), i


def test_gpu_frames_and_host_frames_give_the_same_codes(params, deterministic):
    from PIL import Image
    from lwm_b200.vision_frames import process_frames, process_frames_cuda
    rng = np.random.default_rng(3)
    base = rng.integers(0, 256, (T, 90, 160, 3)).astype(np.uint8)
    clip = np.ascontiguousarray(np.repeat(np.repeat(base, 8, 1), 8, 2))        # 16 frames of 1280x720
    clip[:, ::3] = rng.integers(0, 256, clip[:, ::3].shape).astype(np.uint8)
    model = _model(params, "fp16x2")
    host = process_frames([Image.fromarray(f) for f in clip])
    dev = process_frames_cuda(clip)
    _, idx_host = model.encode(host)
    _, idx_dev = model.encode(dev)
    assert tuple(idx_dev.shape) == (T, 16, 16)
    assert torch.equal(idx_dev.cpu(), idx_host.cpu())


@pytest.mark.parametrize("mode,tol,agree,tie", [("fp16x2", 1e-3, 0.99, 4e-3), ("bf16x3", 1e-4, 0.999, 1e-4)])
def test_encode_parity_holds_under_the_flag(vr, params, deterministic, mode, tol, agree, tie):
    model = _model(params, mode)
    g = torch.Generator().manual_seed(11)
    x = torch.rand(1, 2, 256, 256, 3, generator=g) * 2 - 1
    zq, idx = model.encode(x.cuda())
    ref_zq, ref_idx, ref_h = vr.encode(x, params)
    h = model.ops.conv_gn(model.encoder(x.reshape(2, 256, 256, 3).cuda()), model.p["quant_conv"])
    err = rel_fro(to_np(h), ref_h)
    print("%s ordered encode latent rel err %.2e" % (mode, err))
    assert err < tol
    got = to_np(idx).astype(np.int32)
    assert (got == ref_idx).mean() >= agree
    emb = params["quantize"]["embeddings"].numpy()
    for b in np.argwhere(got != ref_idx):
        zrow = ref_h.reshape(-1, 64)[np.ravel_multi_index(tuple(b[1:]), (2, 16, 16))][None]
        d = vr.vq_distances_f32(zrow, emb)[0]
        assert abs(d[got[tuple(b)]] - d[ref_idx[tuple(b)]]) <= tie * max(1.0, abs(d.min()))


@pytest.mark.parametrize("mode,tol", [("fp16x2", 1e-3), ("bf16x3", 1e-4)])
def test_decode_parity_holds_under_the_flag(vr, deterministic, mode, tol):
    from lwm_b200.vqgan import VQGAN
    p1 = vr.init_params(seed=1, codebook="normal")
    codes = torch.randint(0, 8192, (1, 16, 16), generator=torch.Generator().manual_seed(12))
    y = VQGAN(p1, precision=mode).decode(codes)
    err = rel_fro(to_np(y), vr.decode(codes.numpy(), p1))
    print("%s ordered decode rel err %.2e" % (mode, err))
    assert float(y.abs().max()) <= 1.0 and err < tol


UNORDERED = {"lwm_vq_gn_stats", "lwm_vq_prep_f16", "lwm_vq_conv2d_f16"}
ORDERED = {"lwm_vq_gn_stats_ordered", "lwm_vq_prep_f16_ordered", "lwm_vq_conv2d_f16_ordered"}


@pytest.mark.parametrize("mode", MODES)
def test_entry_points_follow_the_flag(params, monkeypatch, mode):
    from lwm_b200 import _lib
    names, real = [], _lib.call

    def spy(name, *args):
        names.append(name)
        return real(name, *args)

    monkeypatch.setattr(_lib, "call", spy)
    model = _model(params, mode)
    x, codes = _clip()[:2], _codes(15)[:2]
    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(False)
        model.encode(x)
        model.decode(codes)
        off = set(names)
        names.clear()
        torch.use_deterministic_algorithms(True)
        model.encode(x)
        model.decode(codes)
        on = set(names)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert not off & ORDERED, off
    assert "lwm_vq_gn_stats" in off and ("lwm_vq_conv2d_f16" in off) == (mode == "fp16x2")
    assert not on & UNORDERED, on
    assert "lwm_vq_gn_stats_ordered" in on and ("lwm_vq_conv2d_f16_ordered" in on) == (mode == "fp16x2")
    assert on - ORDERED == off - UNORDERED          # everything else is the same launches
