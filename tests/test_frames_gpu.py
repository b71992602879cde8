"""GPU frame preprocessing (`vision_frames.process_frames_cuda`, lwm_vq_frames_prep) is bit-identical to the host path
(`vision_frames.process_frames`, Pillow) on the sweep of tests/test_frames_resample_cpu.py, from host arrays, host tensors
and device tensors, for one frame and for an odd clip length; and the VQGAN codes of GPU-preprocessed frames equal those
of host-preprocessed frames, including at size=64 against the fixture made by the reference's own `_process_frame`, up to
the near-ties that two encodes of the same pixels can also split (`_assert_same_codes`)."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from test_frames_resample_cpu import CONTENT, SIZES, make_frame

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "process_frame_reference.npz")
T_CLIP = 37


def _clip(w, h):
    """T_CLIP frames: random content, with one frame of every other kind of the sweep at the start"""
    frames = [make_frame(w, h, c) for c in CONTENT if c != "random"]
    frames += [make_frame(w, h, "random", seed=s) for s in range(T_CLIP - len(frames))]
    return np.stack(frames)


@pytest.mark.parametrize("w,h", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_gpu_frames_equal_pillow(w, h):
    from lwm_b200.vision_frames import process_frames, process_frames_cuda
    clip = _clip(w, h)
    ref = torch.from_numpy(process_frames([Image.fromarray(f) for f in clip]))
    dev = torch.from_numpy(clip).cuda()
    for got in (process_frames_cuda(clip), process_frames_cuda(torch.from_numpy(clip)), process_frames_cuda(dev)):
        assert got.is_cuda and got.dtype == torch.float32 and tuple(got.shape) == (T_CLIP, 256, 256, 3)
        assert torch.equal(got.cpu(), ref)
    for t in range(4):                       # T = 1: one frame of each content kind, from the host and the device
        assert torch.equal(process_frames_cuda(clip[t:t + 1]).cpu(), ref[t:t + 1])
        assert torch.equal(process_frames_cuda(dev[t:t + 1]).cpu(), ref[t:t + 1])


@pytest.mark.parametrize("size", [64, 63])
def test_gpu_frames_equal_pillow_at_other_sizes(size):
    from lwm_b200.vision_frames import process_frames, process_frames_cuda
    for (w, h) in ((517, 300), (301, 777), (200, 150)):
        clip = np.stack([make_frame(w, h, "random", seed=s) for s in range(3)])
        ref = torch.from_numpy(process_frames([Image.fromarray(f) for f in clip], size))
        assert torch.equal(process_frames_cuda(clip, size).cpu(), ref)


def test_gpu_frames_on_a_side_stream_and_an_empty_clip():
    from lwm_b200.vision_frames import process_frames, process_frames_cuda
    clip = _clip(1280, 720)[:5]
    ref = torch.from_numpy(process_frames([Image.fromarray(f) for f in clip]))
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = process_frames_cuda(clip)
    s.synchronize()
    assert torch.equal(got.cpu(), ref)
    assert tuple(process_frames_cuda(clip[:0]).shape) == (0, 256, 256, 3)


def _small_vqgan(resolution):
    """the encoder of lwm/vqgan.py with two levels and one ResnetBlock per level (VQGAN() itself is fixed to the
    default config, like the reference's)"""
    from lwm_b200.vqgan import VQGANConfig, VQGANModel, init_params
    cfg = VQGANConfig(resolution=resolution, channel_mult=(1, 2), num_res_blocks=1)
    return VQGANModel(cfg, init_params(cfg, seed=5), device="cuda")


def _assert_same_codes(model, pixels, idx_a, idx_b):
    """The encoder's GroupNorm statistics are summed with float atomics in a run-dependent order, so two encodes of the
    SAME pixels can differ in the latent (by up to an fp16 rounding of the default mode's activation planes) and pick
    the other code of a near-tie. Codes must agree everywhere else: at least 99.9 %, and every disagreement a near-tie
    at the latent's accuracy, the bound tests/test_vqgan_gpu.py uses for this mode."""
    assert idx_a.shape == idx_b.shape
    bad = (idx_a != idx_b).reshape(-1).nonzero()[:, 0]
    assert bad.numel() <= 1e-3 * idx_a.numel(), bad.numel()
    if bad.numel():
        z = model.ops.conv_gn(model.encoder(pixels.contiguous()), model.p["quant_conv"]).reshape(-1, 64)[bad].double()
        emb = model.p["quantize"]["embeddings"].double()
        d = (z * z).sum(1, keepdim=True) + (emb * emb).sum(1)[None] - 2 * z @ emb.T
        a, b = idx_a.reshape(-1)[bad].long(), idx_b.reshape(-1)[bad].long()
        gap = (d.gather(1, a[:, None]) - d.gather(1, b[:, None])).abs()[:, 0]
        assert (gap <= 4e-3 * d.min(1).values.abs()).all(), gap.max()


def test_codes_from_gpu_frames_equal_codes_from_host_frames():
    from lwm_b200.vision_frames import process_frames, process_frames_cuda
    model = _small_vqgan(256)
    clip = _clip(1280, 720)[:6]
    host = process_frames([Image.fromarray(f) for f in clip])
    dev = process_frames_cuda(clip)
    assert torch.equal(dev.cpu(), torch.from_numpy(host))      # the encoder gets the same input either way
    _, idx_host = model.encode(host)
    _, idx_dev = model.encode(dev)
    assert tuple(idx_dev.shape) == (6, 128, 128)
    _assert_same_codes(model, dev, idx_dev, idx_host)


def test_codes_from_gpu_frames_equal_codes_from_the_reference_fixture():
    from lwm_b200.vision_frames import process_frames_cuda
    from test_next_rows2_cpu import _images
    gold = np.load(GOLD)
    ims = _images()
    dev = torch.cat([process_frames_cuda(np.asarray(im)[None], 64) for im in ims])
    ref = np.stack([gold["frame_%d" % i] for i in range(len(ims))])
    assert torch.equal(dev.cpu(), torch.from_numpy(ref))
    model = _small_vqgan(64)
    _assert_same_codes(model, dev, model.encode(dev)[1], model.encode(ref)[1])
