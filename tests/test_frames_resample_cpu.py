"""Frame preprocessing on the GPU (lwm_vq_frames_prep) runs Pillow's 8-bit bicubic resize as integer arithmetic over
coefficient tables built on the host (lwm_b200.vision_frames.pass_tables / frame_geometry). Checked here without a GPU:
the tables, driven through oracle/frames_resample.py's numpy restatement of the kernel's two integer passes, equal
Pillow (`vision_frames.process_frames`) bit for bit on down- and upscaling, crop-only inputs, crop edges on .5, odd sizes
and content that drives the bicubic lobes into the clip; and the C entry point validates its arguments before it looks
for a device."""
import ctypes
import os

import numpy as np
import pytest
import torch
from PIL import Image

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "process_frame_reference.npz")

# (width, height)
SIZES = [(640, 360), (1280, 720), (1920, 1080), (3840, 2160), (360, 640), (300, 300), (200, 150), (255, 255),
         (456, 256), (455, 256), (457, 256), (1279, 719)]
CONTENT = ["random", "zeros", "full", "checker"]


def make_frame(w, h, content, seed=0):
    if content == "random":
        return np.random.default_rng(seed + w * 7 + h).integers(0, 256, (h, w, 3), dtype=np.uint8)
    if content == "zeros":
        return np.zeros((h, w, 3), np.uint8)
    if content == "full":
        return np.full((h, w, 3), 255, np.uint8)
    return np.repeat((np.indices((h, w)).sum(0) % 2 * 255).astype(np.uint8)[..., None], 3, 2)   # 1-pixel checkerboard


@pytest.mark.parametrize("content", CONTENT)
@pytest.mark.parametrize("w,h", SIZES, ids=["%dx%d" % s for s in SIZES])
def test_integer_passes_equal_pillow(w, h, content):
    from lwm_b200.vision_frames import process_frames
    from oracle.frames_resample import process_frame
    a = make_frame(w, h, content)
    ref = process_frames([Image.fromarray(a)])[0]
    got = process_frame(a)
    assert got.dtype == np.float32 and got.shape == ref.shape == (256, 256, 3)
    assert np.array_equal(got.view(np.int32), ref.view(np.int32))


@pytest.mark.parametrize("w,h", [(1280, 720), (517, 300), (301, 777), (200, 150)])
@pytest.mark.parametrize("size", [64, 63])
def test_integer_passes_equal_pillow_at_other_sizes(w, h, size):
    """size is a parameter of the reference; an odd size can make PIL's rounded crop box one column or row off"""
    from lwm_b200.vision_frames import process_frames
    from oracle.frames_resample import process_frame
    a = make_frame(w, h, "random", seed=size)
    ref = process_frames([Image.fromarray(a)], size)[0]
    got = process_frame(a, size)
    assert got.shape == ref.shape and np.array_equal(got, ref)


def test_integer_passes_equal_the_reference_fixture():
    """the fixture was made by the reference's own `_process_frame` at size=64"""
    from oracle.frames_resample import process_frame
    from test_next_rows2_cpu import _images
    gold = np.load(GOLD)
    for i, im in enumerate(_images()):
        assert np.array_equal(process_frame(np.asarray(im), 64), gold["frame_%d" % i])


def test_geometry_and_table_shapes():
    from lwm_b200.vision_frames import frame_geometry, pass_tables
    assert frame_geometry(256, 455) == (455, 256, 100, 0, 256, 256)      # left edge 99.5 -> 100
    assert frame_geometry(256, 457) == (457, 256, 100, 0, 256, 256)      # left edge 100.5 -> 100
    assert frame_geometry(720, 1280) == (455, 256, 100, 0, 256, 256)
    assert frame_geometry(640, 360) == (256, 455, 0, 100, 256, 256)
    assert frame_geometry(256, 456) == (456, 256, 100, 0, 256, 256)      # crop only
    assert pass_tables(720, 256)[1].shape == (256, 13)
    assert pass_tables(2160, 256)[1].shape == (256, 35)
    assert pass_tables(150, 256)[1].shape == (256, 5)                   # upscaling: support 2, not scaled
    b, k = pass_tables(256, 256)                                        # a pass that keeps the size: the identity
    assert np.array_equal(b[:, 0], np.arange(256)) and (b[:, 1] == 1).all() and (k == 1 << 22).all()
    for n_in, n_out in ((1280, 455), (720, 256), (150, 256), (3840, 455)):
        b, k = pass_tables(n_in, n_out)
        assert (b[:, 0] >= 0).all() and (b[:, 0] + b[:, 1] <= n_in).all() and (b[:, 1] <= k.shape[1]).all()
        assert (np.diff(b[:, 0]) >= 0).all()
        assert (k[np.arange(k.shape[1])[None, :] >= b[:, 1:2]] == 0).all()
        assert (np.abs(k.sum(1) - (1 << 22)) <= k.shape[1]).all()       # each row sums to 1 up to the rounding


# ---- argument validation of the C entry point, without a GPU ----
P = ctypes.c_void_p(0x1000)      # fake non-null pointer: nothing dereferences it before the device check
N = None
SHAPE, ARG, DEVICE = 2, 3, 1
GOOD = (P, 16, 720, 1280, 3, P, P, 455, 13, P, P, 256, 13, 100, 0, 256, 256, P, N)


def _with(**kw):
    names = ["frames", "T", "H", "W", "C", "xb", "xk", "out_w", "kx", "yb", "yk", "out_h", "ky", "left", "top",
             "crop_w", "crop_h", "out", "stream"]
    args = list(GOOD)
    for k, v in kw.items():
        args[names.index(k)] = v
    return tuple(args)


BAD = [
    (_with(frames=N), ARG, "null"),
    (_with(yk=N), ARG, "null"),
    (_with(out=N), ARG, "null"),
    (_with(C=4), SHAPE, "3-channel"),
    (_with(C=1), SHAPE, "3-channel"),
    (_with(T=-1), SHAPE, "frame sizes"),
    (_with(H=0), SHAPE, "frame sizes"),
    (_with(kx=0), SHAPE, "tables"),
    (_with(out_h=0), SHAPE, "tables"),
    (_with(left=200), SHAPE, "crop window"),
    (_with(top=-1), SHAPE, "crop window"),
    (_with(crop_h=257), SHAPE, "crop window"),
    (_with(crop_w=0), SHAPE, "crop window"),
    (_with(H=100000, out_h=256, ky=1000, crop_w=256, W=100000), SHAPE, "shared memory"),
]


@pytest.mark.parametrize("args,code,frag", BAD, ids=["%s-%d" % (b[2].replace(" ", "_"), i) for i, b in enumerate(BAD)])
def test_frames_prep_rejects_bad_arguments(lib, args, code, frag):
    status = lib.lwm_vq_frames_prep(*args)
    msg = lib.lwm_last_error().decode()
    assert status == code, (status, msg)
    assert frag in msg, msg


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: only meaningful where the device check fails")
def test_frames_prep_well_formed_call_fails_with_device_error_without_gpu(lib):
    for args in (GOOD, _with(T=0)):
        assert lib.lwm_vq_frames_prep(*args) == DEVICE
        assert "no CPU fallback" in lib.lwm_last_error().decode() or "sm_90" in lib.lwm_last_error().decode()


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_process_frames_cuda_raises_without_gpu():
    from lwm_b200 import _lib
    from lwm_b200.vision_frames import process_frames_cuda
    with pytest.raises(_lib.LwmError):
        process_frames_cuda(np.zeros((1, 360, 640, 3), np.uint8))
