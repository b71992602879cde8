"""Frame preprocessing in front of the VQGAN — host mirror of `Sampler._process_frame` (lwm/vision_chat.py:59-74; also
the resize/crop of lwm/vision_generation.py's input path): resize so that the SHORT side becomes `size` (PIL's default
resampling, aspect ratio kept, the long side truncated to int), crop the central size x size window, scale uint8
[0,255] to float32 [-1,1] (x / 127.5 - 1). The reference does this on the host with PIL; so does this mirror — the
result is the `pixel_values` tensor `VQGAN.encode` takes (vision_chat.py:89-100).

`process_frames_cuda` computes the same tensor, bit for bit, on the GPU (lwm_vq_frames_prep): Pillow's 8-bit bicubic
resampling is integer fixed-point arithmetic, and `pass_tables` builds its coefficient tables here exactly as Pillow
does."""
import math

import numpy as np

PRECISION_BITS = 22          # Pillow's 8-bit resampling: 32 - 8 - 2 fractional bits per coefficient
BICUBIC_SUPPORT = 2.0


def process_frame(image, size=256):
    """image: PIL.Image -> float32 array [size, size, C] in [-1, 1]"""
    width, height = image.size
    if width < height:
        new_size = (size, int(size * height / width))
    else:
        new_size = (int(size * width / height), size)
    image = image.resize(new_size)
    left, top = (new_size[0] - size) / 2, (new_size[1] - size) / 2
    image = image.crop((left, top, left + size, top + size))
    return np.array(image, dtype=np.float32) / 127.5 - 1


def process_frames(images, size=256):
    """a list of PIL images (the frames of a clip, or one still image) -> float32 [T, size, size, C]"""
    return np.stack([process_frame(im, size) for im in images])


def frame_geometry(height, width, size=256):
    """The resize and crop `process_frame` applies to a width x height image: (new_w, new_h, left, top, crop_w, crop_h).
    The crop box is PIL's: float edges rounded with Python's round (half to even), e.g. a resized width of 455 puts the
    left edge at 99.5 -> 100 and 457 at 100.5 -> 100. crop_w, crop_h == size unless size is odd."""
    if width < height:
        new_w, new_h = size, int(size * height / width)
    else:
        new_w, new_h = int(size * width / height), size
    left, top = (new_w - size) / 2, (new_h - size) / 2
    x0, y0, x1, y1 = (int(round(v)) for v in (left, top, left + size, top + size))
    return new_w, new_h, x0, y0, x1 - x0, y1 - y0


def _bicubic(x, a=-0.5):
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


_TABLES = {}


def pass_tables(in_size, out_size):
    """Pillow's coefficients of one bicubic resampling pass in_size -> out_size (float64, as its precompute_coeffs and
    normalize_coeffs_8bpc compute them) -> (bounds int32 [out_size, 2] = (first input index, tap count),
    coeffs int32 [out_size, ksize] in units of 2^-22). Pillow skips a pass that keeps the size; it is given here as the
    identity (one tap of 2^22), which the integer pass reproduces exactly. Cached per shape; do not modify."""
    key = (int(in_size), int(out_size))
    if key in _TABLES:
        return _TABLES[key]
    if in_size == out_size:
        bounds = np.stack([np.arange(out_size), np.ones(out_size, np.int64)], 1).astype(np.int32)
        coeffs = np.full((out_size, 1), 1 << PRECISION_BITS, np.int32)
    else:
        scale = in_size / out_size
        filterscale = max(scale, 1.0)
        support = BICUBIC_SUPPORT * filterscale
        ss = 1.0 / filterscale
        ksize = int(math.ceil(support)) * 2 + 1
        bounds = np.zeros((out_size, 2), np.int32)
        coeffs = np.zeros((out_size, ksize), np.int32)
        for xx in range(out_size):
            center = (xx + 0.5) * scale
            xmin = max(int(center - support + 0.5), 0)
            n = min(int(center + support + 0.5), in_size) - xmin
            k = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(n)]
            ww = 0.0
            for w in k:          # left to right like Pillow (Python's sum() compensates, which can differ in the last bit)
                ww += w
            for x, w in enumerate(k):
                w = w / ww if ww != 0.0 else w
                coeffs[xx, x] = int(w * (1 << PRECISION_BITS) + (-0.5 if w < 0 else 0.5))
            bounds[xx] = (xmin, n)
    for a in (bounds, coeffs):
        a.setflags(write=False)
    _TABLES[key] = (bounds, coeffs)
    return bounds, coeffs


_DEVICE_TABLES = {}


def _device_tables(in_size, out_size, device):
    import torch
    key = (int(in_size), int(out_size), device)
    if key not in _DEVICE_TABLES:
        b, k = pass_tables(in_size, out_size)
        _DEVICE_TABLES[key] = (torch.from_numpy(b.copy()).to(device), torch.from_numpy(k.copy()).to(device))
    return _DEVICE_TABLES[key]


def process_frames_cuda(frames, size=256):
    """`process_frames` on the GPU: decoded uint8 RGB frames [T, H, W, 3] (a numpy array such as
    decord's `get_batch(...).asnumpy()`, or a torch tensor on the host or the device) -> float32 CUDA tensor
    [T, size, size, 3] in [-1, 1], bit-identical to `process_frames` on the same frames, ready for `VQGAN.encode`.
    Host frames are uploaded through a pinned buffer on the current stream. There is no CPU path."""
    import torch
    from . import _lib
    if not torch.cuda.is_available():
        raise _lib.LwmError("process_frames_cuda needs an sm_90 GPU: lwm_b200 has no CPU fallback")
    if torch.is_tensor(frames):
        x = frames
    else:
        a = np.ascontiguousarray(frames)
        x = torch.from_numpy(a if a.flags.writeable else a.copy())     # torch tensors cannot be read-only
    if x.dtype != torch.uint8 or x.dim() != 4 or x.shape[-1] != 3:
        raise ValueError("process_frames_cuda: frames must be uint8 [T, H, W, 3] (RGB), got %s %s"
                         % (x.dtype, tuple(x.shape)))
    T, H, W, _ = x.shape
    if H == 0 or W == 0:
        raise ValueError("process_frames_cuda: empty frames %s" % (tuple(x.shape),))
    if x.is_cuda:
        dev = x.device
        x = x.contiguous()
    else:
        dev = torch.device("cuda", torch.cuda.current_device())
        staged = torch.empty(x.shape, dtype=torch.uint8, pin_memory=True)
        staged.copy_(x)
        x = staged.to(dev, non_blocking=True)       # the caching host allocator keeps `staged` until the copy is done
    new_w, new_h, left, top, crop_w, crop_h = frame_geometry(H, W, size)
    xb, xk = _device_tables(W, new_w, dev)
    yb, yk = _device_tables(H, new_h, dev)
    out = torch.empty(T, crop_h, crop_w, 3, dtype=torch.float32, device=dev)
    if T == 0:
        return out
    with torch.cuda.device(dev):
        _lib.call("lwm_vq_frames_prep", _lib.ptr(x), T, H, W, 3, _lib.ptr(xb), _lib.ptr(xk), new_w, xk.shape[1],
                  _lib.ptr(yb), _lib.ptr(yk), new_h, yk.shape[1], left, top, crop_w, crop_h, _lib.ptr(out),
                  _lib.stream_ptr())
    return out
