"""Integer restatement of Pillow's 8-bit bicubic resize (the two separable passes of its ImagingResample) followed by the
crop and scaling of `Sampler._process_frame` (lwm/vision_chat.py:59-74), driven by the product's coefficient tables
(lwm_b200.vision_frames.pass_tables / frame_geometry). TEST INFRASTRUCTURE ONLY: it states, in numpy, the arithmetic
lwm_vq_frames_prep runs, so that the tests can hold the tables and that arithmetic against Pillow itself."""
import numpy as np

PRECISION_BITS = 22


def resample_pass(img, axis, bounds, coeffs):
    """One pass along `axis` of a uint8 image [H, W, C]: out[i] = clip((2^21 + sum_j k[i, j] * in[xmin_i + j]) >> 22)
    over the n_i taps of output index i."""
    x = np.moveaxis(img, axis, 0).astype(np.int64)
    acc = np.full((len(bounds),) + x.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    xmin, n = bounds[:, 0].astype(np.int64), bounds[:, 1].astype(np.int64)
    bshape = (-1,) + (1,) * (x.ndim - 1)
    for j in range(coeffs.shape[1]):
        live = j < n
        src = x[np.where(live, xmin + j, 0)]
        acc += np.where(live, coeffs[:, j], 0).astype(np.int64).reshape(bshape) * src
    assert acc.max() < 2 ** 31 and acc.min() >= -2 ** 31        # Pillow accumulates in int32
    return np.moveaxis(np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8), 0, axis)


def process_frame(arr, size=256):
    """uint8 RGB [H, W, 3] -> float32 [size, size, 3] in [-1, 1], the arithmetic of lwm_vq_frames_prep."""
    from lwm_b200.vision_frames import frame_geometry, pass_tables
    h, w = arr.shape[:2]
    new_w, new_h, left, top, crop_w, crop_h = frame_geometry(h, w, size)
    x = resample_pass(arr, 1, *pass_tables(w, new_w))          # horizontal first, as Pillow
    x = resample_pass(x, 0, *pass_tables(h, new_h))
    x = x[top:top + crop_h, left:left + crop_w]
    return np.subtract(np.divide(x.astype(np.float32), np.float32(127.5)), np.float32(1))
