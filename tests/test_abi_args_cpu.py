"""Argument validation of the C ABI, checked without a GPU: every entry point validates its pure arguments (shapes,
null pointers, flags) BEFORE it looks for a device, so wrong calls get LWM_ERR_SHAPE (2) / LWM_ERR_ARG (3) with a message,
and well-formed calls on a machine without an sm_90 GPU get LWM_ERR_DEVICE (1) — never a silent fallback.
Pointers are fake non-null addresses: nothing dereferences them before the device check."""
import ctypes

import pytest
import torch

P = ctypes.c_void_p(0x1000)      # fake non-null pointer
N = None
SHAPE, ARG, DEVICE = 2, 3, 1


def _status(lib, name, *args):
    from lwm_b200 import _lib
    _lib.load()
    return getattr(lib, name)(*args), lib.lwm_last_error().decode()


BAD_CALLS = [
    # (entry, args, expected status, message fragment)
    ("lwm_attn_fwd_step", (P, P, P, P, P, N, N, N, 1, 2, 128, 128, 64, 0, 0, 1, N, 0, N, 0, 0.1, 1, 1, N), SHAPE, "head_dim"),
    ("lwm_attn_fwd_step", (P, P, P, P, P, N, N, N, 1, 2, 100, 128, 128, 0, 0, 1, N, 0, N, 0, 0.1, 1, 1, N), SHAPE, "multiples of 128"),
    ("lwm_attn_fwd_step", (N, P, P, P, P, N, N, N, 1, 2, 128, 128, 128, 0, 0, 1, N, 0, N, 0, 0.1, 1, 1, N), ARG, "null"),
    ("lwm_attn_fwd_step", (P, P, P, N, N, N, N, N, 1, 2, 128, 128, 128, 0, 0, 1, N, 0, N, 0, 0.1, 1, 1, N), ARG, "last step"),
    ("lwm_attn_fwd_step", (P, P, P, P, P, N, N, N, 1, 2, 128, 128, 128, 0, 0, 1, N, 0, N, 0, 0.1, 1, 0, N), ARG, "carry"),
    ("lwm_attn_fwd_step", (P, P, P, P, P, N, N, N, 1, 2, 128, 128, 128, 1 << 31, 0, 1, N, 0, N, 0, 0.1, 1, 1, N), SHAPE, "int32"),
    ("lwm_attn_bwd_step", (P, P, P, P, P, P, P, P, N, 1, 2, 128, 128, 128, 0, 0, 1, N, 0, N, 0, 0.1, 0, N), ARG, "null"),
    ("lwm_attn_bwd_step", (P, P, P, P, P, P, P, P, P, 1, 2, 128, 192, 128, 0, 0, 1, N, 0, N, 0, 0.1, 0, N), SHAPE, "multiples of 128"),
    ("lwm_attn_absmax", (P, 2, 64, P, N), ARG, "bad arguments"),
    ("lwm_attn_to_f16_scaled", (P, 1, P, P, 12, N), ARG, "n % 8"),
    ("lwm_attn_bwd_prep_f16", (P, 0, P, P, P, 1, 2, 128, 64, N), SHAPE, "head_dim"),
    ("lwm_reduce_cast_f32", (P, 17, P, 1, 64, N), ARG, "1..16 sources"),
    ("lwm_ring_ctx_create", (3, 2, 1024, 0, P), ARG, "bad rank/world"),
    ("lwm_ring_copy", (N, P, 16, N), ARG, "bad arguments"),
    ("lwm_ring_signal", (N, 0, 0, 1, N), ARG, "null context"),
    ("lwm_attn_bwd_prep", (P, P, P, 1, 2, 128, 96, N), SHAPE, "head_dim"),
    ("lwm_attn_bwd_lse", (P, P, 0, 0.0, N), ARG, "bad args"),
    ("lwm_attn_to_f16", (P, P, P, P, 12, N), SHAPE, "multiple of 8"),
    ("lwm_attn_decode_partial", (P, P, P, N, P, P, N, 1, 2, 1, 128, 128, 0, 0, 0, 4, 0.1, N), ARG, "null"),
    ("lwm_attn_decode_merge", (P, P, 0, P, P, 8, N), ARG, "bad args"),
    ("lwm_attn_rope", (P, P, 0, P, P, 2, P, P, 1, 8, 2, 2, 128, 0, N), ARG, "dtype"),
    ("lwm_attn_rope", (P, P, 0, P, P, 1, P, P, 1, 8, 2, 2, 64, 0, N), SHAPE, "head_dim"),
    ("lwm_cast_f32_to_bf16", (P, P, 6, N), SHAPE, "multiple of 4"),
    ("lwm_add_f32", (P, P, 2, N), SHAPE, "multiple of 4"),
    ("lwm_vq_gn_stats", (P, P, 1, 8, 8, 100, 32, N), SHAPE, "C/groups"),
    ("lwm_vq_prep", (P, N, N, N, P, N, 1, 8, 8, 6, 64, 32, 0, 1e-6, N), SHAPE, "C % 4"),
    ("lwm_vq_conv2d", (P, N, P, N, P, N, P, 1, 16, 16, 64, 16, 16, 64, 64, 3, 1, 1, 3, 0, N), ARG, "lo planes"),
    ("lwm_vq_conv2d", (P, N, P, N, P, N, P, 1, 16, 16, 64, 16, 16, 64, 64, 3, 1, 1, 2, 0, N), ARG, "n_pass"),
    ("lwm_vq_conv2d", (P, N, P, N, P, N, P, 1, 16, 16, 64, 12, 16, 64, 64, 3, 1, 1, 1, 0, N), SHAPE, "8 x 16"),
    ("lwm_vq_conv2d", (P, N, P, N, P, N, P, 1, 16, 16, 64, 16, 16, 64, 64, 5, 1, 2, 1, 0, N), SHAPE, "ksize"),
    ("lwm_vq_prep_f16", (P, N, N, N, P, N, P, 0, 1, 8, 8, 64, 64, 32, 0, 1e-6, N), ARG, "null pointer"),
    ("lwm_vq_prep_f16", (P, N, N, N, P, P, N, 0, 1, 8, 8, 64, 64, 32, 0, 1e-6, N), ARG, "x_absmax"),
    ("lwm_vq_prep_f16", (P, N, N, N, P, P, P, 1, 1, 8, 8, 6, 64, 32, 0, 1e-6, N), SHAPE, "C % 4"),
    ("lwm_vq_conv2d_f16", (P, P, P, P, N, P, N, N, 1, 16, 16, 64, 16, 16, 64, 64, 3, 1, 1, 0.0, 32, 0, N), ARG, "w_scale_inv"),
    ("lwm_vq_conv2d_f16", (P, N, P, P, N, P, P, P, 1, 16, 16, 64, 16, 16, 64, 64, 3, 1, 1, 1.0, 32, 0, N), SHAPE, "statistics"),
    ("lwm_vq_conv_cin3", (P, P, P, P, 1, 16, 16, 64, N), SHAPE, "Cout == 128"),
    ("lwm_vq_argmin", (P, P, P, N, P, 16, 8192, 32, N), SHAPE, "e_dim"),
    ("lwm_vq_argmin", (P, P, P, N, N, 16, 8192, 64, N), ARG, "null"),
    ("lwm_vq_gather", (P, P, P, 16, 8192, 6, N), SHAPE, "e_dim"),
    ("lwm_vq_frame_tokens", (P, N, P, 1, 4, 2, 256, 8192, 8193, N), SHAPE, "frame_idx"),
    ("lwm_vq_frame_tokens", (P, N, P, 1, 0, 0, 256, 8192, 8193, N), SHAPE, "at least one frame"),
    ("lwm_vq_unframe_tokens", (N, P, 4, 256, N), ARG, "null"),
]


@pytest.mark.parametrize("name,args,code,frag", BAD_CALLS, ids=["%s-%s" % (c[0][4:], c[3].replace(" ", "_")) for c in BAD_CALLS])
def test_bad_arguments_are_rejected_with_a_message(lib, name, args, code, frag):
    status, msg = _status(lib, name, *args)
    assert status == code, (status, msg)
    assert frag in msg, msg


GOOD_CALLS = [
    ("lwm_attn_fwd_step", (P, P, P, P, P, N, N, N, 1, 2, 128, 128, 128, 0, 0, 1, N, 0, N, 0, 0.1, 1, 1, N)),
    ("lwm_attn_bwd_step", (P, P, P, P, P, P, P, P, P, 1, 2, 128, 128, 128, 0, 0, 1, N, 0, N, 0, 0.1, 1, N)),
    ("lwm_attn_absmax", (P, 1, 64, P, N)),
    ("lwm_attn_bwd_prep_f16", (P, 0, P, P, P, 1, 2, 128, 128, N)),
    ("lwm_attn_rope", (P, P, 1, P, P, 1, P, P, 1, 8, 2, 2, 128, 0, N)),
    ("lwm_vq_conv2d", (P, P, P, P, P, N, P, 1, 16, 16, 64, 16, 16, 64, 64, 3, 1, 1, 3, 0, N)),
    ("lwm_vq_argmin", (P, P, P, N, P, 16, 8192, 64, N)),
    ("lwm_vq_prep_f16", (P, N, N, N, P, P, P, 0, 1, 8, 8, 64, 64, 32, 0, 1e-6, N)),
    ("lwm_vq_prep_f16", (P, N, N, N, P, P, P, 1, 1, 8, 8, 64, 64, 32, 0, 1e-6, N)),
    ("lwm_vq_prep_f16", (P, P, P, P, P, P, N, 0, 1, 8, 8, 128, 128, 32, 1, 1e-6, N)),
    ("lwm_vq_conv2d_f16", (P, P, P, P, N, P, P, P, 1, 16, 16, 64, 16, 16, 128, 128, 3, 1, 1, 0.25, 32, 0, N)),
    ("lwm_vq_conv2d_f16", (P, N, P, P, P, P, N, N, 1, 16, 16, 64, 16, 16, 64, 64, 3, 2, 0, 0.25, 32, 1, N)),
    ("lwm_vq_frame_tokens", (P, N, P, 1, 4, 4, 256, 8192, 8193, N)),
    ("lwm_cast_f32_to_bf16", (P, P, 0, N)),           # even an empty call does not succeed without a device
]


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: only meaningful where the device check fails")
@pytest.mark.parametrize("name,args", GOOD_CALLS, ids=[c[0][4:] for c in GOOD_CALLS])
def test_well_formed_calls_fail_with_device_error_without_gpu(lib, name, args):
    status, msg = _status(lib, name, *args)
    assert status == DEVICE, (status, msg)
    assert "no CPU fallback" in msg or "sm_90" in msg, msg
