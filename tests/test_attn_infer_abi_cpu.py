"""Argument validation of the inference-path entry points, without a GPU: bad shapes and null pointers are rejected
with a message before the device check, and well-formed calls fail with LWM_ERR_DEVICE (no fallback).
Pointers are fake non-null addresses: nothing dereferences them before the device check."""
import ctypes

import pytest
import torch

from helpers import FOLDED_ENTRY_POINTS, abi_row_id, with_options

P = ctypes.c_void_p(0x1000)
N = None
SHAPE, ARG, DEVICE = 2, 3, 1


def _status(lib, name, *args):
    from lwm_b200 import _lib
    _lib.load()
    return getattr(lib, name)(*args), lib.lwm_last_error().decode()


BAD_CALLS = [
    ("lwm_attn_decode_partial", (P, P, P, 0, N, N, N, P, P, N, 1, 2, 1, 128, 128, 0, 0, 0, 4, 0.1, N, N, N), ARG, "null"),
    ("lwm_attn_decode_partial", (P, P, P, 0, N, N, N, P, P, P, 1, 2, 1, 128, 64, 0, 0, 0, 4, 0.1, N, N, N), SHAPE, "head_dim"),
    ("lwm_attn_decode_merge", (P, P, 0, P, 0, P, 8, N), ARG, "bad args"),
    ("lwm_attn_decode_merge", (P, P, 2, N, 0, P, 8, N), ARG, "bad args"),
    ("lwm_attn_mask_pack", (N, 0, 64, 1, 1, 4, 0, 64, 1, P, P, N), ARG, "null"),
    ("lwm_attn_mask_pack", (P, 0, 64, 1, 1, 4, 0, 0, 1, P, P, N), SHAPE, "bad shape"),
    ("lwm_attn_mask_pack", (P, 0, 64, 0, 1, 4, 0, 64, 1, P, P, N), SHAPE, "strides"),
    ("lwm_attn_infer_tilemap", (P, P, 1, 4, 64, N, P, N), ARG, "null"),
    ("lwm_attn_infer_tilemap", (P, P, 1, 0, 64, P, P, N), SHAPE, "bad shape"),
    ("lwm_attn_infer_partial", (P, P, P, P, P, P, N, P, P, P, P, N, 1, 2, 200, 300, 64, 1, 0.1, N), SHAPE, "head_dim"),
    ("lwm_attn_infer_partial", (P, P, P, P, N, P, N, P, P, P, P, N, 1, 2, 200, 300, 128, 1, 0.1, N), ARG, "null"),
    ("lwm_attn_infer_partial", (P, P, P, P, P, P, N, N, P, P, P, N, 1, 2, 200, 300, 128, 1, 0.1, N), ARG, "null"),
    ("lwm_attn_infer_partial", (P, P, P, P, P, P, N, P, P, P, P, N, 1, 2, 200, 300, 128, 3, 0.1, N), ARG, "workspace"),
    ("lwm_attn_infer_partial", (P, P, P, P, P, P, N, P, P, P, P, P, 1, 2, 0, 300, 128, 3, 0.1, N), SHAPE, "bad shape"),
    ("lwm_attn_infer_partial", (P, P, P, P, P, P, N, P, P, P, P, P, 1, 2, 200, 300, 128, 0, 0.1, N), SHAPE, "splits"),
]

# the same rows with the options of the folded entry points turned on: no option slot bypasses these checks
BAD_CALLS += [(n, with_options(n, a, P), c, f) for n, a, c, f in BAD_CALLS if n in FOLDED_ENTRY_POINTS]


@pytest.mark.parametrize("name,args,code,frag", BAD_CALLS,
                         ids=["%s-%d" % (abi_row_id(*c[:2]), i) for i, c in enumerate(BAD_CALLS)])
def test_bad_arguments_are_rejected_with_a_message(lib, name, args, code, frag):
    status, msg = _status(lib, name, *args)
    assert status == code, (status, msg)
    assert frag in msg, msg


GOOD_CALLS = [
    ("lwm_attn_decode_partial", (P, P, P, 0, N, N, N, P, P, P, 1, 2, 1, 128, 128, 0, 0, 0, 4, 0.1, N, N, N)),
    ("lwm_attn_decode_merge", (P, P, 2, P, 0, P, 8, N)),
    ("lwm_attn_mask_pack", (P, 0, 300, 1, 2, 200, 0, 150, 2, P, P, N)),
    ("lwm_attn_infer_tilemap", (N, N, 2, 200, 300, P, P, N)),
    ("lwm_attn_infer_partial", (P, P, P, P, P, P, N, P, P, P, P, N, 1, 2, 200, 300, 128, 1, 0.1, N)),
    ("lwm_attn_infer_partial", (P, P, P, P, P, P, P, P, P, P, P, P, 1, 2, 200, 300, 128, 3, 0.1, N)),
]

GOOD_CALLS += [(n, with_options(n, a, P)) for n, a in GOOD_CALLS if n in FOLDED_ENTRY_POINTS]


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: only meaningful where the device check fails")
@pytest.mark.parametrize("name,args", GOOD_CALLS, ids=["%s-%d" % (abi_row_id(*c), i) for i, c in enumerate(GOOD_CALLS)])
def test_well_formed_calls_fail_with_device_error_without_gpu(lib, name, args):
    status, msg = _status(lib, name, *args)
    assert status == DEVICE, (status, msg)
    assert "no CPU fallback" in msg or "sm_90" in msg, msg
