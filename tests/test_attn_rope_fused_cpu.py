"""`ringattention(..., freqs_cis=, position_ids=)` without a GPU: the argument checks of the rotary keywords, and the
argument validation of the rotating operand passes of the C ABI (lwm_attn_absmax_rope, lwm_attn_stage_rope,
lwm_reduce_cast_rope_f32), which reject bad pointers and dtype codes before they look for a device."""
import ctypes

import pytest
import torch

P = ctypes.c_void_p(0x1000)      # fake non-null pointer
N = None
ARG, DEVICE = 3, 1
SRCS = (ctypes.c_void_p * 2)(0x1000, 0x2000)
SRCS_NULL = (ctypes.c_void_p * 2)(0x1000, None)

BAD_CALLS = [
    ("lwm_attn_absmax_rope", (N, 1, P, P, 1, 8, 2, P, N), "null pointer"),
    ("lwm_attn_absmax_rope", (P, 1, N, P, 1, 8, 2, P, N), "null pointer"),
    ("lwm_attn_absmax_rope", (P, 1, P, N, 1, 8, 2, P, N), "null pointer"),
    ("lwm_attn_absmax_rope", (P, 1, P, P, 1, 8, 2, N, N), "null pointer"),
    ("lwm_attn_absmax_rope", (P, 2, P, P, 1, 8, 2, P, N), "dtype codes"),
    ("lwm_attn_absmax_rope", (P, 0, P, P, 1, 0, 2, P, N), "bad sizes"),
    ("lwm_attn_stage_rope", (N, 0, P, 2, P, P, P, 1, 8, 2, N), "null pointer"),
    ("lwm_attn_stage_rope", (P, 0, N, 2, P, P, P, 1, 8, 2, N), "null pointer"),
    ("lwm_attn_stage_rope", (P, 3, P, 2, P, P, P, 1, 8, 2, N), "dtype codes"),
    ("lwm_attn_stage_rope", (P, 0, P, 0, P, P, P, 1, 8, 2, N), "dst dtype codes"),
    ("lwm_attn_stage_rope", (P, 0, P, 2, N, P, P, 1, 8, 2, N), "needs a scale"),
    ("lwm_attn_stage_rope", (P, 1, P, 1, P, P, P, 1, 8, -1, N), "bad sizes"),
    ("lwm_reduce_cast_rope_f32", (SRCS, 17, P, 0, P, P, 1, 8, 2, N), "1..16 sources"),
    ("lwm_reduce_cast_rope_f32", (SRCS, 2, P, 2, P, P, 1, 8, 2, N), "dst dtype 0 or 1"),
    ("lwm_reduce_cast_rope_f32", (SRCS, 2, N, 1, P, P, 1, 8, 2, N), "bad arguments"),
    ("lwm_reduce_cast_rope_f32", (SRCS, 2, P, 1, N, P, 1, 8, 2, N), "null pointer"),
    ("lwm_reduce_cast_rope_f32", (SRCS_NULL, 2, P, 1, P, P, 1, 8, 2, N), "null source"),
]


def _status(lib, name, *args):
    from lwm_b200 import _lib
    _lib.load()
    return getattr(lib, name)(*args), lib.lwm_last_error().decode()


@pytest.mark.parametrize("name,args,frag", BAD_CALLS, ids=["%s-%d" % (c[0][4:], i) for i, c in enumerate(BAD_CALLS)])
def test_rotating_passes_reject_bad_arguments(lib, name, args, frag):
    status, msg = _status(lib, name, *args)
    assert status == ARG, (status, msg)
    assert frag in msg and name[4:] in msg, msg


GOOD_CALLS = [
    ("lwm_attn_absmax_rope", (P, 1, P, P, 2, 7, 3, P, N)),
    ("lwm_attn_stage_rope", (P, 0, P, 2, P, P, P, 2, 7, 3, N)),
    ("lwm_attn_stage_rope", (P, 1, P, 1, N, P, P, 2, 7, 3, N)),      # the bf16 copy needs no scale
    ("lwm_reduce_cast_rope_f32", (SRCS, 2, P, 1, P, P, 2, 7, 3, N)),
]


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: only meaningful where the device check fails")
@pytest.mark.parametrize("name,args", GOOD_CALLS, ids=["%s-%d" % (c[0][4:], i) for i, c in enumerate(GOOD_CALLS)])
def test_rotating_passes_fail_with_device_error_without_gpu(lib, name, args):
    status, msg = _status(lib, name, *args)
    assert status == DEVICE, (status, msg)


def _qkv(B=1, Sq=128, Sk=128, H=2):
    q = torch.zeros(B, Sq, H, 128, dtype=torch.bfloat16)
    k = torch.zeros(B, Sk, H, 128, dtype=torch.bfloat16)
    return q, k, k.clone()


def _table(max_position=4096):
    from lwm_b200.rope import precompute_freqs_cis
    return precompute_freqs_cis(128, max_position, 1e4, device="cpu")


def test_rotary_keywords_go_together():
    from lwm_b200.ringattention import ringattention
    q, k, v = _qkv()
    pos = torch.arange(128)[None]
    with pytest.raises(ValueError, match="go together"):
        ringattention(q, k, v, freqs_cis=_table())
    with pytest.raises(ValueError, match="go together"):
        ringattention(q, k, v, position_ids=pos)


def test_rotary_needs_a_rotary_table():
    from lwm_b200.ringattention import ringattention
    q, k, v = _qkv()
    with pytest.raises(ValueError, match="precompute_freqs_cis"):
        ringattention(q, k, v, freqs_cis=torch.zeros(4096, 64), position_ids=torch.arange(128)[None])


def test_rotary_needs_equal_query_and_key_lengths():
    from lwm_b200.ringattention import ringattention
    q, k, v = _qkv(Sq=128, Sk=256)
    with pytest.raises(ValueError, match="Sq == Sk"):
        ringattention(q, k, v, freqs_cis=_table(), position_ids=torch.arange(128)[None])


@pytest.mark.parametrize("shape", [(128,), (1, 64), (2, 128), (1, 128, 1)])
def test_rotary_position_ids_must_be_batch_by_local_rows(shape):
    from lwm_b200.ringattention import ringattention
    q, k, v = _qkv(B=1)
    with pytest.raises(ValueError, match="position_ids must be"):
        ringattention(q, k, v, freqs_cis=_table(), position_ids=torch.zeros(shape, dtype=torch.int64))


@pytest.mark.parametrize("bad", [-1, 4096, 1 << 40])
def test_rotary_positions_must_lie_in_the_table(bad):
    from lwm_b200.ringattention import ringattention
    q, k, v = _qkv(B=2)
    pos = torch.arange(128).repeat(2, 1)
    pos[1, 77] = bad
    with pytest.raises(ValueError, match="outside"):
        ringattention(q, k, v, freqs_cis=_table(4096), position_ids=pos)


def test_rotary_keywords_pass_validation_and_then_need_a_gpu():
    """well-formed keywords get as far as the device check of the op itself"""
    from lwm_b200 import _lib
    from lwm_b200.ringattention import ringattention
    q, k, v = _qkv(B=2)
    pos = torch.arange(128).repeat(2, 1) + 4096 - 128
    with pytest.raises(_lib.LwmError, match="sm_90"):
        ringattention(q, k, v, freqs_cis=_table(4096), position_ids=pos)
