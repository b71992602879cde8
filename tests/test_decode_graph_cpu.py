"""The capturable decode step without a GPU:
  * the C ABI of lwm_kv_cache_write_at and lwm_rope_check_positions: declared, exported and bound, and bad arguments
    rejected before the device check;
  * ShardedKVCache's slot kept twice, on the host (cache_index) and in the device cursor: the setter writes both, the
    getter reads the cursor once a decode write has been captured;
  * the guards of a capture (torch.cuda's capture state stood in for): the prefill, host positions, a ring of more than
    one rank and the tensor-core path are refused;
  * decode_attention_mask with the cursor as a 0-d tensor."""
import ctypes
import os

import pytest
import torch

from helpers import abi_row_id

P = ctypes.c_void_p(0x1000)
P_ODD = ctypes.c_void_p(0x1001)
N = None
SHAPE, ARG, DEVICE = 2, 3, 1
NEW_SYMBOLS = ("lwm_kv_cache_write_at", "lwm_rope_check_positions")


def test_decode_graph_symbols_are_declared_exported_and_bound(lib):
    from lwm_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "lwm_b200.h")).read()
    for name in NEW_SYMBOLS:
        assert "int %s(" % name in header
        assert hasattr(lib, name)
        assert name in _lib._SIGNATURES
    assert "#define LWM_DEVICE_ERR_SLOT 1" in header and "#define LWM_DEVICE_ERR_POSITION 2" in header
    from lwm_b200 import rope
    assert (rope.ERR_SLOT, rope.ERR_POSITION) == (1, 2)


# lwm_kv_cache_write_at(k_new, v_new, src_dtype, cache_k, cache_v, k_exp, v_exp, pos, inv_freq, max_position, cursor,
#                       lo, L, max_length, B, H, D, err, stream)
WA = (P, P, 1, P, P, N, N, N, N, 0, P, 0, 64, 256, 2, 4, 128, P, N)
# lwm_rope_check_positions(pos, n, max_position, err, stream)
CP = (P, 4, 4096, P, N)


def _with(args, **at):
    a = list(args)
    for k, val in at.items():
        a[int(k[1:])] = val
    return tuple(a)


BAD_CALLS = [
    ("lwm_kv_cache_write_at", _with(WA, a16=64), SHAPE, "head_dim"),
    ("lwm_kv_cache_write_at", _with(WA, a14=0), SHAPE, "bad sizes"),
    ("lwm_kv_cache_write_at", _with(WA, a15=0), SHAPE, "bad sizes"),
    ("lwm_kv_cache_write_at", _with(WA, a13=0), SHAPE, "bad sizes"),
    ("lwm_kv_cache_write_at", _with(WA, a11=200), SHAPE, "out of range"),      # lo + L > max_length
    ("lwm_kv_cache_write_at", _with(WA, a11=-1), SHAPE, "out of range"),
    ("lwm_kv_cache_write_at", _with(WA, a0=N), ARG, "null pointer"),
    ("lwm_kv_cache_write_at", _with(WA, a4=N), ARG, "null pointer"),
    ("lwm_kv_cache_write_at", _with(WA, a10=N), ARG, "null pointer"),          # cursor
    ("lwm_kv_cache_write_at", _with(WA, a17=N), ARG, "null pointer"),          # error word
    ("lwm_kv_cache_write_at", _with(WA, a5=P), ARG, "go together"),            # k_exp without v_exp
    ("lwm_kv_cache_write_at", _with(WA, a6=P), ARG, "go together"),
    ("lwm_kv_cache_write_at", _with(WA, a7=P, a9=4096), ARG, "position_ids"),  # positions without inv_freq
    ("lwm_kv_cache_write_at", _with(WA, a7=P, a8=P, a9=0), ARG, "max_position"),
    ("lwm_kv_cache_write_at", _with(WA, a2=2), ARG, "dtype codes"),
    ("lwm_kv_cache_write_at", _with(WA, a5=P, a6=P, a3=P_ODD), ARG, "aligned"),
    ("lwm_kv_cache_write_at", _with(WA, a5=P, a6=P_ODD), ARG, "aligned"),
    ("lwm_kv_cache_write_at", _with(WA, a10=P_ODD), ARG, "aligned"),
    ("lwm_rope_check_positions", _with(CP, a1=0), SHAPE, "bad sizes"),
    ("lwm_rope_check_positions", _with(CP, a0=N), ARG, "null pointer"),
    ("lwm_rope_check_positions", _with(CP, a3=N), ARG, "null pointer"),
    ("lwm_rope_check_positions", _with(CP, a2=0), ARG, "max_position"),
]


def _status(lib, name, *args):
    from lwm_b200 import _lib
    _lib.load()
    return getattr(lib, name)(*args), lib.lwm_last_error().decode()


@pytest.mark.parametrize("name,args,code,frag", BAD_CALLS,
                         ids=["%s-%d" % (abi_row_id(*c[:2]), i) for i, c in enumerate(BAD_CALLS)])
def test_bad_arguments_are_rejected_with_a_message(lib, name, args, code, frag):
    status, msg = _status(lib, name, *args)
    assert status == code, (status, msg)
    assert frag in msg, msg


GOOD_CALLS = [("lwm_kv_cache_write_at", WA), ("lwm_kv_cache_write_at", _with(WA, a7=P, a8=P, a9=4096)),
              ("lwm_kv_cache_write_at", _with(WA, a5=P, a6=P)),
              ("lwm_kv_cache_write_at", _with(WA, a5=P, a6=P, a7=P, a8=P, a9=4096, a2=0)),
              ("lwm_kv_cache_write_at", _with(WA, a11=192)), ("lwm_rope_check_positions", CP)]


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: only meaningful where the device check fails")
@pytest.mark.parametrize("name,args", GOOD_CALLS, ids=["%s-%d" % (abi_row_id(*c), i) for i, c in enumerate(GOOD_CALLS)])
def test_well_formed_calls_fail_with_device_error_without_gpu(lib, name, args):
    status, msg = _status(lib, name, *args)
    assert status == DEVICE, (status, msg)


# ------------------------------------------------------------------------------------------------
# the cursor and its host mirror
# ------------------------------------------------------------------------------------------------
def _cache(**kw):
    from lwm_b200.kv_cache import ShardedKVCache
    return ShardedKVCache(2, 64, 2, 4, dtype=torch.float32, device="cpu", **kw)


def test_cache_index_setter_writes_the_mirror_and_the_cursor():
    cache = _cache()
    assert cache._cursor is None            # the constructor allocates only the cache rows
    assert cache.cache_index == 0 and cache.cursor.dim() == 0 and cache.cursor.dtype == torch.int32
    cache.cache_index = 37
    assert cache.cache_index == 37 and int(cache.cursor) == 37
    with pytest.raises(ValueError, match=">= 0"):
        cache.cache_index = -1
    # the host bookkeeping path keeps the two in step
    k = torch.randn(2, 1, 2, 4)
    cache.concatenate(k, k)
    assert cache.cache_index == 38 and int(cache.cursor) == 38
    cache.cache_index = 10
    cache.concatenate(torch.randn(2, 5, 2, 4), torch.randn(2, 5, 2, 4))
    assert cache.cache_index == 15 and int(cache.cursor) == 15
    assert cache.take_errors() == 0


def test_cache_index_reads_the_cursor_once_a_write_was_captured():
    cache = _cache()
    cache.cache_index = 5
    assert int(cache.cursor) == 5          # made on first use, from the host value
    cache._captured = True              # what a captured decode write leaves behind
    cache._cursor[0] = 42               # what replays do to the cursor
    assert cache.cache_index == 42
    cache.cache_index = 3
    assert cache.cache_index == 3 and int(cache.cursor) == 3


@pytest.fixture
def capturing(monkeypatch):
    """torch.cuda's capture state stood in for: the package sees a capture in progress"""
    from lwm_b200 import rope
    monkeypatch.setattr(rope, "capturing", lambda: True)


def _table():
    from lwm_b200.rope import precompute_freqs_cis
    return precompute_freqs_cis(128, 4096, 1e4, device="cpu")


def test_prefill_and_cache_index_are_refused_while_capturing(capturing):
    cache = _cache()
    with pytest.raises(RuntimeError, match="prefill eagerly"):
        cache.concatenate(torch.randn(2, 4, 2, 4), torch.randn(2, 4, 2, 4))
    with pytest.raises(RuntimeError, match="warm-up"):       # the cursor is never made inside a capture
        cache.cursor
    cache._captured = True
    with pytest.raises(RuntimeError, match="cursor"):
        cache.cache_index


def test_host_positions_are_refused_while_capturing(capturing):
    from lwm_b200.rope import check_position_ids
    with pytest.raises(ValueError, match="device tensor"):
        check_position_ids("op", _table(), torch.zeros(1, 1, dtype=torch.int64), (1, 1), "cpu")


def _infer(Q, **kw):
    from lwm_b200.ringattention import ringattention_inference
    q = torch.zeros(1, Q, 2, 128, dtype=torch.bfloat16)
    k = torch.zeros(1, 64, 2, 128, dtype=torch.bfloat16)
    return ringattention_inference(q, k, k, None, **kw)


def test_ringattention_inference_capture_guards(capturing, monkeypatch):
    from lwm_b200 import ringattention as ra
    with pytest.raises(NotImplementedError, match="INFER_MIN_Q"):
        _infer(ra.INFER_MIN_Q)
    with pytest.raises(ValueError, match="device tensor"):
        _infer(1, freqs_cis=_table(), position_ids=torch.zeros(1, 1, dtype=torch.int64), rotate_k=False)
    monkeypatch.setattr(ra, "_resolve_group", lambda axis_name: (None, 0, 2))
    with pytest.raises(NotImplementedError, match="one GPU"):
        _infer(1)


def test_decode_attention_mask_takes_the_cursor():
    from lwm_b200.ringattention import decode_attention_mask
    am = torch.ones(2, 64, dtype=torch.int64)
    am[1, :5] = 0
    for idx in (0, 17, 63, 64):
        for Q in (1, 3):
            want = decode_attention_mask(am, Q, idx, 64)
            got = decode_attention_mask(am, Q, torch.tensor(idx, dtype=torch.int32), 64)
            assert got.dtype == torch.bool and torch.equal(got, want)
    with pytest.raises(ValueError, match="0-d integer"):
        decode_attention_mask(am, 1, torch.tensor([3]), 64)
    with pytest.raises(ValueError, match="0-d integer"):
        decode_attention_mask(am, 1, torch.tensor(3.0), 64)
