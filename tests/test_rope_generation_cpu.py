"""The rotary embedding of the generation path without a GPU: the keyword checks of `ringattention(rotate_k=False)`,
`ringattention_inference(freqs_cis=, position_ids=, rotate_k=)` and `ShardedKVCache.concatenate(freqs_cis=,
position_ids=)`; the argument validation of the C entries that rotate (lwm_attn_decode_partial given position_ids,
lwm_kv_cache_write_rope), which reject bad arguments before they look for a device; and, under gloo, the rotating
prefill write of the sequence-sharded cache with a CPU stand-in for the kernel: every rank keeps the same rows the
un-sharded update would hold."""
import ctypes
import os
import socket

import numpy as np
import pytest
import torch

from helpers import FOLDED_ENTRY_POINTS, abi_row_id, with_options

P = ctypes.c_void_p(0x1000)      # fake non-null pointer
N = None
SHAPE, ARG, DEVICE = 2, 3, 1

# lwm_attn_decode_partial(q, k, v, dtype, k_exp, v_exp, mask, o_part, ml_part, ws, B, H, Q, Sk, D, k_pos0, sb, sq,
#                         splits, scale, position_ids, inv_freq, stream), bf16 (dtype 1) and fp32 (0)
DEC = (P, P, P, 1, N, N, N, P, P, P, 1, 2, 1, 128, 128, 0, 0, 0, 4, 0.1, P, P, N)
# lwm_kv_cache_write_rope(k_new, v_new, dtype, cache_k, cache_v, position_ids, inv_freq, B, n_src, src0, n, L, dst0,
#                         H, D, stream)
KVW = (P, P, 1, P, P, P, P, 2, 8, 0, 8, 64, 8, 2, 128, N)


def _with(args, **at):
    a = list(args)
    for i, x in at.items():
        a[int(i[1:])] = x
    return tuple(a)


DEC32 = _with(DEC, a3=0)

BAD_CALLS = [
    ("lwm_attn_decode_partial", _with(DEC, a20=N), ARG, "null position_ids"),
    ("lwm_attn_decode_partial", _with(DEC, a21=N), ARG, "null position_ids"),
    ("lwm_attn_decode_partial", _with(DEC, a0=N), ARG, "null pointer"),
    ("lwm_attn_decode_partial", _with(DEC, a14=64), SHAPE, "head_dim"),
    ("lwm_attn_decode_partial", _with(DEC32, a20=N), ARG, "null position_ids"),
    ("lwm_attn_decode_partial", _with(DEC32, a12=0), SHAPE, "bad shape"),
    ("lwm_kv_cache_write_rope", _with(KVW, a14=64), SHAPE, "head_dim"),
    ("lwm_kv_cache_write_rope", _with(KVW, a10=0), SHAPE, "bad sizes"),
    ("lwm_kv_cache_write_rope", _with(KVW, a9=1), SHAPE, "out of range"),       # src0 + n > n_src
    ("lwm_kv_cache_write_rope", _with(KVW, a12=57), SHAPE, "out of range"),     # dst0 + n > L
    ("lwm_kv_cache_write_rope", _with(KVW, a12=-1), SHAPE, "out of range"),
    ("lwm_kv_cache_write_rope", _with(KVW, a5=N), ARG, "null pointer"),
    ("lwm_kv_cache_write_rope", _with(KVW, a6=N), ARG, "null pointer"),
    ("lwm_kv_cache_write_rope", _with(KVW, a3=N), ARG, "null pointer"),
    ("lwm_kv_cache_write_rope", _with(KVW, a2=2), ARG, "dtype codes"),
]

# the same rows with the options of the folded entry points turned on: no option slot bypasses these checks
BAD_CALLS += [(n, with_options(n, a, P), c, f) for n, a, c, f in BAD_CALLS if n in FOLDED_ENTRY_POINTS]


def _status(lib, name, *args):
    from lwm_b200 import _lib
    _lib.load()
    return getattr(lib, name)(*args), lib.lwm_last_error().decode()


@pytest.mark.parametrize("name,args,code,frag", BAD_CALLS,
                         ids=["%s-%d" % (abi_row_id(*c[:2]), i) for i, c in enumerate(BAD_CALLS)])
def test_new_entries_reject_bad_arguments(lib, name, args, code, frag):
    status, msg = _status(lib, name, *args)
    assert status == code, (status, msg)
    assert frag in msg, msg


GOOD_CALLS = [("lwm_attn_decode_partial", DEC), ("lwm_attn_decode_partial", DEC32),
              ("lwm_kv_cache_write_rope", KVW), ("lwm_kv_cache_write_rope", _with(KVW, a2=0, a9=3, a10=5, a12=59))]

GOOD_CALLS += [(n, with_options(n, a, P)) for n, a in GOOD_CALLS if n in FOLDED_ENTRY_POINTS]


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: only meaningful where the device check fails")
@pytest.mark.parametrize("name,args", GOOD_CALLS, ids=["%s-%d" % (abi_row_id(*c), i) for i, c in enumerate(GOOD_CALLS)])
def test_new_entries_fail_with_device_error_without_gpu(lib, name, args):
    status, msg = _status(lib, name, *args)
    assert status == DEVICE, (status, msg)
    assert "no CPU fallback" in msg or "sm_90" in msg, msg


# ------------------------------------------------------------------------------------------------
# keyword checks of the three calls
# ------------------------------------------------------------------------------------------------
def _table(max_position=4096):
    from lwm_b200.rope import precompute_freqs_cis
    return precompute_freqs_cis(128, max_position, 1e4, device="cpu")


def _t(*shape):
    return torch.zeros(*shape, 128, dtype=torch.bfloat16)


def _prefill(**kw):
    from lwm_b200.ringattention import ringattention
    return ringattention(_t(1, 128, 2), _t(1, 512, 2), _t(1, 512, 2), rotate_k=False, **kw)


def _infer(Q=4, Sk=64, **kw):
    from lwm_b200.ringattention import ringattention_inference
    return ringattention_inference(_t(1, Q, 2), _t(1, Sk, 2), _t(1, Sk, 2), None, **kw)


def _concat(n=4, **kw):
    from lwm_b200.kv_cache import ShardedKVCache
    cache = ShardedKVCache(1, 64, 2, 128, dtype=torch.bfloat16, device="cpu")
    return cache.concatenate(_t(1, n, 2), _t(1, n, 2), **kw)


CALLS = {"prefill": (_prefill, 128), "inference": (_infer, 4), "concatenate": (_concat, 4)}


@pytest.mark.parametrize("call", sorted(CALLS))
def test_rotary_keywords_go_together(call):
    fn, S = CALLS[call]
    with pytest.raises(ValueError, match="go together"):
        fn(freqs_cis=_table())
    with pytest.raises(ValueError, match="go together"):
        fn(position_ids=torch.arange(S)[None])


@pytest.mark.parametrize("call", sorted(CALLS))
def test_rotary_needs_a_rotary_table(call):
    fn, S = CALLS[call]
    with pytest.raises(ValueError, match="precompute_freqs_cis"):
        fn(freqs_cis=torch.zeros(4096, 64), position_ids=torch.arange(S)[None])


@pytest.mark.parametrize("call", sorted(CALLS))
@pytest.mark.parametrize("bad", range(4))
def test_rotary_position_ids_must_be_batch_by_new_rows(call, bad):
    fn, S = CALLS[call]
    shape = [(S,), (1, S - 1), (2, S), (1, S, 1)][bad]
    with pytest.raises(ValueError, match="position_ids must be"):
        fn(freqs_cis=_table(), position_ids=torch.zeros(shape, dtype=torch.int64))


@pytest.mark.parametrize("call", sorted(CALLS))
@pytest.mark.parametrize("bad", [-1, 4096, 1 << 40])
def test_rotary_positions_must_lie_in_the_table(call, bad):
    fn, S = CALLS[call]
    pos = torch.arange(S)[None].clone()
    pos[0, S // 2] = bad
    with pytest.raises(ValueError, match="outside"):
        fn(freqs_cis=_table(4096), position_ids=pos)


def test_inference_rotate_k_needs_equal_query_and_key_rows():
    with pytest.raises(ValueError, match="Q_loc == S_loc"):
        _infer(Q=4, Sk=64, freqs_cis=_table(), position_ids=torch.arange(4)[None])


def test_concatenate_with_rotation_needs_the_cache_dtype():
    from lwm_b200.kv_cache import ShardedKVCache
    cache = ShardedKVCache(1, 64, 2, 128, dtype=torch.bfloat16, device="cpu")
    k = torch.zeros(1, 1, 2, 128)
    with pytest.raises(ValueError, match="cache dtype"):
        cache.concatenate(k, k, freqs_cis=_table(), position_ids=torch.zeros(1, 1, dtype=torch.int64))


def test_well_formed_keywords_then_need_a_gpu():
    """valid keywords get as far as the device check of each op (the prefill with Sq != Sk and rotate_k=False, the
    decode call with rotate_k=False and Q != S_loc, the training branch with rotate_k=True and Q == S_loc)"""
    from lwm_b200 import _lib
    pos = torch.arange(128)[None] + 4096 - 128
    with pytest.raises(_lib.LwmError, match="sm_90"):
        _prefill(freqs_cis=_table(4096), position_ids=pos)
    with pytest.raises(_lib.LwmError, match="sm_90"):
        _infer(Q=1, Sk=64, freqs_cis=_table(4096), position_ids=pos[:, :1], rotate_k=False)
    with pytest.raises(_lib.LwmError, match="sm_90"):
        _infer(Q=64, Sk=64, freqs_cis=_table(4096), position_ids=pos[:, :64], rotate_k=True)


# ------------------------------------------------------------------------------------------------
# the rotating prefill write under gloo, with a CPU stand-in for lwm_kv_cache_write_rope
# ------------------------------------------------------------------------------------------------
def _rope_cpu(x, pos, inv_freq):
    """x [B,n,H,D] fp32 rotated at pos [B,n] (the table builder's float32 angles, a complex64 multiply)"""
    ang = (pos.double()[..., None] * inv_freq.double()).float()            # [B,n,64]
    c, s = torch.cos(ang.double()).float()[:, :, None], torch.sin(ang.double()).float()[:, :, None]
    a, b = x[..., 0::2], x[..., 1::2]
    return torch.stack((a * c - b * s, a * s + b * c), dim=-1).reshape(x.shape)


def _write_rope_cpu(k_src, v_src, src0, n, cache_k, cache_v, dst0, pos, inv_freq):
    rows = slice(src0, src0 + n)
    cache_k[:, dst0:dst0 + n] = _rope_cpu(k_src[:, rows], pos[:, rows], inv_freq)
    cache_v[:, dst0:dst0 + n] = v_src[:, rows]


def _problem(world):
    B, H, D, max_len, prompt = 2, 2, 128, 16 * world, 5 * world
    g = torch.Generator().manual_seed(world)
    k_new, v_new = torch.randn(B, prompt, H, D, generator=g), torch.randn(B, prompt, H, D, generator=g)
    # left padding: padded rows (position -1 in the reference) are mapped to position 0 by the caller
    pos = torch.arange(prompt)[None].repeat(B, 1) - torch.tensor([[0], [3]])
    pos = pos.clamp(min=0) + 1000
    steps = [(torch.randn(B, 1, H, D, generator=g), torch.randn(B, 1, H, D, generator=g)) for _ in range(world * 3)]
    return B, H, D, max_len, prompt, k_new, v_new, pos, steps


def _rope_cache_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from lwm_b200.kv_cache import ShardedKVCache

        class CpuCache(ShardedKVCache):
            write_rope = staticmethod(_write_rope_cpu)

        B, H, D, max_len, prompt, k_new, v_new, pos, steps = _problem(world)
        table = _table(1 << 16)
        cache = CpuCache(B, max_len, H, D, dtype=torch.float32, device="cpu")
        ql = prompt // world
        mine = slice(rank * ql, (rank + 1) * ql)
        cache.concatenate(k_new[:, mine], v_new[:, mine], freqs_cis=table, position_ids=pos[:, mine])      # prefill
        for i, (kk, vv) in enumerate(steps):                                                             # decode
            ck, cv = cache.concatenate(kk, vv, freqs_cis=table, position_ids=pos[:, -1:] + 1 + i)
        ret[rank] = (ck.numpy(), cv.numpy(), cache.cache_index)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2, 4])
def test_rotating_cache_write_matches_the_unsharded_update(world):
    import torch.multiprocessing as mp
    B, H, D, max_len, prompt, k_new, v_new, pos, steps = _problem(world)
    inv = _table(1 << 16).inv_freq
    ref_k, ref_v = torch.zeros(B, max_len, H, D), torch.zeros(B, max_len, H, D)
    ref_k[:, :prompt], ref_v[:, :prompt] = _rope_cpu(k_new, pos, inv), v_new
    idx = prompt
    for i, (kk, vv) in enumerate(steps):
        ref_k[:, idx], ref_v[:, idx] = _rope_cpu(kk, pos[:, -1:] + 1 + i, inv)[:, -1], vv[:, -1]
        idx += 1
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ret = mp.Manager().dict()
    mp.spawn(_rope_cache_worker, args=(world, port, ret), nprocs=world, join=True)
    L = max_len // world
    for r in range(world):
        ck, cv, ci = ret[r]
        assert ci == idx
        assert np.array_equal(ck, ref_k[:, r * L:(r + 1) * L].numpy())
        assert np.array_equal(cv, ref_v[:, r * L:(r + 1) * L].numpy())
