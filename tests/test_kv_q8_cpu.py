"""The 8-bit KV cache without a GPU:
  * the format (tests/kv_q8_model.py) against its definition on sweeps: the exponent rule, half-to-even rounding, the
    +-127 clamp, the NaN code, all-zero groups and groups at the exponent clamp;
  * the exactness claim, exhaustively: every code at every exponent dequantizes exactly to fp32 and to bf16;
  * the C ABI of the two new entry points and of lwm_attn_decode_partial's 8-bit cache arguments: declared, exported
    and bound, and bad arguments rejected before the device check;
  * ShardedKVCache(dtype=torch.int8) bookkeeping under gloo at world 1, 2 and 4, with a CPU stand-in for the
    quantizing write: a prefill whose slice crosses rank boundaries, decode writes on rank edges, and overflow."""
import ctypes
import math
import os
import socket

import numpy as np
import pytest
import torch

import kv_q8_model as m8
from helpers import abi_row_id

P = ctypes.c_void_p(0x1000)
P_ODD = ctypes.c_void_p(0x1001)
N = None
SHAPE, ARG, DEVICE = 2, 3, 1


def _q(row):
    """one 128-element row -> (codes list, exps list)"""
    codes, exps = m8.quantize_rows(torch.tensor(row, dtype=torch.float32)[None])
    return codes[0].tolist(), exps[0].tolist()


# ------------------------------------------------------------------------------------------------
# the format
# ------------------------------------------------------------------------------------------------
def test_exponent_rule_on_a_magnitude_sweep():
    g = torch.Generator().manual_seed(0)
    for p in range(-149, 128):
        for mant in (1.0, 1.4999, 1.5, 1.99999):
            mx = mant * 2.0 ** p
            if not math.isfinite(mx) or np.float32(mx) == 0 or np.isinf(np.float32(mx)):
                continue
            x = (torch.rand(128, generator=g) * 2 - 1) * float(np.float32(mx))
            x[5] = float(np.float32(mx))
            x[37], x[70], x[101] = -float(np.float32(mx)), float(np.float32(mx)) / 3, float(np.float32(mx))
            codes, exps = m8.quantize_rows(x[None])
            m = float(np.float32(mx))
            want = min(max(math.floor(math.log2(m)) - 6, m8.EXP_MIN), m8.EXP_MAX)
            assert exps[0].tolist()[0] == want, (p, mant)
            assert abs(codes[0, 5].item()) <= 127


def test_round_half_to_even_and_the_127_clamp():
    row = [0.0] * 128
    row[0] = 64.0                      # group 0: m = 64 -> e = 0
    row[1], row[2], row[3], row[4] = 2.5, 3.5, -2.5, -0.5
    row[5] = 126.5                     # rounds to 126 (even)
    row[32] = 127.5                    # group 1: e = 0, rounds to 128 -> clamped to 127
    row[33] = -127.5
    row[64] = 64.0 * 2 ** -20          # group 2: e = -20
    row[65] = 1.5 * 2 ** -20           # 1.5 -> 2
    codes, exps = _q(row)
    assert exps == [0, 0, -20, 0]
    assert codes[1:6] == [2, 4, -2, 0, 126]
    assert codes[32:34] == [127, -127]
    assert codes[64:66] == [64, 2]


def test_nan_code_and_zero_groups():
    row = [0.0] * 128
    row[0], row[1], row[2] = math.nan, math.inf, -math.inf
    row[3] = 3.0                       # group 0: finite max 3 -> e = -5
    row[96] = -0.0                     # group 3: all zeros, one negative zero
    row[40] = math.nan                 # group 1: no finite nonzero element
    codes, exps = _q(row)
    assert codes[:4] == [-128, -128, -128, 96]
    assert exps == [-5, 0, 0, 0]
    assert codes[40] == -128 and codes[96] == 0
    back = m8.dequantize_rows(torch.tensor(codes, dtype=torch.int8)[None], torch.tensor(exps, dtype=torch.int8)[None])
    assert torch.isnan(back[0, :3]).all() and back[0, 3] == 3.0 and torch.isnan(back[0, 40])


def test_groups_at_the_exponent_clamp():
    tiny = float(np.float32(2.0 ** -130))         # below 2^-120: e clamps to -126, small elements flush to 0
    row = [0.0] * 128
    row[0], row[1] = tiny, float(np.float32(2.0 ** -149))
    row[32] = float(np.float32(2.0 ** -119))      # just above the clamp: e = -125
    row[64] = float(np.finfo(np.float32).max)     # e = 121
    row[65] = -float(np.finfo(np.float32).max)
    codes, exps = _q(row)
    assert exps == [-126, -125, 121, 0]
    assert codes[0] == 0 and codes[1] == 0        # 2^-130 / 2^-126 = 1/16 -> 0
    assert codes[32] == 64
    assert codes[64:66] == [127, -127]            # (2 - 2^-23) * 2^127 / 2^121 = 128 - 2^-17 -> 128 -> 127


def test_round_trip_error_is_half_a_step():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(64, 128, generator=g) * torch.logspace(-30, 30, 64, base=2.0)[:, None]
    codes, exps = m8.quantize_rows(x)
    back = m8.dequantize_rows(codes, exps)
    step = torch.pow(2.0, exps.double()).repeat_interleave(32, -1)
    assert ((back - x.double()).abs() <= step / 2).all()


def test_every_code_at_every_exponent_is_exact_in_fp32_and_bf16():
    codes = torch.arange(-127, 128, dtype=torch.float64)                     # 255 codes (-128 is NaN)
    exps = torch.arange(m8.EXP_MIN, m8.EXP_MAX + 1, dtype=torch.float64)    # 248 exponents
    vals = codes[:, None] * torch.pow(2.0, exps)[None]
    assert torch.isfinite(vals).all()
    assert torch.equal(vals.float().double(), vals)
    assert torch.equal(vals.to(torch.bfloat16).double(), vals)


# ------------------------------------------------------------------------------------------------
# C ABI
# ------------------------------------------------------------------------------------------------
NEW_SYMBOLS = ("lwm_kv_cache_write_q8", "lwm_kv_dequant_q8")


def test_q8_symbols_are_declared_exported_and_bound(lib):
    from lwm_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "lwm_b200.h")).read()
    for name in NEW_SYMBOLS:
        assert "int %s(" % name in header
        assert hasattr(lib, name)
        assert name in _lib._SIGNATURES
    assert lib.lwm_abi_version() == 5


# lwm_kv_cache_write_q8(k_src, v_src, src_dtype, k_data, k_exp, v_data, v_exp, pos, inv_freq, B, n_src, src0, n, L,
#                       dst0, H, D, stream)
KW = (P, P, 1, P, P, P, P, N, N, 2, 8, 0, 8, 64, 0, 4, 128, N)
# lwm_attn_decode_partial(q, k, v, dtype, k_exp, v_exp, mask, o_part, ml_part, workspace, B, H, Q, Sk, D, k_pos0,
#                         mask_stride_b, mask_stride_q, splits, scale, pos, inv_freq, stream) on the 8-bit cache
DEC = (P, P, P, 1, P, P, N, P, P, P, 1, 2, 1, 128, 128, 0, 0, 0, 4, 0.1, N, N, N)
# lwm_kv_dequant_q8(data, exp, out, out_dtype, B, L, H, D, stream)
DQ = (P, P, P, 0, 2, 64, 4, 128, N)


def _with(args, **at):
    a = list(args)
    for k, val in at.items():
        a[int(k[1:])] = val
    return tuple(a)


BAD_CALLS = [
    ("lwm_kv_cache_write_q8", _with(KW, a16=64), SHAPE, "head_dim"),
    ("lwm_kv_cache_write_q8", _with(KW, a12=0), SHAPE, "bad sizes"),
    ("lwm_kv_cache_write_q8", _with(KW, a11=1), SHAPE, "out of range"),
    ("lwm_kv_cache_write_q8", _with(KW, a14=57), SHAPE, "out of range"),
    ("lwm_kv_cache_write_q8", _with(KW, a6=N), ARG, "null pointer"),
    ("lwm_kv_cache_write_q8", _with(KW, a7=P), ARG, "position_ids"),
    ("lwm_kv_cache_write_q8", _with(KW, a2=2), ARG, "dtype codes"),
    ("lwm_kv_cache_write_q8", _with(KW, a4=P_ODD), ARG, "aligned"),
    ("lwm_attn_decode_partial", _with(DEC, a14=64), SHAPE, "head_dim"),
    ("lwm_attn_decode_partial", _with(DEC, a3=3), ARG, "dtype codes"),
    ("lwm_attn_decode_partial", _with(DEC, a4=N), ARG, "null pointer"),       # v_exp without k_exp
    ("lwm_attn_decode_partial", _with(DEC, a9=N), ARG, "null pointer"),
    ("lwm_attn_decode_partial", _with(DEC, a21=P), ARG, "position_ids"),
    ("lwm_attn_decode_partial", _with(DEC, a5=P_ODD), ARG, "aligned"),
    ("lwm_attn_decode_partial", _with(DEC, a13=0), SHAPE, "bad shape"),
    ("lwm_kv_dequant_q8", _with(DQ, a7=64), SHAPE, "head_dim"),
    ("lwm_kv_dequant_q8", _with(DQ, a5=0), SHAPE, "bad sizes"),
    ("lwm_kv_dequant_q8", _with(DQ, a2=N), ARG, "null pointer"),
    ("lwm_kv_dequant_q8", _with(DQ, a3=2), ARG, "dtype codes"),
    ("lwm_kv_dequant_q8", _with(DQ, a0=P_ODD), ARG, "aligned"),
    ("lwm_attn_decode_partial", _with(DEC, a5=N), ARG, "null pointer"),       # k_exp without v_exp
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


GOOD_CALLS = [("lwm_kv_cache_write_q8", KW), ("lwm_kv_cache_write_q8", _with(KW, a7=P, a8=P, a2=0)),
              ("lwm_attn_decode_partial", DEC), ("lwm_attn_decode_partial", _with(DEC, a20=P, a21=P)),
              ("lwm_kv_dequant_q8", DQ), ("lwm_attn_decode_partial", _with(DEC, a3=0))]


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: only meaningful where the device check fails")
@pytest.mark.parametrize("name,args", GOOD_CALLS, ids=["%s-%d" % (abi_row_id(*c), i) for i, c in enumerate(GOOD_CALLS)])
def test_well_formed_calls_fail_with_device_error_without_gpu(lib, name, args):
    status, msg = _status(lib, name, *args)
    assert status == DEVICE, (status, msg)


# ------------------------------------------------------------------------------------------------
# the Python surface without a GPU
# ------------------------------------------------------------------------------------------------
def test_quantized_kv_enforces_the_format():
    from lwm_b200.kv_cache import QuantizedKV
    c = QuantizedKV.zeros(2, 16, 3, device="cpu")
    assert tuple(c.shape) == (2, 16, 3, 128) and tuple(c.exp.shape) == (2, 3, 16, 4)
    assert c.nbytes == 2 * 16 * 3 * 132 and c.dtype == torch.int8
    with pytest.raises(TypeError):
        QuantizedKV(c.data.float(), c.exp)
    with pytest.raises(ValueError, match="exp must be"):
        QuantizedKV(c.data, c.exp.transpose(1, 2).contiguous())
    with pytest.raises(ValueError, match="contiguous"):
        QuantizedKV(c.data, c.exp.transpose(1, 2).contiguous().transpose(1, 2))
    with pytest.raises(ValueError, match="dtype"):
        c.dequantize(torch.float16)
    from lwm_b200 import _lib
    with pytest.raises(_lib.LwmError, match="sm_90"):
        c.dequantize(torch.float32)


def test_attention_ops_reject_unsupported_quantized_calls():
    from lwm_b200.kv_cache import QuantizedKV
    from lwm_b200.ringattention import ringattention, ringattention_inference
    from lwm_b200.rope import precompute_freqs_cis
    c = QuantizedKV.zeros(1, 128, 2, device="cpu")
    q = torch.zeros(1, 1, 2, 128)
    plain = torch.zeros(1, 128, 2, 128)
    table = precompute_freqs_cis(128, 4096, 1e4, device="cpu")
    pos = torch.zeros(1, 1, dtype=torch.int32)
    for op in (ringattention_inference, ringattention):
        args = (None,) if op is ringattention_inference else (None, None)
        with pytest.raises(ValueError, match="both"):
            op(q, c, plain, *args)
        with pytest.raises(ValueError, match="both"):
            op(q, plain, c, *args)
        with pytest.raises(ValueError, match="bfloat16 or float32"):
            op(q.half(), c, c, *args)
        with pytest.raises(ValueError, match="rotate_k=False"):
            op(q, c, c, *args, freqs_cis=table, position_ids=pos, rotate_k=True)
        with pytest.raises(ValueError, match="generation only"):
            op(q.clone().requires_grad_(), c, c, *args)


# ------------------------------------------------------------------------------------------------
# ShardedKVCache(dtype=torch.int8) under gloo, with a CPU stand-in for lwm_kv_cache_write_q8
# ------------------------------------------------------------------------------------------------
def _rope_cpu(x, pos, inv_freq):
    """x [B,n,H,D] fp32 rotated at pos [B,n] (the table builder's float32 angles, a complex64 multiply)"""
    ang = (pos.double()[..., None] * inv_freq.double()).float()
    c, s = torch.cos(ang.double()).float()[:, :, None], torch.sin(ang.double()).float()[:, :, None]
    a, b = x[..., 0::2], x[..., 1::2]
    return torch.stack((a * c - b * s, a * s + b * c), dim=-1).reshape(x.shape)


def _write_q8_cpu(k_src, v_src, src0, n, cache_k, cache_v, dst0, pos=None, inv_freq=None):
    rows = slice(src0, src0 + n)
    k = k_src[:, rows].float()
    if pos is not None:
        k = _rope_cpu(k, pos[:, rows], inv_freq).to(k_src.dtype)
    for src, cache in ((k, cache_k), (v_src[:, rows], cache_v)):
        codes, exps = m8.quantize_rows(src)
        cache.data[:, dst0:dst0 + n] = codes
        cache.exp[:, :, dst0:dst0 + n] = exps.permute(0, 2, 1, 3)


def _problem(world):
    B, H, D, max_len = 2, 2, 128, 16 * world
    prompt = 9 * world                          # more than one rank's 16 slots: the prefill crosses rank boundaries
    g = torch.Generator().manual_seed(world + 10)
    k_new = torch.randn(B, prompt, H, D, generator=g) * torch.logspace(-8, 8, D, base=2.0)
    v_new = torch.randn(B, prompt, H, D, generator=g)
    k_new[0, 1, 0, :32] = 0.0                   # an all-zero group
    v_new[1, 2, 1, 7] = math.nan
    pos = (torch.arange(prompt)[None].repeat(B, 1) - torch.tensor([[0], [3]])).clamp(min=0) + 1000
    steps = [(torch.randn(B, 1, H, D, generator=g), torch.randn(B, 1, H, D, generator=g))
             for _ in range(max_len - prompt)]      # fill the cache to the last slot: decode writes on every rank edge
    return B, H, D, max_len, prompt, k_new, v_new, pos, steps


def _table():
    from lwm_b200.rope import precompute_freqs_cis
    return precompute_freqs_cis(128, 1 << 16, 1e4, device="cpu")


def _q8_cache_worker(rank, world, port, rope, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from lwm_b200.kv_cache import QuantizedKV, ShardedKVCache

        class CpuCache(ShardedKVCache):
            write_q8 = staticmethod(_write_q8_cpu)

        B, H, D, max_len, prompt, k_new, v_new, pos, steps = _problem(world)
        kw = lambda p: dict(freqs_cis=_table(), position_ids=p) if rope else {}    # noqa: E731
        cache = CpuCache(B, max_len, H, D, dtype=torch.int8, device="cpu")
        ql = prompt // world
        mine = slice(rank * ql, (rank + 1) * ql)
        ck, cv = cache.concatenate(k_new[:, mine], v_new[:, mine], **kw(pos[:, mine]))
        assert isinstance(ck, QuantizedKV) and isinstance(cv, QuantizedKV)
        for i, (kk, vv) in enumerate(steps):
            ck, cv = cache.concatenate(kk, vv, **kw(pos[:, -1:] + 1 + i))
        overflow = None
        try:
            cache.concatenate(k_new[:, :1].repeat(1, 2, 1, 1), v_new[:, :1].repeat(1, 2, 1, 1))
        except ValueError as e:
            overflow = str(e)
        ret[rank] = (ck.data.numpy(), ck.exp.numpy(), cv.data.numpy(), cv.exp.numpy(), cache.cache_index, overflow)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("rope", [False, True], ids=["plain", "rope"])
@pytest.mark.parametrize("world", [1, 2, 4])
def test_quantized_cache_write_matches_the_unsharded_update(world, rope):
    import torch.multiprocessing as mp
    B, H, D, max_len, prompt, k_new, v_new, pos, steps = _problem(world)
    inv = _table().inv_freq
    ref_k, ref_v = torch.zeros(B, max_len, H, D), torch.zeros(B, max_len, H, D)
    ref_k[:, :prompt] = _rope_cpu(k_new, pos, inv) if rope else k_new
    ref_v[:, :prompt] = v_new
    for i, (kk, vv) in enumerate(steps):
        ref_k[:, prompt + i] = (_rope_cpu(kk, pos[:, -1:] + 1 + i, inv) if rope else kk)[:, -1]
        ref_v[:, prompt + i] = vv[:, -1]
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ret = mp.Manager().dict()
    mp.spawn(_q8_cache_worker, args=(world, port, rope, ret), nprocs=world, join=True)
    L = max_len // world
    want = [m8.to_cache_layout(*m8.quantize_rows(t)) for t in (ref_k, ref_v)]
    for r in range(world):
        kd, ke, vd, ve, ci, overflow = ret[r]
        assert ci == max_len
        assert overflow is not None and "overflow" in overflow
        for (d, e), (wd, we) in zip(((kd, ke), (vd, ve)), want):
            assert np.array_equal(d, wd[:, r * L:(r + 1) * L].numpy())
            assert np.array_equal(e, we[:, :, r * L:(r + 1) * L].numpy())
