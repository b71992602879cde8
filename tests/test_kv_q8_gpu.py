"""GPU tests of the 8-bit KV cache (lwm_b200/csrc/kv_q8.cuh, DESIGN.md §5):
  * write: every byte of data and exp equals the torch reference quantizer (tests/kv_q8_model.py), for bf16 and fp32
    sources, with and without the rotary embedding (reference: lwm_kv_cache_write_rope into a source-dtype cache, then
    the reference quantizer), decode and prefill writes, and rows of NaN, +-inf, zeros, tiny and huge magnitudes;
  * decode: the GEMV kernel on the 8-bit cache is bit-identical to the same call on cache.dequantize(q.dtype), for q
    bf16 / fp32, masked or not, with and without q rotation, at the kernel's split and warp edges, at 131072 and
    2^20 + 3 keys, and on the replicated and the q-sharded ring protocols emulated with threads;
  * prefill and multi-row: ringattention(..., rotate_k=False) and ringattention_inference with Q >= 8 equal the calls on
    the dequantized cache;
  * end to end: a 4096-row prefill through ShardedKVCache.concatenate with the rotary keywords and 64 decode steps;
  * error against float64 attention on the un-quantized cache at 131072 keys, within the float64 model's prediction;
  * memory: B*L*H*264 bytes per rank."""
import math

import pytest
import torch

import kv_q8_model as m8
import score_distributions as sd
from thread_comm import run_ranks

pytestmark = pytest.mark.gpu
D = 128
SPLIT_SKS = [1, 3, 4, 15, 16, 17, 2047, 2048, 2049, 4097, 6145, 256 * 2048 + 1]


def _randn(shape, seed, scale=1.0, dtype=torch.float32):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


def _quantized(k, v):
    """QuantizedKV caches holding k / v [B,L,H,128] (bf16 or fp32), written by lwm_kv_cache_write_q8"""
    from lwm_b200.kv_cache import QuantizedKV, kv_cache_write_q8
    B, L, H, _ = k.shape
    ck, cv = QuantizedKV.zeros(B, L, H), QuantizedKV.zeros(B, L, H)
    kv_cache_write_q8(k.contiguous(), v.contiguous(), 0, L, ck, cv, 0)
    return ck, cv


def _same(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape
    assert torch.equal(torch.isnan(a), torch.isnan(b))
    a0, b0 = torch.nan_to_num(a, nan=0.0), torch.nan_to_num(b, nan=0.0)
    bad = (a0 != b0).nonzero()
    assert bad.numel() == 0, [(tuple(i.tolist()), a0[tuple(i)].item(), b0[tuple(i)].item()) for i in bad[:8]]


def _table():
    from lwm_b200.rope import precompute_freqs_cis
    return precompute_freqs_cis(128, 1 << 21, 1e4, device="cuda")


# ------------------------------------------------------------------------------------------------
# the write
# ------------------------------------------------------------------------------------------------
def _special_rows(x):
    """plant non-finite, zero, tiny and huge rows and groups into x [B,n,H,128] (fp32 values)"""
    x[0, 0, 0, 3] = math.nan
    x[0, 0, 0, 40] = math.inf
    x[0, 0, 1, 77] = -math.inf
    x[0, 0, 1, 96:] = 0.0                                   # an all-zero group
    if x.shape[1] > 1:
        x[0, 1, 0] = 0.0                                    # an all-zero row
        x[1, 1, 1, :32] = math.nan                          # a group without a finite element
    x[1, 0, 0] *= 2.0 ** -125                               # tiny: below the exponent clamp, partly subnormal
    x[1, 0, 1] *= 2.0 ** 120                                # huge
    x[1, -1, 0, :64] = 3.0e38
    return x


@pytest.mark.parametrize("n,src0,dst0", [(1, 0, 5), (37, 3, 11)], ids=["decode", "prefill"])
@pytest.mark.parametrize("rope", [False, True], ids=["plain", "rope"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_write_bytes_match_the_reference_quantizer(dtype, rope, n, src0, dst0):
    from lwm_b200.kv_cache import QuantizedKV, kv_cache_write_q8, kv_cache_write_rope
    B, H, L, n_src = 2, 3, 64, src0 + n + 2
    seed = 7 * n + rope + 2 * (dtype == torch.float32)
    k = _special_rows(_randn((B, n_src, H, D), seed) * 4.0).to(dtype)
    v = _special_rows(_randn((B, n_src, H, D), seed + 1)).to(dtype)
    pos = inv = None
    if rope:
        pos = (torch.arange(n_src, device="cuda", dtype=torch.int32)[None].repeat(B, 1) * 37 + 1000).contiguous()
        inv = _table().inv_freq
    ck, cv = QuantizedKV.zeros(B, L, H), QuantizedKV.zeros(B, L, H)
    kv_cache_write_q8(k, v, src0, n, ck, cv, dst0, pos, inv)
    if rope:        # the reference rows: the rope write into a cache of the source dtype
        rk, rv = torch.zeros(B, L, H, D, dtype=dtype, device="cuda"), torch.zeros(B, L, H, D, dtype=dtype, device="cuda")
        kv_cache_write_rope(k, v, src0, n, rk, rv, dst0, pos, inv)
        k_rows, v_rows = rk[:, dst0:dst0 + n], rv[:, dst0:dst0 + n]
    else:
        k_rows, v_rows = k[:, src0:src0 + n], v[:, src0:src0 + n]
    torch.cuda.synchronize()
    for cache, rows in ((ck, k_rows), (cv, v_rows)):
        codes, exps = m8.quantize_rows(rows.float())
        assert torch.equal(cache.data[:, dst0:dst0 + n], codes)
        assert torch.equal(cache.exp[:, :, dst0:dst0 + n], exps.permute(0, 2, 1, 3))
        untouched = torch.ones(L, dtype=torch.bool)
        untouched[dst0:dst0 + n] = False
        assert not cache.data[:, untouched].any() and not cache.exp[:, :, untouched].any()
        # the dequantization is exact: it equals the model's values in either dtype
        ref = m8.from_cache(cache.data, cache.exp)
        for out_dtype in (torch.float32, torch.bfloat16):
            _same(cache.dequantize(out_dtype).double(), ref)


# ------------------------------------------------------------------------------------------------
# decode: bit-identical to the call on the dequantized cache
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Sk", SPLIT_SKS)
@pytest.mark.parametrize("Q", [1, 3, 7])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_decode_partials_at_split_and_warp_edges(Sk, Q, dtype):
    from lwm_b200 import ringattention as ra
    B, H, W = 2, 2, 4
    gen = torch.Generator().manual_seed(Sk * 10 + Q)
    mask = (torch.rand(B, 1, Q, W * Sk, generator=gen) < 0.5).to(torch.uint8).cuda()
    seed = 3 * Sk + Q + (dtype == torch.float32)
    q = _randn((B, Q, H, D), seed, 1.0, dtype)
    ck, cv = _quantized(_randn((B, Sk, H, D), seed + 1, 0.5, dtype), _randn((B, Sk, H, D), seed + 2, 64.0, dtype))
    kd, vd = ck.dequantize(dtype), cv.dequantize(dtype)
    for r, m in ((3, mask), (0, None)):
        o8, ml8 = ra.decode_partial(q, ck, cv, m, r * Sk)
        o, ml = ra.decode_partial(q, kd, vd, m, r * Sk)
        torch.cuda.synchronize()
        assert torch.equal(o8, o) and torch.equal(ml8, ml), (r, Sk, Q)


@pytest.mark.parametrize("rope", [False, True], ids=["plain", "rope"])
@pytest.mark.parametrize("masked", [True, False], ids=["pad", "nomask"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("K", [131072, 2 ** 20 + 3])
def test_long_cache_decode_is_bit_identical(K, dtype, masked, rope):
    from lwm_b200 import ringattention as ra
    B, H = 2, 2
    seed = K + 4 * (dtype == torch.float32) + 2 * masked + rope
    q = _randn((B, 1, H, D), seed, 1.0, dtype)
    ck, cv = _quantized(_randn((B, K, H, D), seed + 1, 1.0, dtype), _randn((B, K, H, D), seed + 2, 1.0, dtype))
    mask = None
    if masked:
        pad = torch.ones(B, K, dtype=torch.int32, device="cuda")
        pad[0, :1000] = 0
        pad[1, :K // 3 + 1] = 0
        mask = ra.decode_attention_mask(pad, 1, K - 9, K)
    kw = {}
    if rope:
        kw = dict(freqs_cis=_table(), position_ids=torch.full((B, 1), K - 9, dtype=torch.int32), rotate_k=False)
    with torch.no_grad():
        out8 = ra.ringattention_inference(q, ck, cv, mask, **kw)
        out = ra.ringattention_inference(q, ck.dequantize(dtype), cv.dequantize(dtype), mask, **kw)
    torch.cuda.synchronize()
    assert out8.dtype == dtype and torch.equal(out8, out)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_replicated_ring_is_bit_identical(world, dtype):
    from lwm_b200 import ringattention as ra
    B, H, Sl = 2, 3, 2500
    q = _randn((B, 1, H, D), 11 * world, 1.0, dtype)
    k = torch.cat([_randn((B, Sl, H, D), 100 * world + r, 2.0 ** -r, dtype) for r in range(world)], 1)
    v = torch.cat([_randn((B, Sl, H, D), 200 * world + r, 2.0 ** (3 * r), dtype) for r in range(world)], 1)
    ck, cv = _quantized(k, v)
    kd, vd = ck.dequantize(dtype), cv.dequantize(dtype)
    pad = torch.ones(B, world * Sl, dtype=torch.int32, device="cuda")
    pad[0, :Sl + 17] = 0
    mask = ra.decode_attention_mask(pad, 1, world * Sl - 5, world * Sl)

    def shard(c, r):
        from lwm_b200.kv_cache import QuantizedKV
        return QuantizedKV(c.data[:, r * Sl:(r + 1) * Sl].contiguous(), c.exp[:, :, r * Sl:(r + 1) * Sl].contiguous())

    def rank_fn(r, comm):
        keys = slice(r * Sl, (r + 1) * Sl)
        o8 = ra._infer_replicated(q, shard(ck, r), shard(cv, r), mask, r, comm)
        o = ra._infer_replicated(q, kd[:, keys].contiguous(), vd[:, keys].contiguous(), mask, r, comm)
        return o8, o

    outs = run_ranks(world, rank_fn)
    torch.cuda.synchronize()
    for o8, o in outs:
        assert torch.equal(o8, o) and torch.equal(o8, outs[0][0])


@pytest.mark.parametrize("world,Ql", [(2, 2), (2, 3), (4, 1)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_sharded_ring_gemv_is_bit_identical(world, Ql, dtype):
    """the q-sharded protocol below INFER_MIN_Q rows (the GEMV path) on threads: bit-identity only (DESIGN §3.6)"""
    from lwm_b200 import ringattention as ra
    from lwm_b200.kv_cache import QuantizedKV
    B, H, Sl = 2, 2, 3000
    q = _randn((B, world * Ql, H, D), 5 * world + Ql, 1.0, dtype)
    ck, cv = _quantized(_randn((B, world * Sl, H, D), 9, 1.0, dtype), _randn((B, world * Sl, H, D), 10, 1.0, dtype))
    kd, vd = ck.dequantize(dtype), cv.dequantize(dtype)
    mask = (torch.rand(B, 1, world * Ql, world * Sl, generator=torch.Generator().manual_seed(world)) < 0.7).cuda()
    pos = torch.arange(world * Ql, dtype=torch.int32, device="cuda")[None].repeat(B, 1) + world * Sl - world * Ql
    inv = _table().inv_freq

    def rank_fn(r, comm):
        rows, keys = slice(r * Ql, (r + 1) * Ql), slice(r * Sl, (r + 1) * Sl)
        k8 = QuantizedKV(ck.data[:, keys].contiguous(), ck.exp[:, :, keys].contiguous())
        v8 = QuantizedKV(cv.data[:, keys].contiguous(), cv.exp[:, :, keys].contiguous())
        res = []
        for rope in (None, (pos[:, rows].contiguous(), None, inv)):
            o8 = ra._infer_sharded(q[:, rows].contiguous(), k8, v8, mask[:, :, rows], comm, rope=rope)
            o = ra._infer_sharded(q[:, rows].contiguous(), kd[:, keys].contiguous(), vd[:, keys].contiguous(),
                                  mask[:, :, rows], comm, rope=rope)
            res.append((o8, o))
        return res

    for res in run_ranks(world, rank_fn):
        for o8, o in res:
            assert torch.equal(o8, o)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------
# prefill and multi-row calls: the dequantized shard through the existing ops
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_prefill_and_multi_row_calls_equal_the_dequantized_cache(dtype):
    from lwm_b200 import ringattention as ra
    B, H, Sq, Sk = 1, 4, 512, 2048
    q = _randn((B, Sq, H, D), 21, 1.0, dtype)
    ck, cv = _quantized(_randn((B, Sk, H, D), 22, 1.0, dtype), _randn((B, Sk, H, D), 23, 1.0, dtype))
    kd, vd = ck.dequantize(dtype), cv.dequantize(dtype)
    table = _table()
    pos = (torch.arange(Sq, dtype=torch.int32, device="cuda") + Sk - Sq)[None]
    bias = torch.zeros(B, 1, 1, Sk, device="cuda", dtype=dtype)
    bias[..., :100] = torch.finfo(dtype).min
    with torch.no_grad():
        for kw in ({}, dict(freqs_cis=table, position_ids=pos, rotate_k=False)):
            out8 = ra.ringattention(q, ck, cv, bias, None, **kw)
            out = ra.ringattention(q, kd, vd, bias, None, **kw)
            assert torch.equal(out8, out)
        mask = torch.ones(B, 1, 16, Sk, dtype=torch.bool, device="cuda")
        mask[..., :33] = False
        for kw in ({}, dict(freqs_cis=table, position_ids=pos[:, :16], rotate_k=False)):
            out8 = ra.ringattention_inference(q[:, :16], ck, cv, mask, **kw)
            out = ra.ringattention_inference(q[:, :16], kd, vd, mask, **kw)
            assert torch.equal(out8, out)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------
# end to end on one GPU
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_prefill_then_decode_through_the_cache(dtype):
    from lwm_b200 import ringattention as ra
    from lwm_b200.kv_cache import QuantizedKV, ShardedKVCache
    B, H, prompt, steps, max_len = 1, 4, 4096, 64, 4224    # the prefill op takes whole 128-key tiles of the cache
    table = _table()
    cache = ShardedKVCache(B, max_len, H, D, dtype=torch.int8)
    xq, xk, xv = (_randn((B, prompt, H, D), 30 + i, 1.0, dtype) for i in range(3))
    pos = torch.arange(prompt, dtype=torch.int32, device="cuda")[None]
    pad = torch.ones(B, max_len, dtype=torch.int32, device="cuda")
    with torch.no_grad():
        ck, cv = cache.concatenate(xk, xv, freqs_cis=table, position_ids=pos)
        assert isinstance(ck, QuantizedKV)
        kw = dict(freqs_cis=table, position_ids=pos, rotate_k=False)
        # the cached prefill (the scan branch): q against the whole cache
        out8 = ra.ringattention(xq, ck, cv, None, None, **kw)
        out = ra.ringattention(xq, ck.dequantize(dtype), cv.dequantize(dtype), None, None, **kw)
        assert torch.equal(out8, out)
        for i in range(steps):
            q1, k1, v1 = (_randn((B, 1, H, D), 1000 + 3 * i + j, 1.0, dtype) for j in range(3))
            p1 = torch.full((B, 1), prompt + i, dtype=torch.int32, device="cuda")
            ck, cv = cache.concatenate(k1, v1, freqs_cis=table, position_ids=p1)
            mask = ra.decode_attention_mask(pad, 1, prompt + i, max_len)
            kw = dict(freqs_cis=table, position_ids=p1, rotate_k=False)
            out8 = ra.ringattention_inference(q1, ck, cv, mask, **kw)
            out = ra.ringattention_inference(q1, ck.dequantize(dtype), cv.dequantize(dtype), mask, **kw)
            assert torch.equal(out8, out), i
    assert cache.cache_index == prompt + steps
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------
# error against the un-quantized cache
# ------------------------------------------------------------------------------------------------
ERROR_CASES = ["noise1", "noise3", "sink", "recency", "peaked"]
ERR_TOL = {torch.float32: 1e-5, torch.bfloat16: 3e-3}


def _error_problem(case, H, K):
    """q [1,1,H,D], k, v [1,K,H,D] float32 on the device"""
    if case.startswith("noise"):
        sigma = float(case[5:])
        return _randn((1, 1, H, D), 51, sigma), _randn((1, K, H, D), 52), _randn((1, K, H, D), 53)
    kw = dict(gap=18.0) if case == "sink" else {}
    q = sd.shard(case, "q", K - 128, 128, K, H, **kw)[:, -1:]         # the last position's query row
    k = sd.shard(case, "k", 0, K, K, H, **kw)
    v = sd.shard(case, "v", 0, K, K, H, **kw)
    return q.cuda(), k.cuda(), v.cuda()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("case", ERROR_CASES)
def test_error_against_the_unquantized_cache(case, dtype):
    from lwm_b200 import ringattention as ra
    H, K = 4, 131072
    q, k, v = _error_problem(case, H, K)
    q, k, v = q.to(dtype), k.to(dtype), v.to(dtype)
    predicted, ref = m8.predicted_error(q, k, v)
    ck, cv = _quantized(k, v)
    with torch.no_grad():
        out8 = ra.ringattention_inference(q, ck, cv, None)
        out = ra.ringattention_inference(q, k, v, None)
    err8, err = m8.row_error(out8, ref), m8.row_error(out, ref)
    print("kv_q8 error %-8s q %s: int8 cache %.2e (model %.2e), %s cache %.2e"
          % (case, str(dtype)[6:], err8, predicted, str(dtype)[6:], err))
    assert err8 <= predicted + ERR_TOL[dtype], (err8, predicted)


# ------------------------------------------------------------------------------------------------
# memory
# ------------------------------------------------------------------------------------------------
def test_cache_allocates_264_bytes_per_key_and_head():
    from lwm_b200.kv_cache import ShardedKVCache
    B, L, H = 2, 4096, 32
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    cache = ShardedKVCache(B, L, H, D, dtype=torch.int8)
    after = torch.cuda.memory_allocated()
    assert cache.cached_key.nbytes + cache.cached_value.nbytes == B * L * H * 264
    assert after - before == B * L * H * 264
