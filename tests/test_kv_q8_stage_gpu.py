"""GPU tests of the tensor-core paths reading the 8-bit KV cache directly (lwm_kv_q8_absmax, lwm_kv_q8_stage):
  * kernels: the |max| bits and the staged fp16 / e4m3 bytes from the codes equal lwm_attn_absmax /
    lwm_attn_to_f16_scaled / lwm_attn_to_e4m3_scaled on the cache dequantized to fp32 and to bf16, on caches with NaN
    codes, all-zero groups and rows, exponents -126 and 121 and groups far below the tensor max (fp16 and e4m3
    subnormals and zeros), whole and one batch row at a time;
  * ops, bit for bit against the same call on ck.dequantize(q.dtype), cv.dequantize(q.dtype): ringattention in the
    fp16, bf16 and fp8 modes (q bf16 and fp32, with and without the rotary keywords, bias or segment ids, Sq != Sk,
    causal and not), ringattention_inference at Q = 8, 16, 300 on one GPU and on the q-sharded protocol (threads,
    world 2 and 4), and the peer-memory executor (ranks as threads, world 2 and 4) in the fp16, fp8 and bf16 ops;
  * no copy: the fp16- and fp8-mode calls run with QuantizedKV.dequantize patched to raise, and the peak memory of the
    cached prefill is below the explicit-dequantize composition's by at least the dequantized K + V bytes."""
import threading

import pytest
import torch

from thread_comm import run_ranks

pytestmark = pytest.mark.gpu
D = 128


def _ra():
    from lwm_b200 import ringattention as ra
    return ra


def _same(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape
    assert torch.equal(torch.isnan(a), torch.isnan(b))
    a0, b0 = torch.nan_to_num(a, nan=0.0), torch.nan_to_num(b, nan=0.0)
    bad = (a0 != b0).nonzero()
    assert bad.numel() == 0, [(tuple(i.tolist()), a0[tuple(i)].item(), b0[tuple(i)].item()) for i in bad[:8]]


def _same_f16(a, b):
    """fp16 bits: the same NaN positions, every other element bit for bit (signed zeros included)"""
    assert a.dtype == b.dtype == torch.float16 and a.shape == b.shape
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb)
    ai, bi = a.view(torch.int16), b.view(torch.int16)
    bad = ((ai != bi) & ~na).nonzero()
    assert bad.numel() == 0, [(tuple(i.tolist()), a[tuple(i)].item(), b[tuple(i)].item()) for i in bad[:8]]


def _same_e4m3(a, b):
    """e4m3 bytes: the same NaN positions (0x7f / 0xff), every other byte equal"""
    a, b = a.view(torch.uint8), b.view(torch.uint8)
    na, nb = (a & 0x7f) == 0x7f, (b & 0x7f) == 0x7f
    assert torch.equal(na, nb)
    bad = ((a != b) & ~na).nonzero()
    assert bad.numel() == 0, [(tuple(i.tolist()), a[tuple(i)].item(), b[tuple(i)].item()) for i in bad[:8]]


def _no_dequantize(monkeypatch):
    from lwm_b200.kv_cache import QuantizedKV

    def refuse(self, dtype):
        raise AssertionError("the 8-bit cache was dequantized")
    monkeypatch.setattr(QuantizedKV, "dequantize", refuse)


def _randn(shape, seed, dtype=torch.float32):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(shape, generator=g, device="cuda").to(dtype)


def _quantized(k, v):
    """QuantizedKV caches holding k / v [B,L,H,128] (bf16 or fp32), written by lwm_kv_cache_write_q8"""
    from lwm_b200.kv_cache import QuantizedKV, kv_cache_write_q8
    B, L, H, _ = k.shape
    ck, cv = QuantizedKV.zeros(B, L, H), QuantizedKV.zeros(B, L, H)
    kv_cache_write_q8(k.contiguous(), v.contiguous(), 0, L, ck, cv, 0)
    return ck, cv


def _kv(B, Sk, H, seed, dtype):
    """8-bit k / v caches of random rows whose magnitudes vary by 2^-8 .. 2^8 from row to row"""
    g = torch.Generator(device="cuda").manual_seed(seed + 1000)
    kv = []
    for i in range(2):
        x = _randn((B, Sk, H, D), seed + i, torch.float32)
        x *= torch.exp2(torch.randint(-8, 9, (B, Sk, H, 1), generator=g, device="cuda").float())
        kv.append(x.to(dtype))
    return _quantized(*kv)


def _table():
    from lwm_b200.rope import precompute_freqs_cis
    return precompute_freqs_cis(128, 1 << 16, 1e4, device="cuda")


# ------------------------------------------------------------------------------------------------
# the kernels against the passes on the dequantized cache
# ------------------------------------------------------------------------------------------------
def _codes_cache(B, L, H, case, seed):
    """a QuantizedKV [B,L,H,128] made from codes and exponents directly. case: 'typical' (exponents -16 .. -2),
    'spread' (-40 .. 1: most groups far below the tensor max, staged as subnormals or zeros), 'extremes' (-126 .. 121,
    both ends present), 'no_finite' (only NaN and zero codes: scale 1)"""
    from lwm_b200.kv_cache import QuantizedKV
    g = torch.Generator().manual_seed(seed)
    data = torch.randint(-127, 128, (B, L, H, D), dtype=torch.int8, generator=g)
    lo, hi = {"typical": (-16, -1), "spread": (-40, 2), "extremes": (-126, 122), "no_finite": (-3, 3)}[case]
    exp = torch.randint(lo, hi, (B, H, L, 4), dtype=torch.int8, generator=g)
    if case == "extremes":
        exp[0, 0, 0, 0], exp[B - 1, H - 1, L - 1, 3] = -126, 121
    if case == "no_finite":
        data = torch.where(torch.rand(data.shape, generator=g) < 0.5, -128, 0).to(torch.int8)
    data.view(-1)[::97] = -128                    # NaN codes
    data[0, 0, 0, 32:64] = 0                      # an all-zero group
    data[B - 1, L - 1, H - 1] = 0                 # an all-zero row
    return QuantizedKV(data.cuda(), exp.cuda())


@pytest.mark.parametrize("case", ["typical", "spread", "extremes", "no_finite"])
@pytest.mark.parametrize("H", [1, 3, 32])
@pytest.mark.parametrize("L", [1, 3, 129, 2049])
def test_absmax_and_staging_equal_the_passes_on_the_dequantized_cache(L, H, case):
    ra = _ra()
    B = 2
    c = _codes_cache(B, L, H, case, seed=L * 131 + H)
    bits8 = torch.zeros(1, dtype=torch.int32, device="cuda")
    ra.kv_q8_absmax(c, bits8)
    rows8 = torch.zeros(1, dtype=torch.int32, device="cuda")
    for b in range(B):
        ra.kv_q8_absmax(c[b], rows8)
    assert torch.equal(rows8, bits8)
    if case == "no_finite":
        assert int(bits8) == 0
    for dt in (torch.float32, torch.bfloat16):
        x = c.dequantize(dt)
        bits = torch.zeros(1, dtype=torch.int32, device="cuda")
        ra.PeerOpsF16.absmax(x, bits)                                     # lwm_attn_absmax
        assert torch.equal(bits8, bits), (dt, int(bits8), int(bits))
        for ops, code, same in ((ra.PeerOpsF16, 2, _same_f16), (ra.PeerOpsE4m3, 3, _same_e4m3)):
            s, s8 = (torch.empty(1, dtype=torch.float32, device="cuda") for _ in range(2))
            ops.scale_of(x, s)
            ops.scale_of(c, s8)
            assert torch.equal(s, s8), (ops.__name__, dt, s.item(), s8.item())
            ref = torch.empty(x.shape, dtype=ops.op_dtype, device="cuda")
            ops.stage(x, ref, s)                          # lwm_attn_to_f16_scaled / lwm_attn_to_e4m3_scaled
            got = torch.full(x.shape, 1.0, dtype=torch.float32, device="cuda").to(ops.op_dtype)
            ra.kv_q8_stage(c, got, code, s)
            same(got, ref)
            by_row = torch.full(x.shape, 1.0, dtype=torch.float32, device="cuda").to(ops.op_dtype)
            for b in range(B):
                ops.stage(c[b], by_row[b], s)
            same(by_row, ref)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------
# ringattention
# ------------------------------------------------------------------------------------------------
# (Sq, Sk, causal, mask): the cached prefill (Sq < Sk) with the call-site bias, causal and not, with segment ids, and
# Sq == Sk
PREFILLS = [(256, 1024, False, "bias"), (256, 1024, True, "bias"), (256, 1024, True, "seg"), (512, 512, True, "bias")]


def _mask_args(kind, B, Sq, Sk, dtype):
    if kind == "bias":
        bias = torch.zeros(B, 1, 1, Sk, device="cuda", dtype=dtype)
        bias[0, ..., :100] = torch.finfo(dtype).min
        bias[-1, ..., 300:317] = torch.finfo(dtype).min
        return bias, None
    S = max(Sq, Sk)
    seg = torch.zeros(B, S, dtype=torch.int32, device="cuda")
    seg[:, S // 3:] = 1
    seg[-1, 2 * S // 3:] = 2
    return None, seg


@pytest.mark.parametrize("rope", [False, True], ids=["plain", "rope"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("precision", ["fp16", "bf16", "fp8"])
def test_ringattention_on_the_cache_equals_the_dequantized_call(precision, dtype, rope, monkeypatch):
    ra = _ra()
    B, H = 2, 4
    table = _table()
    cases = []
    with torch.no_grad():
        for i, (Sq, Sk, causal, kind) in enumerate(PREFILLS):
            q = _randn((B, Sq, H, D), 31 + i, dtype)
            ck, cv = _kv(B, Sk, H, 41 + 2 * i, dtype)
            bias, seg = _mask_args(kind, B, Sq, Sk, dtype)
            kw = dict(blockwise_kwargs=dict(causal_block_size=1 if causal else None), precision=precision)
            if rope:
                pos = (torch.arange(Sq, dtype=torch.int32, device="cuda") + Sk - Sq)[None].repeat(B, 1)
                kw.update(freqs_cis=table, position_ids=pos, rotate_k=False)
            ref = ra.ringattention(q, ck.dequantize(dtype), cv.dequantize(dtype), bias, seg, **kw)
            cases.append((q, ck, cv, bias, seg, kw, ref))
        if precision != "bf16":      # the bf16 mode dequantizes into its bf16 operands (exact)
            _no_dequantize(monkeypatch)
        for q, ck, cv, bias, seg, kw, ref in cases:
            out = ra.ringattention(q, ck, cv, bias, seg, **kw)
            assert out.dtype == dtype
            _same(out, ref)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------
# ringattention_inference with tensor cores
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Q", [8, 16, 300])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_inference_on_the_cache_equals_the_dequantized_call(dtype, Q, monkeypatch):
    ra = _ra()
    B, H, Sk = 2, 4, 1000
    q = _randn((B, Q, H, D), 50 + Q, dtype)
    ck, cv = _kv(B, Sk, H, 60, dtype)
    kd, vd = ck.dequantize(dtype), cv.dequantize(dtype)
    mask = torch.rand(B, 1, Q, Sk, generator=torch.Generator().manual_seed(Q)).cuda() < 0.8
    mask[0, 0, 1] = False                           # a row without a visible key
    pos = (torch.arange(Q, dtype=torch.int32, device="cuda") + Sk - Q)[None].repeat(B, 1)
    table = _table()
    kws = ({}, dict(freqs_cis=table, position_ids=pos, rotate_k=False))
    with torch.no_grad():
        refs = [ra.ringattention_inference(q, kd, vd, m, **kw) for kw in kws for m in (mask, None)]
        _no_dequantize(monkeypatch)
        outs = [ra.ringattention_inference(q, ck, cv, m, **kw) for kw in kws for m in (mask, None)]
    for o, r in zip(outs, refs):
        _same(o, r)
    torch.cuda.synchronize()


@pytest.mark.parametrize("world,Ql", [(2, 8), (4, 3)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_sharded_inference_on_the_cache_equals_the_dequantized_call(dtype, world, Ql, monkeypatch):
    """the q-sharded protocol with world * Q_loc >= INFER_MIN_Q rows (tensor cores), ranks as threads"""
    ra = _ra()
    from lwm_b200.kv_cache import QuantizedKV
    assert world * Ql >= ra.INFER_MIN_Q
    B, H, Sl = 2, 2, 700
    q = _randn((B, world * Ql, H, D), 70 + world, dtype)
    ck, cv = _kv(B, world * Sl, H, 80 + world, dtype)
    kd, vd = ck.dequantize(dtype), cv.dequantize(dtype)
    mask = (torch.rand(B, 1, world * Ql, world * Sl, generator=torch.Generator().manual_seed(world)) < 0.7).cuda()
    pos = torch.arange(world * Ql, dtype=torch.int32, device="cuda")[None].repeat(B, 1) + world * (Sl - Ql)
    inv = _table().inv_freq
    _no_dequantize(monkeypatch)

    def rank_fn(r, comm):
        rows, keys = slice(r * Ql, (r + 1) * Ql), slice(r * Sl, (r + 1) * Sl)
        k8 = QuantizedKV(ck.data[:, keys].contiguous(), ck.exp[:, :, keys].contiguous())
        v8 = QuantizedKV(cv.data[:, keys].contiguous(), cv.exp[:, :, keys].contiguous())
        res = []
        with torch.no_grad():
            for rope in (None, (pos[:, rows].contiguous(), None, inv)):
                o8 = ra._infer_sharded(q[:, rows].contiguous(), k8, v8, mask[:, :, rows], comm, rope=rope)
                o = ra._infer_sharded(q[:, rows].contiguous(), kd[:, keys].contiguous(), vd[:, keys].contiguous(),
                                      mask[:, :, rows], comm, rope=rope)
                res.append((o8, o))
        return res

    for res in run_ranks(world, rank_fn):
        for o8, o in res:
            _same(o8, o)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------
# the peer-memory executor, ranks as threads on one GPU
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("ops_name,dtype", [("PeerOpsF16", torch.float32), ("PeerOpsF16", torch.bfloat16),
                                            ("PeerOpsE4m3", torch.float32), ("PeerOpsE4m3", torch.bfloat16),
                                            ("PeerOpsBf16", torch.bfloat16)],
                         ids=["f16-fp32", "f16-bf16", "e4m3-fp32", "e4m3-bf16", "bf16-bf16"])
def test_peer_ring_on_the_cache_equals_the_dequantized_shards(ops_name, dtype, world, monkeypatch):
    """rp.run_forward on each rank's 8-bit shards (staged into the heap one batch row at a time, from the codes) and on
    the same shards dequantized: the same output bits"""
    ra = _ra()
    from lwm_b200 import ring_peer as rp, ring_schedule as rs
    from lwm_b200.kv_cache import QuantizedKV
    from peer_emulation import EmuTransport, EmuWorld
    ops = getattr(ra, ops_name)
    B, Sl, H, causal = 2, 256, 2, True
    q = _randn((B, world * Sl, H, D), 90 + world, dtype)
    ck, cv = _kv(B, world * Sl, H, 95 + world, dtype)
    kd, vd = ck.dequantize(dtype), cv.dequantize(dtype)
    bias = torch.zeros(B, world * Sl, device="cuda")
    bias[0, 37:300] = torch.finfo(torch.float32).min
    _no_dequantize(monkeypatch)
    dev = torch.device("cuda", 0)
    emu = EmuWorld(world, device=dev)
    outs, fails = {}, []

    def worker(rank):
        try:
            torch.cuda.set_device(dev)
            tr = EmuTransport(emu, rank)
            plan = rs.make_peer_plan(world, rank, Sl, Sl, causal, "zigzag")
            sl = slice(rank * Sl, (rank + 1) * Sl)
            k8 = QuantizedKV(ck.data[:, sl].contiguous(), ck.exp[:, :, sl].contiguous())
            v8 = QuantizedKV(cv.data[:, sl].contiguous(), cv.exp[:, :, sl].contiguous())
            with torch.no_grad():
                for name, k, v in (("q8", k8, v8), ("deq", kd[:, sl].contiguous(), vd[:, sl].contiguous())):
                    out, _ = rp.run_forward(plan, q[:, sl].contiguous(), k, v, bias, None, causal, ops, tr,
                                            dtype == torch.float32)
                    outs[(name, rank)] = out
        except BaseException:   # noqa: BLE001  (reported by the main thread)
            import traceback
            fails.append(traceback.format_exc())
            emu.barrier.abort()

    ts = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    torch.cuda.synchronize()
    assert not any(t.is_alive() for t in ts) and not fails, fails[:1]
    for r in range(world):
        _same(outs[("q8", r)], outs[("deq", r)])


# ------------------------------------------------------------------------------------------------
# memory
# ------------------------------------------------------------------------------------------------
def _peak_above(fn):
    """-> (fn's result, peak allocated bytes during fn above what was allocated before it)"""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


@pytest.mark.parametrize("precision", ["fp16", "fp8"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_cached_prefill_allocates_no_dequantized_shard(dtype, precision):
    """B = 1, H = 32, 4096 queries against a 32768-key cache, causal, with the call-site bias: the call on the cache
    peaks at least the dequantized K + V bytes (1 GiB in fp32, 512 MiB in bf16) below the explicit composition"""
    ra = _ra()
    B, H, Sq, Sk = 1, 32, 4096, 32768
    q = _randn((B, Sq, H, D), 7, dtype)
    ck, cv = _kv(B, Sk, H, 8, dtype)
    bias = torch.zeros(B, 1, 1, Sk, device="cuda", dtype=dtype)
    kw = dict(blockwise_kwargs=dict(causal_block_size=1), precision=precision)
    with torch.no_grad():
        ref, peak_deq = _peak_above(lambda: ra.ringattention(q, ck.dequantize(dtype), cv.dequantize(dtype), bias, **kw))
        out, peak_q8 = _peak_above(lambda: ra.ringattention(q, ck, cv, bias, **kw))
    _same(out, ref)
    dequantized = 2 * B * Sk * H * D * torch.empty((), dtype=dtype).element_size()
    print("%s %s: peak above the inputs %.1f MiB (dequantize first) -> %.1f MiB (from the codes), saved %.1f MiB"
          % (precision, dtype, peak_deq / 2 ** 20, peak_q8 / 2 ** 20, (peak_deq - peak_q8) / 2 ** 20))
    assert peak_deq - peak_q8 >= dequantized, (peak_deq, peak_q8, dequantized)
