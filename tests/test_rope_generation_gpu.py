"""The rotary embedding inside the generation path, on an H100: keys rotated as they enter the KV cache
(`ShardedKVCache.concatenate(freqs_cis=, position_ids=)`), queries rotated inside `ringattention_inference` and the
cached prefill (`ringattention(rotate_k=False)`).

Contract: each fused call is bit-identical to the composition on the same inputs (apply_rotary_emb, then the plain
cache update, then the plain op): outputs, dK and dV are torch.equal; dQ may differ by the order of the backward
kernels' fp32 dQ sums, so it is held to the larger of a small bound and twice the composition's own run-to-run spread.

  * kernels: lwm_attn_decode_partial_rope(_f32) against lwm_attn_rope + lwm_attn_decode_partial(_f32) at the split and
    warp edges of the GEMV kernel; lwm_kv_cache_write_rope against lwm_attn_rope + copy_ at decode slots and at prefill
    slices that straddle shard boundaries;
  * the ops on one GPU; the replicated and q-sharded protocols on threads (tests/thread_comm.py); the cached prefill on
    the peer-memory executor (tests/peer_emulation.py); a left-padded prefill + 16 decode steps end to end."""
import threading

import pytest
import torch

from helpers import rel_fro, to_np

pytestmark = pytest.mark.gpu
D = 128
TOL_DQ = {torch.float32: 1e-5, torch.bfloat16: 4e-3}
DT = {torch.float32: 0, torch.bfloat16: 1}


def _table(theta, max_position):
    from lwm_b200.rope import precompute_freqs_cis
    return precompute_freqs_cis(D, max_position, theta)


def _rope(x, pos, table, conj=False):
    """lwm_attn_rope on one tensor, in its dtype"""
    from lwm_b200 import _lib
    B, S, H, _ = x.shape
    y = torch.empty(x.shape, dtype=x.dtype, device=x.device)
    p = pos.to(torch.int32).contiguous()
    _lib.call("lwm_attn_rope", _lib.ptr(x.contiguous()), None, DT[x.dtype], _lib.ptr(y), None, DT[x.dtype],
              _lib.ptr(p), _lib.ptr(table.inv_freq), B, S, H, 0, D, int(conj), _lib.stream_ptr())
    return y


def _randn(shape, seed, dtype, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


def _eq(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, what
    assert torch.equal(a, b), "%s differs: max |diff| %.3e" % (what, float((a.float() - b.float()).abs().max()))


# ------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------
SPLIT_SKS = [1, 3, 4, 15, 16, 17, 2047, 2048, 2049, 4097, 6145, 256 * 2048 + 1]
THETAS = [(1e4, 0), (5e7, (1 << 20) - 9), (1e7, 12345)]


@pytest.mark.parametrize("Sk", SPLIT_SKS)
@pytest.mark.parametrize("Q", [1, 3, 7])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_rotating_decode_partial_is_rope_then_the_plain_partial(Sk, Q, dtype):
    from lwm_b200 import ringattention as ra
    B, H = (2, 2) if Sk < 100000 else (1, 2)
    theta, off = THETAS[(Sk + Q) % len(THETAS)]
    table = _table(theta, off + 4096)
    q = _randn((B, Q, H, D), Sk + Q, dtype, 3.0)
    k = _randn((B, Sk, H, D), Sk + Q + 1, dtype)
    v = _randn((B, Sk, H, D), Sk + Q + 2, dtype)
    g = torch.Generator().manual_seed(Sk)
    pos = (off + torch.randint(0, 4096, (B, Q), generator=g)).to(torch.int32).cuda()
    mask = (torch.rand(B, 1, Q, 2 * Sk, generator=g) < 0.5).to(torch.uint8).cuda()
    mask[..., Sk + Sk // 2] = 1
    for m, k_pos0 in ((None, 0), (mask, Sk)):
        o_ref, ml_ref = ra.decode_partial(_rope(q, pos, table), k, v, m, k_pos0)
        o, ml = ra.decode_partial(q, k, v, m, k_pos0, rope=(pos, table.inv_freq))
        _eq(o, o_ref, "o_part")
        _eq(ml, ml_ref, "ml_part")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("B,H", [(1, 32), (3, 2)])
def test_cache_write_is_rope_then_copy(B, H, dtype):
    """decode slots (first, last, middle row of a shard) and the prefill slices of a 4-way ring whose new rows straddle
    shard boundaries"""
    from lwm_b200.kv_cache import kv_cache_write_rope
    theta, off = THETAS[B % len(THETAS)]
    table = _table(theta, off + 8192)
    L, W = 96, 4
    ck = _randn((B, L, H, D), 1, dtype)
    cv = _randn((B, L, H, D), 2, dtype)
    # decode: one new row
    for i, dst in enumerate((0, L - 1, 37)):
        k1, v1 = _randn((B, 1, H, D), 10 + i, dtype, 4.0), _randn((B, 1, H, D), 20 + i, dtype)
        p1 = (off + 5000 + torch.arange(B)[:, None] * 7 + i).to(torch.int32).cuda()
        want_k, want_v = ck.clone(), cv.clone()
        want_k[:, dst].copy_(_rope(k1, p1, table)[:, -1])
        want_v[:, dst].copy_(v1[:, -1])
        kv_cache_write_rope(k1, v1, 0, 1, ck, cv, dst, p1, table.inv_freq)
        _eq(ck, want_k, "decode k")
        _eq(cv, want_v, "decode v")
    # prefill: n_new = 150 rows from cache_index 30 over 4 shards of L rows
    ci, n_new = 30, 150
    kn, vn = _randn((B, n_new, H, D), 30, dtype, 4.0), _randn((B, n_new, H, D), 31, dtype)
    pn = (off + torch.arange(n_new)[None].repeat(B, 1) + torch.arange(B)[:, None]).to(torch.int32).cuda()
    kr = _rope(kn, pn, table)
    for r in range(W):
        lo = r * L
        a, b = max(ci, lo), min(ci + n_new, lo + L)
        if b <= a:
            continue
        sk, sv = _randn((B, L, H, D), 40 + r, dtype), _randn((B, L, H, D), 50 + r, dtype)
        want_k, want_v = sk.clone(), sv.clone()
        want_k[:, a - lo:b - lo].copy_(kr[:, a - ci:b - ci])
        want_v[:, a - lo:b - lo].copy_(vn[:, a - ci:b - ci])
        kv_cache_write_rope(kn, vn, a - ci, b - a, sk, sv, a - lo, pn, table.inv_freq)
        _eq(sk, want_k, "prefill k, shard %d" % r)
        _eq(sv, want_v, "prefill v, shard %d" % r)


# ------------------------------------------------------------------------------------------------
# ringattention_inference on one GPU
# ------------------------------------------------------------------------------------------------
def _gen_mask(B, Q, K, cache_index):
    """the generation mask: left padding AND causal from cache_index (decode_attention_mask)"""
    from lwm_b200.ringattention import decode_attention_mask
    am = torch.ones(B, K, dtype=torch.int64)
    for b in range(B):
        am[b, :3 + 5 * b] = 0
    return decode_attention_mask(am.cuda(), Q, cache_index, K)


def _infer_run(q, k, v, mask, table, pos, rotate_k, fused, do):
    from lwm_b200.rope import apply_rotary_emb, rotate
    from lwm_b200.ringattention import ringattention_inference
    q, k, v = [t.detach().clone().requires_grad_(True) for t in (q, k, v)]
    if fused:
        out = ringattention_inference(q, k, v, mask, freqs_cis=table, position_ids=pos, rotate_k=rotate_k)
    elif rotate_k:
        out = ringattention_inference(*apply_rotary_emb(q, k, table, q.dtype, position_ids=pos), v, mask)
    else:
        out = ringattention_inference(rotate(q, table, q.dtype, position_ids=pos.to(torch.int32)), k, v, mask)
    out.backward(do)
    return out.detach(), q.grad, k.grad, v.grad


def _assert_same(run, dtype):
    """dtype: the operand precision that bounds dQ (bf16 for fp32 inputs in the bf16 precision mode)"""
    ref, ref2, got = run(False), run(False), run(True)
    for n, a, b in zip(("out", "dq", "dk", "dv"), got, ref):
        if n != "dq":
            _eq(a, b, n)
    spread = rel_fro(to_np(ref2[1]), to_np(ref[1]))
    err = rel_fro(to_np(got[1]), to_np(ref[1]))
    assert err <= max(TOL_DQ[dtype], 2 * spread), (err, spread)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("Q", [1, 4, 8, 300])
@pytest.mark.parametrize("K", [4096, 131072])
@pytest.mark.parametrize("masked", [True, False], ids=["generation_mask", "no_mask"])
def test_inference_with_a_rotated_cache_is_the_composition(masked, K, Q, dtype):
    B, H = 2, 2
    theta, off = THETAS[(K + Q) % len(THETAS)]
    table = _table(theta, off + K + 8)
    q, k, v, do = (_randn((B, Q, H, D), s, dtype) for s in (K + Q, K + Q + 1, K + Q + 2, K + Q + 3))
    k = _randn((B, K, H, D), K + Q + 1, dtype)
    v = _randn((B, K, H, D), K + Q + 2, dtype)
    ci = K - Q - 5
    pos = (off + ci + torch.arange(Q)[None].repeat(B, 1)).cuda()
    mask = _gen_mask(B, Q, K, ci) if masked else None
    _assert_same(lambda fused: _infer_run(q, k, v, mask, table, pos, False, fused, do), dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("S", [1, 4, 8, 300])
def test_inference_rotating_q_and_k_is_the_composition(S, dtype):
    """training's non-scan branch: q and k are the same rows, under the causal + padding mask"""
    from lwm_b200.ringattention import causal_attention_mask
    B, H = 2, 2
    theta, off = THETAS[S % len(THETAS)]
    table = _table(theta, off + S + 8)
    q, k, v, do = (_randn((B, S, H, D), 7 * S + i, dtype) for i in range(4))
    am = torch.ones(B, S, dtype=torch.int64)
    am[1, :S // 3] = 0
    p = am.cumsum(-1) - 1
    pos = torch.where(am > 0, p, torch.zeros_like(p)).cuda() + off     # left padding mapped into the table
    mask = causal_attention_mask(am.cuda())
    _assert_same(lambda fused: _infer_run(q, k, v, mask, table, pos, True, fused, do), dtype)


# ------------------------------------------------------------------------------------------------
# ringattention(rotate_k=False): the cached prefill on one GPU
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("Sq,Sk", [(128, 512), (256, 1024), (1024, 1024)])
def test_cached_prefill_is_the_composition(Sq, Sk, dtype, precision):
    from lwm_b200.rope import rotate
    from lwm_b200.ringattention import attention_bias_from_mask, ringattention
    B, H = 2, 2
    theta, off = THETAS[Sq % len(THETAS)]
    table = _table(theta, off + Sk + 8)
    q, do = _randn((B, Sq, H, D), Sq, dtype), _randn((B, Sq, H, D), Sq + 1, dtype)
    k, v = _randn((B, Sk, H, D), Sk + 2, dtype), _randn((B, Sk, H, D), Sk + 3, dtype)
    am = torch.ones(B, Sk, dtype=torch.int64)
    am[0, :7] = 0
    am[1, Sk - 50:] = 0
    bias = attention_bias_from_mask(am.cuda(), torch.float32 if dtype == torch.float32 else torch.bfloat16)
    pos = (off + torch.arange(Sq)[None].repeat(B, 1)).cuda()

    def run(fused):
        qq, kk, vv = [t.detach().clone().requires_grad_(True) for t in (q, k, v)]
        if fused:
            out = ringattention(qq, kk, vv, bias, precision=precision, freqs_cis=table, position_ids=pos, rotate_k=False)
        else:
            out = ringattention(rotate(qq, table, dtype, position_ids=pos.to(torch.int32)), kk, vv, bias,
                                precision=precision)
        out.backward(do)
        return out.detach(), qq.grad, kk.grad, vv.grad
    _assert_same(run, torch.bfloat16 if precision == "bf16" else dtype)


# ------------------------------------------------------------------------------------------------
# emulated rings: the inference protocols on threads, the prefill on the peer executor
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_replicated_protocol_rotates_the_same_query_on_every_rank(world, dtype):
    from lwm_b200 import ringattention as ra
    from thread_comm import run_ranks
    B, H, Sl = 2, 2, 4096
    table = _table(5e7, (1 << 20) + 8)
    q = _randn((B, 1, H, D), world, dtype)
    k, v = _randn((B, world * Sl, H, D), world + 1, dtype), _randn((B, world * Sl, H, D), world + 2, dtype)
    ci = world * Sl - 9
    mask = _gen_mask(B, 1, world * Sl, ci)
    pos = torch.full((B, 1), (1 << 20) - 3, dtype=torch.int32, device="cuda")
    qr = _rope(q, pos, table)

    def body(r, comm):
        kl, vl = k[:, r * Sl:(r + 1) * Sl].contiguous(), v[:, r * Sl:(r + 1) * Sl].contiguous()
        got = ra._infer_replicated(q, kl, vl, mask, r, comm, rope=(pos, None, table.inv_freq))
        want = ra._infer_replicated(qr, kl, vl, mask, r, comm)
        torch.cuda.synchronize()
        return got, want
    for got, want in run_ranks(world, body):
        _eq(got, want, "out")


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("Ql", [1, 2, 40])
@pytest.mark.parametrize("rotate_k", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_sharded_protocol_is_the_composition(world, Ql, rotate_k, dtype):
    """q rows and their positions all-gathered and staged rotated (tensor cores from world*Q_loc >= INFER_MIN_Q, else
    the GEMV kernel); with tensor cores also the backward: dK, dV bit-identical, dQ summed in the same rank order"""
    from lwm_b200 import ringattention as ra
    from thread_comm import run_ranks
    B, H = 2, 2
    Sl = Ql if rotate_k else 2048
    Qg, K = world * Ql, world * Sl
    table = _table(1e4, 1 << 16)
    q, do = _randn((B, Qg, H, D), Qg + world, dtype), _randn((B, Qg, H, D), Qg + world + 1, dtype)
    k, v = _randn((B, K, H, D), K + 2, dtype), _randn((B, K, H, D), K + 3, dtype)
    if rotate_k:
        from lwm_b200.ringattention import causal_attention_mask
        am = torch.ones(B, K, dtype=torch.int64)
        am[1, :K // 4] = 0
        mask = causal_attention_mask(am.cuda())
        pos = (am.cumsum(-1) - 1).clamp(min=0).cuda() + 100
    else:
        ci = K - Qg - 3
        mask = _gen_mask(B, Qg, K, ci)
        pos = (ci + torch.arange(Qg)[None].repeat(B, 1)).cuda()
    pos = pos.to(torch.int32)
    tc = Qg >= ra.INFER_MIN_Q
    qr, kr = _rope(q, pos, table), (_rope(k, pos, table) if rotate_k else k)

    def body(r, comm):
        rows, keys = slice(r * Ql, (r + 1) * Ql), slice(r * Sl, (r + 1) * Sl)
        ql, pl, dl = q[:, rows].contiguous(), pos[:, rows].contiguous(), do[:, rows].contiguous()
        ml = mask[:, :, rows]
        res = []
        for fused in (True, False):
            qq = ql if fused else qr[:, rows].contiguous()
            kk = (k if fused else kr)[:, keys].contiguous()
            vl = v[:, keys].contiguous()
            rope = (pl, pl if rotate_k else None, table.inv_freq) if fused else None
            saved = {} if tc else None
            out = ra._infer_sharded(qq, kk, vl, ml, comm, saved=saved, rope=rope)
            grads = ()
            if tc:
                dq, dk, dv = ra._infer_sharded_bwd(saved, dl, comm, inv_freq=table.inv_freq)
                if not fused:
                    dq = _rope(dq, pl, table, conj=True)
                    dk = _rope(dk, pl, table, conj=True) if rotate_k else dk
                grads = (dq, dk, dv)
            res.append((out,) + grads)
        torch.cuda.synchronize()
        return res
    for got, want in run_ranks(world, body):
        for n, a, b in zip(("out", "dq", "dk", "dv"), got, want):
            if n == "dq":
                assert rel_fro(to_np(a), to_np(b)) <= TOL_DQ[dtype]
            else:
                _eq(a, b, n)


@pytest.mark.parametrize("world", [2, 4])
def test_cached_prefill_on_the_peer_ring_is_the_composition(world):
    """run_forward / run_backward with rope_k=False: q rotated in its staging, k taken as the rotated cache; dQ gets
    the conjugate rotation on its way back to its owner, dK is the gradient w.r.t. the cache as passed"""
    from lwm_b200 import ring_peer as rp, ring_schedule as rs
    from lwm_b200.ringattention import PeerOpsBf16, PeerOpsF16
    from peer_emulation import EmuTransport, EmuWorld
    B, H, Sl = 2, 2, 256
    S = world * Sl
    dev = torch.device("cuda", 0)
    table = _table(5e7, (1 << 20) + 16)
    passes = []
    for prec in ("fp16", "bf16"):
        for dt in (torch.float32, torch.bfloat16):
            q, k, v, do = (_randn((B, S, H, D), world * 10 + i, dt) for i in range(4))
            pos = ((1 << 20) - S - 3 + torch.arange(S)[None].repeat(B, 1)).to(torch.int32).cuda()
            passes.append((prec, dt, (q, k, v, do, pos)))
    emu = EmuWorld(world, device=dev)
    results, fails = {}, []

    def worker(rank):
        try:
            torch.cuda.set_device(dev)
            tr = EmuTransport(emu, rank)
            plan = rs.make_peer_plan(world, rank, Sl, Sl, True, "contiguous")
            sl = slice(rank * Sl, (rank + 1) * Sl)
            mine = []
            for prec, dt, (q, k, v, do, pos) in passes:
                ops = PeerOpsF16 if prec == "fp16" else PeerOpsBf16
                want_f32 = dt == torch.float32
                ql, kl, vl, dl = [t[:, sl].contiguous() for t in (q, k, v, do)]
                pl = pos[:, sl].contiguous()
                rope = (pl, table.inv_freq)
                out, res = rp.run_forward(plan, ql, kl, vl, None, None, True, ops, tr, want_f32, rope, False)
                dq, dk, dv = rp.run_backward(plan, res, kl, vl, dl, None, None, True, ops, tr, want_f32, rope, False)
                fused = (out, dq, dk, dv)
                qr = _rope(ql, pl, table)
                out, res = rp.run_forward(plan, qr, kl, vl, None, None, True, ops, tr, want_f32)
                dqr, dk, dv = rp.run_backward(plan, res, kl, vl, dl, None, None, True, ops, tr, want_f32)
                mine.append((fused, (out, _rope(dqr, pl, table, conj=True), dk, dv)))
            torch.cuda.synchronize()
            results[rank] = mine
        except BaseException:   # noqa: BLE001  (reported by the main thread)
            import traceback
            fails.append((rank, traceback.format_exc()))
            emu.barrier.abort()

    ts = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    torch.cuda.synchronize()
    assert not any(t.is_alive() for t in ts), "rank threads did not finish"
    assert not fails, fails[0][1]
    for r in range(world):
        for i, (fused, comp) in enumerate(results[r]):
            dt = passes[i][1]
            for n, a, b in zip(("out", "dq", "dk", "dv"), fused, comp):
                if n == "dq":
                    assert rel_fro(to_np(a), to_np(b)) <= TOL_DQ[dt], (r, i)
                else:
                    _eq(a, b, "%s rank %d pass %d" % (n, r, i))


# ------------------------------------------------------------------------------------------------
# end to end: a left-padded prefill through the cache, then 16 decode steps
# ------------------------------------------------------------------------------------------------
def _e2e_inputs(dtype, prompt, steps):
    B, H = 2, 4
    am = torch.ones(B, prompt + steps, dtype=torch.int64)
    am[1, :11] = 0                                   # left padding of the second sequence
    p = am.cumsum(-1) - 1
    pos = torch.where(am > 0, p, torch.zeros_like(p)).cuda()    # padded rows (-1 in the reference) mapped to 0
    g = [_randn((B, prompt + steps, H, D), 70 + i, dtype) for i in range(3)]
    return B, H, am.cuda(), pos, g


def _e2e(rank, comm, world, dtype, fused, prompt=256, steps=16, max_len=512):
    from lwm_b200.kv_cache import ShardedKVCache
    from lwm_b200.ringattention import decode_attention_mask, _infer_replicated, _infer_sharded, ringattention_inference
    from lwm_b200.rope import apply_rotary_emb
    B, H, am, pos, (q, k, v) = _e2e_inputs(dtype, prompt, steps)
    table = _table(1e4, 4096)
    pad = torch.cat([am, torch.zeros(B, max_len - am.shape[1], dtype=am.dtype, device="cuda")], 1)
    cache = ShardedKVCache(B, max_len, H, D, dtype=dtype, comm=comm)
    outs = []

    def attend(qq, ck, cv, mask, p):
        qq = qq.contiguous()            # (the protocol functions take contiguous rows, as ringattention_inference passes)
        kw = dict(freqs_cis=table, position_ids=p, rotate_k=False) if fused else {}
        if not fused:
            qq = apply_rotary_emb(qq, qq[:, :, :0], table, dtype, position_ids=p)[0]
        if comm is None:
            return ringattention_inference(qq, ck, cv, mask, **kw)
        rope = (p.to(torch.int32), None, table.inv_freq) if fused else None
        if qq.shape[1] == 1:
            return _infer_replicated(qq, ck, cv, mask, rank, comm, rope=rope)
        return _infer_sharded(qq, ck, cv, mask, comm, rope=rope)

    def write(kk, vv, p):
        if fused:
            return cache.concatenate(kk, vv, freqs_cis=table, position_ids=p)
        return cache.concatenate(apply_rotary_emb(kk, kk[:, :, :0], table, dtype, position_ids=p)[0], vv)

    ql = prompt // world
    rows = slice(rank * ql, (rank + 1) * ql)
    ck, cv = write(k[:, rows], v[:, rows], pos[:, rows])
    mask = decode_attention_mask(pad, prompt, 0, max_len)[:, :, rows]
    outs.append(attend(q[:, rows], ck, cv, mask, pos[:, rows]))
    for t in range(prompt, prompt + steps):
        ck, cv = write(k[:, t:t + 1], v[:, t:t + 1], pos[:, t:t + 1])
        mask = decode_attention_mask(pad, 1, t, max_len)
        outs.append(attend(q[:, t:t + 1], ck, cv, mask, pos[:, t:t + 1]))
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("world", [1, 4])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_left_padded_generation_end_to_end(world, dtype):
    from thread_comm import run_ranks
    if world == 1:
        res = [[_e2e(0, None, 1, dtype, fused) for fused in (True, False)]]
    else:
        res = run_ranks(world, lambda r, comm: [_e2e(r, comm, world, dtype, fused) for fused in (True, False)])
    for r, (got, want) in enumerate(res):
        assert len(got) == 17
        for i, (a, b) in enumerate(zip(got, want)):
            _eq(a, b, "rank %d step %d" % (r, i))
