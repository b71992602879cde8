"""Attention dropout on the GPU: the device mask against its numpy restatement bit for bit, the public op and the step
functions against the float64 oracle under the same mask, reproducibility, the p = 0 / deterministic path, rows left
without a surviving key, a 32K-token sequence, and both ring executors with their ranks as threads on one GPU.

Tolerances are those of the same cases without dropout (tests/test_attn_public_op_gpu.py, tests/ring_emulated_inputs.py):
relative Frobenius error 1e-3 for fp32 results of the fp16 precision mode, 3e-3 for bf16 results, 5e-3 for the bf16
precision mode."""
import numpy as np
import pytest
import torch

from attn_dropout_model import attention_dropout_ref, drop_mask, drop_u16, threshold
from helpers import rel_fro, to_np

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _kw(p, seed, causal=True, deterministic=False):
    return dict(blockwise_kwargs=dict(causal_block_size=1 if causal else None, deterministic=deterministic,
                                      attn_pdrop=p, dropout_rng=seed))


def _tol(precision, dtype):
    if precision == "bf16":
        return 5e-3
    return 1e-3 if dtype == torch.float32 else 3e-3


def test_device_mask_is_the_numpy_mask():
    from lwm_b200 import _lib
    for seed, p, b, h, q0, k0, nq, nk in ((1, 0.1, 0, 0, 0, 0, 64, 512), (-7, 0.5, 3, 17, (1 << 20) - 40, 5, 96, 300),
                                         (2 ** 62 + 12345, 0.9, 1, 31, 1 << 20, (1 << 20) - 256, 128, 384)):
        thr = threshold(p)
        out = torch.empty(nq * nk, dtype=torch.uint8, device=DEV)
        _lib.call("lwm_attn_dropout_mask", seed, thr, b, h, q0, k0, nq, nk, _lib.ptr(out), _lib.stream_ptr())
        got = out.cpu().numpy().reshape(nq, nk).astype(bool)
        want = drop_u16(seed, b, h, q0 + np.arange(nq), k0 + np.arange(nk)) < thr
        assert np.array_equal(got, want), (seed, b, h)


def _masks(B, S, kind):
    from oracle.attn_dense import finfo_min
    if kind != "bias+seg":
        return None, None
    bias = torch.zeros(B, 1, 1, S)
    bias[0, ..., :45] = finfo_min("bf16")
    seg = torch.zeros(B, S, dtype=torch.int32)
    seg[:, S // 3:] = 1
    seg[B - 1, 2 * S // 3 + 7:] = 2
    return bias, seg


CASES = [  # causal, masks, B, Sq, Sk, H, precision, dtype
    (True, None, 1, 1024, 1024, 2, "fp16", torch.float32),
    (True, None, 1, 1024, 1024, 2, "fp16", torch.bfloat16),
    (True, None, 2, 512, 512, 3, "bf16", torch.bfloat16),
    (False, None, 1, 512, 1024, 2, "fp16", torch.float32),
    (False, None, 1, 1024, 512, 2, "bf16", torch.float32),
    (True, "bias+seg", 2, 1024, 1024, 2, "fp16", torch.float32),
    (True, "bias+seg", 2, 2048, 2048, 2, "bf16", torch.bfloat16),
    (False, "bias+seg", 1, 1024, 1024, 2, "fp16", torch.bfloat16),
]


@pytest.mark.parametrize("causal,masks,B,Sq,Sk,H,precision,dtype", CASES)
def test_op_matches_float64_oracle(causal, masks, B, Sq, Sk, H, precision, dtype):
    from lwm_b200 import ringattention as ra
    g = torch.Generator().manual_seed(Sq + Sk + H)
    q = torch.randn(B, Sq, H, 128, generator=g)
    k, v = [torch.randn(B, Sk, H, 128, generator=g) for _ in range(2)]
    do = torch.randn(B, Sq, H, 128, generator=g)
    if dtype == torch.bfloat16:
        q, k, v, do = [t.to(torch.bfloat16).float() for t in (q, k, v, do)]
    bias, seg = _masks(B, max(Sq, Sk), masks)
    seed, p = 1000 + Sq, 0.15
    qd, kd, vd = [t.to(DEV, dtype).requires_grad_(True) for t in (q, k, v)]
    out = ra.ringattention(qd, kd, vd, None if bias is None else bias.to(DEV), None if seg is None else seg.to(DEV),
                           precision=precision, **_kw(p, seed, causal))
    out.backward(do.to(DEV, dtype))
    torch.cuda.synchronize()
    drop = drop_mask(seed, threshold(p), B, H, 0, Sq, 0, Sk)
    ref = attention_dropout_ref(q.numpy(), k.numpy(), v.numpy(), do.numpy(), drop,
                                attn_bias=None if bias is None else bias.numpy(),
                                segment_ids=None if seg is None else seg.numpy(), causal=causal)
    tol = _tol(precision, dtype)
    for name, got, want in zip(("out", "dq", "dk", "dv"), (out, qd.grad, kd.grad, vd.grad), ref[:4]):
        got = to_np(got)
        assert np.isfinite(got).all(), name
        assert rel_fro(got, want) < tol, (name, rel_fro(got, want))
    dead = ~ref[4].transpose(0, 2, 1)      # rows without a surviving key (padding, or every visible key dropped)
    assert np.all(to_np(out)[dead] == 0) and np.all(to_np(qd.grad)[dead] == 0)


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
def test_rope_fused_call_equals_rotating_first(precision):
    from lwm_b200 import ringattention as ra
    from lwm_b200.rope import apply_rotary_emb, precompute_freqs_cis
    B, S, H = 1, 1024, 2
    table = precompute_freqs_cis(128, 4096)
    g = torch.Generator().manual_seed(3)
    q, k, v, do = [torch.randn(B, S, H, 128, generator=g).to(DEV, torch.bfloat16) for _ in range(4)]
    pos = (torch.arange(S, dtype=torch.int32) + 7)[None].to(DEV)
    kw = _kw(0.2, 99)
    res = []
    for fused in (True, False):
        qd, kd, vd = [t.clone().requires_grad_(True) for t in (q, k, v)]
        if fused:
            out = ra.ringattention(qd, kd, vd, precision=precision, freqs_cis=table, position_ids=pos, **kw)
        else:
            out = ra.ringattention(*apply_rotary_emb(qd, kd, table, qd.dtype, position_ids=pos), vd,
                                   precision=precision, **kw)
        out.backward(do)
        res.append([out.detach(), qd.grad, kd.grad, vd.grad])
    torch.cuda.synchronize()
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][3], res[1][3])
    for a, b in zip(res[0][1:3], res[1][1:3]):      # dQ (and dK through the rotation) up to their reduction order
        assert rel_fro(to_np(a), to_np(b)) < _tol(precision, torch.bfloat16)


def _run_op(q, k, v, do, **kw):
    from lwm_b200 import ringattention as ra
    qd, kd, vd = [t.clone().requires_grad_(True) for t in (q, k, v)]
    out = ra.ringattention(qd, kd, vd, **kw)
    out.backward(do)
    torch.cuda.synchronize()
    return [out.detach(), qd.grad, kd.grad, vd.grad]


def _qkv(B=1, S=1024, H=2, seed=4):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, S, H, 128, generator=g).to(DEV, torch.bfloat16) for _ in range(4)]


def test_no_dropout_is_the_plain_path():
    """deterministic=True, or attn_pdrop = 0: the same bits and the same launches as a call without dropout kwargs
    (dQ compared under torch.use_deterministic_algorithms, which fixes its reduction order)"""
    from torch.profiler import ProfilerActivity, profile
    q, k, v, do = _qkv()
    names = []
    outs = []
    torch.use_deterministic_algorithms(True)
    try:
        for kw in (dict(blockwise_kwargs=dict(causal_block_size=1)), _kw(0.3, 5, deterministic=True), _kw(0.0, 5),
                   _kw(2 ** -18, 5)):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                outs.append(_run_op(q, k, v, do, **kw))
            names.append([e.name for e in prof.events() if e.device_type.name == "CUDA"])
    finally:
        torch.use_deterministic_algorithms(False)
    for o, n in zip(outs[1:], names[1:]):
        assert all(torch.equal(a, b) for a, b in zip(outs[0], o))
        assert sorted(n) == sorted(names[0])
    assert any("attn_fwd_kernel" in n for n in names[0]) and any("attn_bwd_kernel" in n for n in names[0])


def test_same_seed_same_bits_other_seed_other_output():
    q, k, v, do = _qkv()
    torch.use_deterministic_algorithms(True)
    try:
        a = _run_op(q, k, v, do, **_kw(0.1, 42))
        b = _run_op(q, k, v, do, **_kw(0.1, 42))
    finally:
        torch.use_deterministic_algorithms(False)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    c = _run_op(q, k, v, do, **_kw(0.1, 43))
    assert not torch.equal(a[0], c[0])
    # dropout_rng=None: a seed from torch's default CPU generator
    torch.manual_seed(8)
    d = _run_op(q, k, v, do, **_kw(0.1, None))
    torch.manual_seed(8)
    e = _run_op(q, k, v, do, **_kw(0.1, None))
    assert torch.equal(d[0], e[0]) and torch.equal(d[2], e[2])


@pytest.mark.parametrize("f16", [False, True])
def test_map_steps_equal_plain_steps(f16):
    """fwd_step / bwd_step against mapped_fwd_step / mapped_bwd_step (block map) with dropout: out, lse, dK, dV bit
    for bit, dQ up to the order of its fp32 reductions. Two steps: a carry through the block map's clean tiles."""
    from lwm_b200 import ringattention as ra
    B, S, H = 2, 1024, 2
    half = S // 2
    q, k, v, do = _qkv(B, S, H, seed=11)
    bias = torch.zeros(B, S, device=DEV)       # the call site's zero bias: the map's tiles are all clean but causal ones
    bias[1, :200] = -3e38
    drop = (77, threshold(0.25))
    res = []
    for mapped in (False, True):
        fwd = ra.mapped_fwd_step if mapped else ra.fwd_step
        bwd = ra.mapped_bwd_step if mapped else ra.bwd_step
        sc, q16, k16, v16, d16 = None, q, k, v, do
        if f16:
            (q16, sq), (k16, sk), (v16, sv), (d16, sd) = [ra.to_f16(t) for t in (q, k, v, do)]
        out = torch.empty_like(q)
        o32 = torch.empty(q.shape, dtype=torch.float32, device=DEV) if f16 else None
        lse = torch.empty(B, H, S, device=DEV)
        acc = (torch.empty(B, S, H, 128, device=DEV), torch.empty(B, H, S, device=DEV), torch.empty(B, H, S, device=DEV))
        blocks = [(k0, k16[:, k0:k0 + half].contiguous(), v16[:, k0:k0 + half].contiguous()) for k0 in (0, half)]
        for i, (k0, kb, vb) in enumerate(blocks):
            kw = dict(scales=(sq, sk, sv), out_f32=o32) if f16 else {}
            fwd(q16, kb, vb, out, lse, *acc, 0, k0, True, bias, None, i == 0, i == 1, dropout=drop, **kw)
        delta = torch.empty(B, H, S, device=DEV)
        ra.bwd_prep(o32 if f16 else out, d16, delta, scale_do=sd if f16 else None)
        nlse = ra.lse_for_bwd(lse, f16=f16)
        dq = torch.zeros(B, S, H, 128, device=DEV)
        dks, dvs = [], []
        for k0, kb, vb in blocks:
            kw = dict(scales=(sq, sk, sv, sd)) if f16 else {}
            dks.append(torch.empty(B, half, H, 128, device=DEV))
            dvs.append(torch.empty(B, half, H, 128, device=DEV))
            bwd(q16, kb, vb, d16, nlse, delta, dq, dks[-1], dvs[-1], 0, k0, True, bias, None, init=True, dropout=drop,
                **kw)
        torch.cuda.synchronize()
        res.append((out, lse, dq, torch.cat(dks, 1), torch.cat(dvs, 1)))
    (o0, l0, q0, k0_, v0), (o1, l1, q1, k1, v1) = res
    assert torch.equal(o0, o1) and torch.equal(l0, l1) and torch.equal(k0_, k1) and torch.equal(v0, v1)
    assert float((q0 - q1).abs().max()) <= 1e-5 * float(q0.abs().max())


def test_row_whose_only_key_is_dropped():
    """causal row 0 sees key 0 only: find a seed that drops it (for head 0 of batch row 0) with the numpy mask"""
    p = 0.5
    thr = threshold(p)
    seed = next(s for s in range(1000) if drop_u16(s, 0, 0, [0], [0])[0, 0] < thr
                and drop_u16(s, 0, 1, [0], [0])[0, 0] >= thr)
    q, k, v, do = _qkv(1, 512, 2, seed=5)
    for precision in ("fp16", "bf16"):
        out, dq, dk, dv = _run_op(q, k, v, do, precision=precision, **_kw(p, seed))
        for t in (out, dq, dk, dv):
            assert torch.isfinite(t.float()).all()
        assert torch.all(out[0, 0, 0] == 0) and torch.all(dq[0, 0, 0] == 0)
        assert torch.any(out[0, 0, 1] != 0)          # head 1 keeps its key
        # the dropped entry gives key 0 nothing from row 0: with row 0's dO negated, dK and dV do not change (they are
        # accumulated in a fixed order, so any contribution would show in the bits; negation keeps |dO|max, and with
        # it the fp16 mode's power-of-two scale of dO)
        do2 = do.clone()
        do2[0, 0, 0] = -do[0, 0, 0]
        _, dq2, dk2, dv2 = _run_op(q, k, v, do2, precision=precision, **_kw(p, seed))
        assert torch.equal(dk, dk2) and torch.equal(dv, dv2) and torch.all(dq2[0, 0, 0] == 0)


def test_32k_tokens_against_row_oracle():
    """S = 32768, causal, fp16 mode: sampled query rows of out / dq, and dk / dv of every key row (their sums run over
    all queries), against float64 under the same mask"""
    from lwm_b200 import ringattention as ra
    B, S, H = 1, 32768, 1
    p, seed = 0.1, 2024
    g = torch.Generator().manual_seed(0)
    q, k, v, do = [torch.randn(B, S, H, 128, generator=g) for _ in range(4)]
    qd, kd, vd = [t.to(DEV).requires_grad_(True) for t in (q, k, v)]
    out = ra.ringattention(qd, kd, vd, precision="fp16", **_kw(p, seed))
    out.backward(do.to(DEV))
    torch.cuda.synchronize()
    thr = threshold(p)
    qn, kn, vn, dn = [t[0, :, 0].double().numpy() for t in (q, k, v, do)]
    # dk / dv over every (query, key) pair, in blocks of query rows
    dk_ref, dv_ref = np.zeros_like(kn), np.zeros_like(vn)
    rows = np.arange(0, S, 997)
    o_ref, dq_ref = [], []
    n = 1024
    for r0 in range(0, S, n):
        qs, kp = np.arange(r0, r0 + n), np.arange(r0 + n)
        keep = (kp[None, :] <= qs[:, None]) & ~(drop_u16(seed, 0, 0, qs, kp) < thr)
        s = np.where(keep, qn[qs] @ kn[:r0 + n].T / np.sqrt(128), -np.inf)
        m = s.max(1, keepdims=True)
        live = np.isfinite(m[:, 0])
        pr = np.where(keep, np.exp(s - np.where(live[:, None], m, 0)), 0)
        pr /= np.maximum(pr.sum(1, keepdims=True), 1e-300)
        o = pr @ vn[:r0 + n]
        dp = dn[qs] @ vn[:r0 + n].T
        ds = pr * (dp - (dn[qs] * o).sum(1, keepdims=True)) / np.sqrt(128)
        dv_ref[:r0 + n] += pr.T @ dn[qs]
        dk_ref[:r0 + n] += ds.T @ qn[qs]
        sel = rows[(rows >= r0) & (rows < r0 + n)]
        o_ref.append(o[sel - r0])
        dq_ref.append((ds @ kn[:r0 + n])[sel - r0])
    o_ref, dq_ref = np.concatenate(o_ref), np.concatenate(dq_ref)
    got = [to_np(t)[0, :, 0] for t in (out, qd.grad, kd.grad, vd.grad)]
    assert rel_fro(got[0][rows], o_ref) < 1e-3
    assert rel_fro(got[1][rows], dq_ref) < 1e-3
    assert rel_fro(got[2], dk_ref) < 1e-3
    assert rel_fro(got[3], dv_ref) < 1e-3


# ------------------------------------------------------------------------------------------------ executors
RING_B = 2      # the peer executor launches one batch row at a time: each must still draw its own mask


def _ring_inputs(world, Sl, B=1, H=2):
    from oracle.attn_dense import finfo_min
    S = Sl * world
    g = torch.Generator().manual_seed(world * 10 + Sl)
    q, k, v, do = [torch.randn(B, S, H, 128, generator=g).to(torch.bfloat16).float() for _ in range(4)]
    bias = torch.zeros(B, S)
    bias[0, :45] = finfo_min("fp32")
    seg = torch.zeros(B, S, dtype=torch.int32)
    seg[:, S // 2 + 64:] = 1
    return q, k, v, do, bias, seg


def _check_ring(world, Sl, results, dropout, tol):
    q, k, v, do, bias, seg = _ring_inputs(world, Sl, B=RING_B)
    B, S, H, _ = q.shape
    drop = drop_mask(dropout[0], dropout[1], B, H, 0, S, 0, S)
    ref = attention_dropout_ref(q.numpy(), k.numpy(), v.numpy(), do.numpy(), drop, attn_bias=bias.numpy(),
                                segment_ids=seg.numpy(), causal=True)
    for r in range(world):
        sl = slice(r * Sl, (r + 1) * Sl)
        for j, (got, want) in enumerate(zip(results[r], ref[:4])):
            assert np.isfinite(got).all()
            e = rel_fro(got, want[:, sl])
            assert e < tol, (r, j, e)


@pytest.mark.parametrize("world,layout", [(2, "zigzag"), (4, "zigzag"), (2, "contiguous"), (4, "contiguous")])
def test_peer_executor_with_dropout(world, layout):
    import threading
    from lwm_b200 import ring_peer as rp, ring_schedule as rs
    from lwm_b200.ringattention import PeerOpsF16, with_dropout
    from peer_emulation import EmuTransport, EmuWorld
    Sl = 512
    dev = torch.device("cuda", 0)
    emu = EmuWorld(world, device=dev)
    q, k, v, do, bias, seg = _ring_inputs(world, Sl, B=RING_B)
    dropout = (31337 + world, threshold(0.2))
    results, fails = {}, []

    def worker(rank):
        try:
            torch.cuda.set_device(dev)
            tr = EmuTransport(emu, rank)
            plan = rs.make_peer_plan(world, rank, Sl, Sl, True, layout)
            sl = slice(rank * Sl, (rank + 1) * Sl)
            ql, kl, vl, dl = [t[:, sl].to(dev).contiguous() for t in (q, k, v, do)]
            ops = with_dropout(PeerOpsF16, dropout)
            out, res = rp.run_forward(plan, ql, kl, vl, bias.to(dev), seg.to(dev), True, ops, tr, True)
            dq, dk, dv = rp.run_backward(plan, res, kl, vl, dl, bias.to(dev), seg.to(dev), True, ops, tr, True)
            results[rank] = [t.double().cpu().numpy() for t in (out, dq, dk, dv)]
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
    assert not any(t.is_alive() for t in ts), "rank threads did not finish"
    assert not fails, fails[0]
    _check_ring(world, Sl, results, dropout, 1e-3)


@pytest.mark.parametrize("world,layout,precision", [(2, "zigzag", "fp16"), (4, "zigzag", "bf16"),
                                                    (2, "contiguous", "bf16"), (4, "contiguous", "fp16")])
def test_nccl_executor_with_dropout(monkeypatch, world, layout, precision):
    from lwm_b200 import ring_exec as rx, ringattention as ra
    from nccl_emulation import EmuComm, EmuGroup, EmuP2P, run_threads
    monkeypatch.setattr(rx, "_Comm", EmuComm)
    monkeypatch.setenv("LWM_RING_TRANSPORT", "nccl")
    Sl = 512
    emu = EmuP2P(world)
    q, k, v, do, bias, seg = _ring_inputs(world, Sl, B=RING_B)
    dropout = (-99 - world, threshold(0.2))

    def rank_fn(rank):
        torch.cuda.set_device(0)
        grp = EmuGroup(emu, rank)
        sl = slice(rank * Sl, (rank + 1) * Sl)
        ql, kl, vl, dl = [t[:, sl].to(DEV, torch.bfloat16).contiguous() for t in (q, k, v, do)]
        out, res = ra.ring_forward(ql, kl, vl, bias.to(DEV), seg.to(DEV), True, grp, rank, world, layout, precision,
                                   dropout=dropout)
        dq, dk, dv = ra.ring_backward(res, kl, vl, dl, bias.to(DEV), seg.to(DEV), True, grp, rank, world, layout,
                                      precision, dropout=dropout)
        return [t.double().cpu().numpy() for t in (out, dq, dk, dv)]

    results = run_threads(world, emu, rank_fn)
    _check_ring(world, Sl, results, dropout, _tol(precision, torch.bfloat16))
