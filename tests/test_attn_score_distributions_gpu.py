"""Attention on sink-dominated long-context score distributions (tests/score_distributions.py) against float64, on
the GPU: the public op on one GPU, `ringattention_inference` (tensor-core and GEMV paths) and the peer-memory ring
executor on emulated ranks.

A sink key `gap` nats above a bulk of N(0, sigma^2) logits puts every bulk p at about e^-gap against the row max. The
fp16 mode's forward packs P as p * 2^15 (DESIGN.md §5); packed as p itself, the bulk's mass went fp16-subnormal or zero
from a gap of about 10 nats while l kept it, and the output drifted from the oracle (and the backward with it, through
delta = rowsum(dO o O)). Every asserted bound is one the CPU model of the kernels (tests/test_attn_sink_model_cpu.py)
meets with a factor of 2 to spare, and one the GPU meets with that margin too:
  fp16 mode  out and dv < 1e-3 at every gap; dq and dk < 1e-3 up to a gap of 14. From a gap of 16 on the global dq / dk
             are printed, not asserted (DESIGN.md §5): dS of the sink key is P (dP - delta) with dP - delta about the
             bulk's mass times dP, so the 1e-4 relative error of the forward's fp32 accumulation, which delta
             inherits, is amplified by 1 / (bulk mass); and the dS of the bulk keys goes fp16-subnormal ('dk_bulk').
             The model, given the GPU output's 1e-4 error in delta, gives 6e-4 .. 4e-3 there; the GPU 1e-3 .. 5e-3.
  bf16 mode  out and dv < 5e-3 (the suite's legacy-mode bound); its dq / dk are printed, not asserted: the delta of
             the legacy mode comes from the bf16-rounded output, which the same 1 / (bulk mass) amplifies.
The recency control's fp16 dq is printed only: k's rising channel 0 makes dq = sum dS k a difference of large terms
(1.0e-3 measured, with or without the boost).
Every case prints every error, and the dk / dv errors over the keys other than key 0 ('dk_bulk', 'dv_bulk')."""
import threading

import numpy as np
import pytest
import torch

import score_distributions as sd

pytestmark = pytest.mark.gpu

TOL = {"fp16": 1e-3, "bf16": 5e-3}
GRADS_ASSERTED = {"fp16": ("out", "dq", "dk", "dv"), "bf16": ("out", "dv")}
SINK_ASSERTED = {"fp16": ("out", "dv"), "bf16": ("out", "dv")}   # gaps of 16 and more
MAX_GAP_DQ_DK = 14.0
KW = dict(axis_name="sp", float32_logits=True, cache_idx=None,
          blockwise_kwargs=dict(causal_block_size=1, deterministic=True, attn_pdrop=0.0, query_chunk_size=1024,
                                key_chunk_size=1024))


def _rel(a, r):
    a, r = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(r, dtype=torch.float64)
    return float((a - r).norm() / r.norm().clamp_min(1e-300))


def _inputs(kind, S, H, **kw):
    """global q, k, v, dO [1, S, H, 128] (float32, bf16 values), the sampled rows, and dO zero outside them"""
    from oracle.attn_rows import sample_rows
    q, k, v, do = [sd.shard(kind, n, 0, S, S, H, **kw) for n in ("q", "k", "v", "do")]
    rows = sample_rows(S)
    keep = torch.zeros(S, dtype=torch.bool)
    keep[rows] = True
    do[0, ~keep] = 0
    return q, k, v, do, rows


def _refs(q, k, v, do, rows):
    from oracle.attn_rows import attention_rows
    return [attention_rows(q[0, rows, h], rows, k[0, :, h], v[0, :, h], do[0, rows, h]) for h in range(q.shape[2])]


def _errors(got, refs, rows):
    """got: dict(out, dq, dk, dv) of global [S, H, 128] float64 tensors. Max over heads."""
    e = {}
    for h, ref in enumerate(refs):
        pairs = dict(out=(got["out"][rows, h], ref["out"]), dq=(got["dq"][rows, h], ref["dq"]),
                     dk=(got["dk"][:, h], ref["dk"]), dv=(got["dv"][:, h], ref["dv"]),
                     dk_bulk=(got["dk"][1:, h], ref["dk"][1:]), dv_bulk=(got["dv"][1:, h], ref["dv"][1:]))
        for n, (a, r) in pairs.items():
            e[n] = max(e.get(n, 0.0), _rel(a, r))
        dq_other = got["dq"][:, h].clone()
        dq_other[rows] = 0
        e["dq_unsampled_abs"] = max(e.get("dq_unsampled_abs", 0.0), float(dq_other.abs().max()))
    return e


def _check(label, errs, asserted):
    for prec, e in errs.items():
        print("%s %s %s" % (label, prec, {n: ("%.2e" % x) for n, x in e.items()}))
    for prec, e in errs.items():
        for n in asserted[prec]:
            assert e[n] < TOL[prec], (label, prec, n, e)


def _public_op(kind, S, H, **kw):
    """the public op on one GPU in both precision modes, forward and backward, on the sampled rows (out, dq) and
    every key (dk, dv) — the pattern of lwm_b200/selftest.sampled_parity on these inputs"""
    from lwm_b200 import ringattention as ra
    q, k, v, do, rows = _inputs(kind, S, H, **kw)
    refs = _refs(q, k, v, do, rows)
    errs = {}
    for prec in ("fp16", "bf16"):
        qd, kd, vd = [t.cuda().requires_grad_(True) for t in (q, k, v)]
        out = ra.ringattention(qd, kd, vd, None, None, precision=prec, **KW)
        out.backward(do.cuda())
        torch.cuda.synchronize()
        assert out.dtype == torch.float32
        got = dict(out=out.detach()[0].double().cpu(), dq=qd.grad[0].double().cpu(), dk=kd.grad[0].double().cpu(),
                   dv=vd.grad[0].double().cpu())
        errs[prec] = _errors(got, refs, rows)
        assert errs[prec]["dq_unsampled_abs"] == 0.0, (prec, errs[prec])
    return errs


@pytest.mark.parametrize("sigma", [0.5, 1.0])
@pytest.mark.parametrize("gap", [0.0, 14.0, 16.0, 17.0, 18.0])
def test_public_op_sink_32k(gap, sigma):
    errs = _public_op("sink", 32768, 2, gap=gap, sigma=sigma)
    _check("S=32768 H=2 sink gap=%g sigma=%g" % (gap, sigma), errs,
           GRADS_ASSERTED if gap <= MAX_GAP_DQ_DK else SINK_ASSERTED)


@pytest.mark.parametrize("kind", ["recency", "peaked"])
def test_public_op_controls_32k(kind):
    errs = _public_op(kind, 32768, 2)
    # recency: the rising channel 0 of k makes dq = sum dS k a difference of large terms (model 9.5e-4)
    asserted = dict(GRADS_ASSERTED, fp16=("out", "dk", "dv") if kind == "recency" else GRADS_ASSERTED["fp16"])
    _check("S=32768 H=2 %s" % kind, errs, asserted)


@pytest.mark.parametrize("gap", [17.0, 18.0])
def test_public_op_sink_128k(gap):
    errs = _public_op("sink", 131072, 1, gap=gap, sigma=0.5)
    _check("S=131072 H=1 sink gap=%g sigma=0.5" % gap, errs, SINK_ASSERTED)


@pytest.mark.parametrize("sigma", [0.5, 1.0])
@pytest.mark.parametrize("gap", [20.0, 22.0])
def test_public_op_sink_forward_at_large_gaps(gap, sigma):
    """the backward runs and is printed (dk_bulk reaches 0.2 .. 0.8, DESIGN.md §5); only the forward is asserted"""
    errs = _public_op("sink", 32768, 2, gap=gap, sigma=sigma)
    _check("S=32768 H=2 sink gap=%g sigma=%g (forward asserted)" % (gap, sigma), errs, dict(fp16=("out",), bf16=("out",)))


# ------------------------------------------------------------------------------------------ ringattention_inference
INFER_K = 131072


def _infer_inputs(Q, dtype, H=1):
    """the last Q rows of a 131072-token sink sequence as queries, the whole sequence as the KV cache: one head,
    repeated H times on the device (every head has the same float64 result)"""
    kw = dict(gap=18.0, sigma=0.5)
    q = sd.shard("sink", "q", INFER_K - 128 * ((Q + 127) // 128), 128 * ((Q + 127) // 128), INFER_K, 1, **kw)[:, -Q:]
    k = sd.shard("sink", "k", 0, INFER_K, INFER_K, 1, **kw)
    v = sd.shard("sink", "v", 0, INFER_K, INFER_K, 1, **kw)
    host = [t.contiguous().to(dtype) for t in (q, k, v)]
    dev = [t.cuda().expand(-1, -1, H, -1).contiguous() for t in host]
    return host, dev


def _infer_mask(kind, Q):
    if kind == "none":
        return None
    from lwm_b200.ringattention import decode_attention_mask
    return decode_attention_mask(torch.ones(1, INFER_K, dtype=torch.int32), Q, INFER_K - Q, INFER_K)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mask", ["none", "decode"])
@pytest.mark.parametrize("Q", [128, 256])
def test_inference_tensor_core_path_sink(Q, mask, dtype):
    """H * ceil(Q / 128) = 132 CTAs: the tensor-core path then runs each Q tile over the whole cache in one CTA, with
    no key split (ringattention.infer_partial splits the keys only to fill the SMs). So every row packs all 131072
    keys' P against the sink's max, as a long-context call with many heads does; with B = H = 1 the keys would be
    split 66 or 132 ways, and only the split holding key 0 would see the sink."""
    from lwm_b200.ringattention import ringattention_inference
    from oracle.attn_dense import attention_inference_dense
    H = 132 // ((Q + 127) // 128)
    (q, k, v), (qd, kd, vd) = _infer_inputs(Q, dtype, H)
    m = _infer_mask(mask, Q)
    out = ringattention_inference(qd, kd, vd, None if m is None else m.cuda())
    torch.cuda.synchronize()
    assert out.dtype == dtype and out.shape == (1, Q, H, 128)
    del kd, vd
    ref = torch.from_numpy(attention_inference_dense(q.double().numpy(), k.double().numpy(), v.double().numpy(),
                                                     None if m is None else m.numpy()))
    err = _rel(out.double().cpu(), ref.expand(-1, -1, H, -1))
    tol = 1e-3 if dtype == torch.float32 else 3e-3
    print("inference tensor cores Q=%d H=%d K=%d mask=%s %s err=%.2e tol=%.0e" % (Q, H, INFER_K, mask, dtype, err, tol))
    assert err < tol


@pytest.mark.parametrize("Q", [1, 4])
def test_inference_gemv_path_sink(Q):
    """the GEMV decode kernel works in fp32 throughout: a control, unaffected by the fp16 forward's P"""
    from lwm_b200.ringattention import ringattention_inference
    from oracle.attn_dense import attention_inference_dense
    (q, k, v), (qd, kd, vd) = _infer_inputs(Q, torch.float32)
    out = ringattention_inference(qd, kd, vd, None)
    torch.cuda.synchronize()
    ref = attention_inference_dense(q.double().numpy(), k.double().numpy(), v.double().numpy(), None)
    err = _rel(out.double().cpu(), ref)
    print("inference GEMV Q=%d K=%d err=%.2e" % (Q, INFER_K, err))
    assert err < 1e-4


# ------------------------------------------------------------------------------------------ peer-memory ring
@pytest.mark.parametrize("world,layout", [(2, "zigzag"), (4, "contiguous")])
def test_peer_ring_sink_on_rank0(world, layout):
    """the peer-memory executor with the real kernels, ranks as threads on one GPU (tests/peer_emulation.py), the
    sink on rank 0: every other rank's rows merge a carry whose max sits on another rank's key"""
    from lwm_b200 import ring_peer as rp, ring_schedule as rs
    from lwm_b200.ringattention import PeerOpsBf16, PeerOpsF16
    from peer_emulation import EmuTransport, EmuWorld
    Sl, gap, sigma = 16384, 18.0, 0.5
    S = world * Sl
    q, k, v, do, rows = _inputs("sink", S, 1, gap=gap, sigma=sigma)
    refs = _refs(q, k, v, do, rows)
    dev = torch.device("cuda", 0)
    emu = EmuWorld(world, device=dev)
    results, fails = {}, []

    def worker(rank):
        try:
            torch.cuda.set_device(dev)
            assert torch.cuda.current_stream(dev) == torch.cuda.default_stream(dev)
            tr = EmuTransport(emu, rank)
            plan = rs.make_peer_plan(world, rank, Sl, Sl, True, layout)
            sl = slice(rank * Sl, (rank + 1) * Sl)
            mine = {}
            for prec, ops in (("fp16", PeerOpsF16), ("bf16", PeerOpsBf16)):
                ql, kl, vl, dl = [t[:, sl].to(dev).contiguous() for t in (q, k, v, do)]
                out, res = rp.run_forward(plan, ql, kl, vl, None, None, True, ops, tr, True)
                dq, dk, dv = rp.run_backward(plan, res, kl, vl, dl, None, None, True, ops, tr, True)
                mine[prec] = [t[0].double().cpu() for t in (out, dq, dk, dv)]
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
    errs = {}
    for prec in ("fp16", "bf16"):
        got = {n: torch.cat([results[r][prec][i] for r in range(world)]) for i, n in enumerate(("out", "dq", "dk", "dv"))}
        errs[prec] = _errors(got, refs, rows)
    _check("peer world=%d %s Sl=%d sink gap=%g sigma=%g" % (world, layout, Sl, gap, sigma), errs, SINK_ASSERTED)
