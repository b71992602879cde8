"""The two-sided NCCL ring executor (lwm_b200/ring_exec.py) with the REAL CUDA step functions, P ranks as threads on
one GPU. The transport is tests/nccl_emulation.py (mailboxes in place of NCCL send/recv; its docstring gives the
ordering argument); everything else is production code: ring_forward / ring_backward's dispatch, the plans of
ring_schedule.py, CudaOps / CudaOpsF16 and the kernels.

What this covers that no other test does: the NCCL executor's own bookkeeping with real kernels. CudaOpsF16 gives every
q chunk and every K/V block its own power-of-two fp16 scale (the inputs of tests/ring_emulated_inputs.py give every
rank's shard its own magnitude) and caches the conversions for a pass; _f32_residuals maps the bf16 output chunks to
their fp32 copies for the backward's delta; CudaOps.accumulate adds the dK/dV partials of peers per batch entry into
row slices; run_backward stages its own dK/dV rows through copies for B > 1; sub-stepped plans and deeper K/V prefetch.

  (a) oracle parity through the production dispatch (LWM_RING_TRANSPORT=nccl), bf16 operands, both precision modes,
      with and without masks, passes back to back; in the fp16 mode also the fp32 values before the bf16 rounding
  (b) sub-stepped plans (n_sub_first = n_sub_last = 2, 4) and LWM_RING_PREFETCH = 1, 2, all through rx.run_*
  (c) protocol accounting from the message log, in every run of (a) and (b): the messages of every (src, dst, channel)
      and pass are exactly those the plans give (Q / dO / output permutations by plan.q_sends, K/V blocks by the
      receiver's remote blocks, one dK and one dV partial per remote block back to its owner), no message is left
      unmatched, and CudaOpsF16 converts every distinct operand block exactly once per pass
  (d) fp16 mode: power-of-two scaling of dO or V scales the results bit for bit; a repeated pass is bit-identical
  (e) the peer transport's fallback to this executor, with real kernels, for fp32 inputs
  (f) one NaN / +inf / -inf in rank 1's k or dO reaches only the results that read it (tests/test_nonfinite_gpu.py)

The reference is the float64 dense oracle (oracle/attn_dense.py) on the global tensors. Tolerances are those of
tests/ring_multi_gpu_worker.py (tests/ring_emulated_inputs.py). Not covered: the real NCCL side streams, the
high-priority group clone, and overlap between transfers and kernels; they need two or more GPUs
(tests/test_ring_multi_gpu.py)."""
import collections
import threading

import numpy as np
import pytest
import torch

from nccl_emulation import EmuComm, EmuGroup, EmuP2P, run_threads
from nonfinite_checks import (BAD_B, BAD_COL, BAD_H, BADS, SL_RING, TOL, _check, _check_other_slices, _dq_close,
                              _ring_inputs, _same_sets)
from ring_emulated_inputs import B, D, H, NPAD, TOL_BF16_MODE, TOL_BF16_RESULT, TOL_F32_READOUT, _inputs

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
_TLS = threading.local()     # per rank thread: the ops objects ring_forward / ring_backward made, fp16 conversions
_INPUTS, _REFS = {}, {}


# ------------------------------------------------------------------------------------------------ harness
def _rec_ops_f16():
    """CudaOpsF16 whose final casts keep their fp32 source: dq (per chunk), dk and dv before the bf16 rounding"""
    from lwm_b200.ringattention import CudaOpsF16

    class RecOpsF16(CudaOpsF16):
        def __init__(self):
            super().__init__()
            self.cast_src = []

        def cast(self, src, dst):
            self.cast_src.append(src.clone())
            super().cast(src, dst)
    return RecOpsF16


@pytest.fixture
def emulated(monkeypatch):
    """the NCCL executor's transport replaced by the thread emulation; ra._ops_for and ra.to_f16 record, per rank
    thread, the ops objects made and the fp16 conversions done"""
    from lwm_b200 import ring_exec as rx, ringattention as ra
    rec = _rec_ops_f16()
    to_f16 = ra.to_f16

    def ops_for(precision):
        ops = rec() if precision == "fp16" else ra.CudaOps
        _TLS.made.append(ops)
        return ops

    def counting_to_f16(x, stream=None):
        _TLS.conversions += 1
        return to_f16(x, stream)

    monkeypatch.setattr(rx, "_Comm", EmuComm)
    monkeypatch.setattr(ra, "_ops_for", ops_for)
    monkeypatch.setattr(ra, "to_f16", counting_to_f16)
    return rec


def _np(t):
    return t.detach().double().cpu().numpy()


def _global_inputs(world, Sl, seed, masks):
    key = (world, Sl, seed, masks)
    if key not in _INPUTS:
        _INPUTS[key] = _inputs(world, Sl, seed, masks)
    return _INPUTS[key]


def _reference(world, Sl, seed, masks, causal):
    """float64 (out, dq, dk, dv) of the global inputs"""
    from oracle.attn_dense import attention_dense, attention_dense_grads
    key = (world, Sl, seed, masks, causal)
    if key not in _REFS:
        q, k, v, do, bias, seg = _global_inputs(world, Sl, seed, masks)
        kw = dict(causal=causal)
        if bias is not None:
            kw.update(attn_bias=bias.numpy(), segment_ids=seg.numpy())
        n = [t.double().numpy() for t in (q, k, v, do)]
        _REFS[key] = (attention_dense(*n[:3], **kw),) + tuple(attention_dense_grads(*n, **kw))
    return _REFS[key]


def _pass(prec, seed, masks, scale=None, driver="dispatch", n_sub=1):
    """one forward + backward: scale = None or (which of "do" / "v", power of two) applied to the global inputs"""
    return dict(prec=prec, seed=seed, masks=masks, scale=scale, driver=driver, n_sub=n_sub)


def _pass_tensors(world, Sl, p):
    q, k, v, do, bias, seg = _global_inputs(world, Sl, p["seed"], p["masks"])
    if p["scale"] is not None:
        which, f = p["scale"]
        do, v = (do * f, v) if which == "do" else (do, v * f)
    return q, k, v, do, bias, seg


def _plans(world, Sl, causal, layout, p):
    """{rank: (forward plan, backward plan)} as the pass's driver makes them"""
    from lwm_b200 import ring_schedule as rs
    if p["driver"] == "dispatch":       # ring_forward / ring_backward
        n = rs.auto_sub(world, Sl, layout)
        return {r: (rs.make_plan(world, r, Sl, Sl, causal, layout, n_sub_first=n),
                    rs.make_plan(world, r, Sl, Sl, causal, layout, n_sub_first=n, n_sub_last=n)) for r in range(world)}
    n = p["n_sub"]
    return {r: (rs.make_plan(world, r, Sl, Sl, causal, layout, n_sub_first=n, n_sub_last=n),) * 2 for r in range(world)}


def _run(world, layout, causal, Sl, passes, rec):
    """every pass, back to back, in the same `world` rank threads -> [per pass {rank: results}]"""
    from lwm_b200 import ring_exec as rx, ringattention as ra
    emu = EmuP2P(world)
    tensors = [_pass_tensors(world, Sl, p) for p in passes]
    masks = [(None if t[4] is None else t[4].to(DEV), None if t[5] is None else t[5].to(DEV)) for t in tensors]
    plans = [_plans(world, Sl, causal, layout, p) for p in passes]

    def rank_fn(rank):
        torch.cuda.set_device(DEV)
        # the emulation's ordering argument: every rank enqueues on the same (default) stream
        assert torch.cuda.current_stream() == torch.cuda.default_stream()
        grp = EmuGroup(emu, rank)
        sl = slice(rank * Sl, (rank + 1) * Sl)
        mine = []
        for i, p in enumerate(passes):
            fp16 = p["prec"] == "fp16"
            ql, kl, vl, dl = [t[:, sl].to(DEV, torch.bfloat16).contiguous() for t in tensors[i][:4]]
            bias, seg = masks[i]
            fplan, bplan = plans[i][rank]
            _TLS.made, _TLS.conversions = [], 0
            grp.tag = (i, "fwd")
            if p["driver"] == "dispatch":
                out, res = ra.ring_forward(ql, kl, vl, bias, seg, causal, grp, rank, world, layout, p["prec"])
                fops = _TLS.made[-1]
            else:
                fops = rec() if fp16 else ra.CudaOps
                out, res = rx.run_forward(fplan, ql, kl, vl, bias, seg, causal, grp, fops)
                res = ra._f32_residuals(fops, res)
            n_fwd = _TLS.conversions
            grp.tag = (i, "bwd")
            _TLS.conversions = 0
            if p["driver"] == "dispatch":
                dq, dk, dv = ra.ring_backward(res, kl, vl, dl, bias, seg, causal, grp, rank, world, layout, p["prec"])
                bops = _TLS.made[-1]
            else:
                bops = rec() if fp16 else ra.CudaOps
                dq, dk, dv = rx.run_backward(bplan, res, kl, vl, dl, bias, seg, causal, grp, bops)
            n_bwd = _TLS.conversions
            assert all(t.dtype == torch.bfloat16 for t in (out, dq, dk, dv))
            r = dict(out=_np(out), dq=_np(dq), dk=_np(dk), dv=_np(dv))
            n_q = len(fplan.q_chunks)
            if fp16:
                # the backward's residuals are the un-rounded fp32 output chunks the forward kept
                assert [o.dtype for o in res["out_chunks"]] == [torch.float32] * n_q
                assert sorted(map(id, res["out_chunks"])) == sorted(map(id, fops.out_f32.values()))
                assert len(bops.cast_src) == n_q + 2
                pos = [qc.pos0 for qc in fplan.q_chunks]
                r.update(out32=list(zip(pos, map(_np, res["out_chunks"]))),
                         dq32=list(zip(pos, map(_np, bops.cast_src[:n_q]))),
                         dk32=_np(bops.cast_src[n_q]), dv32=_np(bops.cast_src[n_q + 1]))
                # every distinct operand block converted exactly once per pass: the q chunks and the K and V of every
                # visible block in the forward; the q and dO chunks and the K and V blocks in the backward
                n_kv_f = sum(len(st.kv) for st in fplan.steps)
                n_kv_b = sum(len(st.kv) for st in bplan.steps)
                r["conversions"] = (n_fwd, len(fops._cache), n_bwd, len(bops._cache))
                assert r["conversions"] == (n_q + 2 * n_kv_f,) * 2 + (2 * n_q + 2 * n_kv_b,) * 2, r["conversions"]
            else:
                assert n_fwd == n_bwd == 0
            emu.end_pass(rank)
            mine.append(r)
        return mine

    results = run_threads(world, emu, rank_fn)
    for i in range(len(passes)):
        _check_protocol(emu, i, plans[i], torch.bfloat16)
    assert len(emu.received) == len(emu.log) and not emu.pending()
    return [{r: results[r][i] for r in range(world)} for i in range(len(passes))]


def _check_protocol(emu, i, plans, op_dtype):
    """(c): the log of pass i against the plans. Channel 0: the q (forward) / dO (backward) rows by the sender's
    plan.q_sends, the K and V of every block the receiver's plan takes from the sender, step by step, then the output
    (forward) / dQ (backward) rows by the receiver's q_sends. Channel 1 (backward): the fp32 dK and dV partial of every
    block the sender took from the receiver, once each, step by step."""
    world = emu.world
    for phase in (0, 1):
        P = [plans[r][phase] for r in range(world)]
        got, want = collections.defaultdict(list), collections.defaultdict(list)
        for m in emu.log:
            if m.tag == (i, ("fwd", "bwd")[phase]):
                got[(m.src, m.dst, m.channel)].append((m.shape, m.dtype, m.nbytes))

        def msg(rows, dtype):
            return ((B, rows, H, D), dtype, B * rows * H * D * torch.empty((), dtype=dtype).element_size())
        for src in range(world):
            for dst in range(world):
                if src == dst:
                    continue
                gather = [l for (_, l, peer) in P[src].q_sends if peer == dst]
                assert gather == [qc.length for qc in P[dst].q_chunks if qc.owner == src]
                seq = [msg(l, op_dtype) for l in gather]
                seq += [msg(kv.length, op_dtype) for st in P[dst].steps for kv in st.kv if kv.owner == src
                        for _ in "kv"]
                seq += [msg(l, op_dtype) for (_, l, peer) in P[dst].q_sends if peer == src]
                if seq:
                    want[(src, dst, 0)] = seq
                if phase:
                    ret = [msg(kv.length, torch.float32) for st in P[src].steps for kv in st.kv if kv.owner == dst
                           for _ in "kv"]
                    if ret:
                        want[(src, dst, 1)] = ret
        assert dict(got) == dict(want), "pass %d %s: the messages differ from the plans" % (i, ("fwd", "bwd")[phase])


def _assemble(chunks, S):
    """[(pos0, [B,rows,H,D])] of every rank -> the global [B,S,H,D] array; every row exactly once"""
    g = np.zeros((B, S, H, D))
    cover = np.zeros(S, int)
    for pos0, a in chunks:
        g[:, pos0:pos0 + a.shape[1]] = a
        cover[pos0:pos0 + a.shape[1]] += 1
    assert (cover == 1).all()
    return g


def _rel(got, ref, masked_rows):
    if masked_rows:            # padded query rows (batch 0) are arbitrary in the oracle
        got, ref = got.copy(), ref.copy()
        got[0, :NPAD], ref[0, :NPAD] = 0, 0
    return float(np.linalg.norm(got - ref) / max(np.linalg.norm(ref), 1e-300))


def _oracle_errors(world, Sl, causal, passes, runs, label):
    """-> worst err/tol over every pass, rank and result: bf16 results at their mode's bound, and in the fp16 mode the
    fp32 values before the rounding at 1e-3"""
    worst = 0.0
    for p, run in zip(passes, runs):
        ref = _reference(world, Sl, p["seed"], p["masks"], causal)
        fp16 = p["prec"] == "fp16"
        f32 = None
        if fp16:
            S = world * Sl
            f32 = (_assemble([c for r in range(world) for c in run[r]["out32"]], S),
                   _assemble([c for r in range(world) for c in run[r]["dq32"]], S))
        for r in range(world):
            sl = slice(r * Sl, (r + 1) * Sl)
            checks = [(run[r][n], TOL_BF16_RESULT if fp16 else TOL_BF16_MODE, j) for j, n in
                      enumerate(("out", "dq", "dk", "dv"))]
            if fp16:
                checks += [(f32[0][:, sl], TOL_F32_READOUT, 0), (f32[1][:, sl], TOL_F32_READOUT, 1),
                           (run[r]["dk32"], TOL_F32_READOUT, 2), (run[r]["dv32"], TOL_F32_READOUT, 3)]
            errs = [(_rel(got, ref[j][:, sl], p["masks"] and r == 0 and j in (0, 1)), tol) for got, tol, j in checks]
            print("%s %s masks=%d rank %d errs(out,dq,dk,dv%s)=%s" % (
                label, p["prec"], p["masks"], r, ",out32,dq32,dk32,dv32" if fp16 else "",
                ["%.2e" % e for e, _ in errs]))
            assert all(np.isfinite(e) for e, _ in errs), (label, r, errs)
            worst = max(worst, max(e / t for e, t in errs))
    return worst


# ------------------------------------------------------------------------------------------------ (a) and (c)
@pytest.mark.parametrize("world,layout,causal,Sl", [(2, "zigzag", True, 512), (4, "zigzag", True, 512),
                                                    (8, "zigzag", True, 256), (4, "contiguous", True, 512),
                                                    (3, "contiguous", False, 512)])
def test_dispatch_matches_the_oracle(emulated, monkeypatch, world, layout, causal, Sl):
    """ring_forward -> ring_backward with LWM_RING_TRANSPORT=nccl and bf16 operands, every pass of both precision modes
    without and with masks (padding bias and segment ids: the block maps), back to back in the same threads"""
    monkeypatch.setenv("LWM_RING_TRANSPORT", "nccl")
    passes = [_pass(prec, (500 if m == 0 else 600) + world, m) for prec in ("fp16", "bf16") for m in (0, 1)]
    runs = _run(world, layout, causal, Sl, passes, emulated)
    worst = _oracle_errors(world, Sl, causal, passes, runs, "(a) world=%d %s" % (world, layout))
    print("(a) world=%d %s causal=%d worst err/tol=%.3f" % (world, layout, causal, worst))
    assert worst <= 1.0, "worst err/tol = %.3f" % worst


# ------------------------------------------------------------------------------------------------ (b) and (c)
@pytest.mark.parametrize("prefetch", ["1", "2", "all"])
@pytest.mark.parametrize("n_sub", [2, 4])
@pytest.mark.parametrize("layout", ["zigzag", "contiguous"])
def test_sub_steps_and_prefetch_depth(emulated, monkeypatch, layout, n_sub, prefetch):
    """rx.run_forward / run_backward over plans whose first and last steps are cut into n_sub pieces (pieces of 256 or
    128 rows: whole 128-row tiles), K/V exchanges posted 1, 2 or all steps ahead; CudaOpsF16 (with _f32_residuals, as
    ring_forward applies it) and CudaOps, with and without masks"""
    world, Sl = 4, 1024
    monkeypatch.setenv("LWM_RING_PREFETCH", prefetch)
    passes = [_pass(prec, 700 + m, m, driver="rx", n_sub=n_sub) for prec in ("fp16", "bf16") for m in (1, 0)]
    runs = _run(world, layout, True, Sl, passes, emulated)
    worst = _oracle_errors(world, Sl, True, passes, runs, "(b) %s n_sub=%d prefetch=%s" % (layout, n_sub, prefetch))
    print("(b) %s n_sub=%d prefetch=%s worst err/tol=%.3f" % (layout, n_sub, prefetch, worst))
    assert worst <= 1.0, "worst err/tol = %.3f" % worst


# ------------------------------------------------------------------------------------------------ (d)
def test_fp16_mode_power_of_two_exactness_and_repeatability(emulated, monkeypatch):
    """every fp16 scale is a power of two, so dO -> 2^k dO gives the same out and exactly 2^k dk, 2^k dv; V -> 2^k V
    exactly 2^k out, 2^k dk and the same dv; dq (fp32 atomics in no fixed order) within 1e-6. The same inputs run
    again after a different pass give the same out, dk and dv bit for bit. Checked on the bf16 results and on the fp32
    values before the rounding."""
    world, Sl, layout = 4, 512, "zigzag"
    monkeypatch.setenv("LWM_RING_TRANSPORT", "nccl")
    seed = 800
    passes = [_pass("fp16", seed, 1)]
    for k in (-20, 20):
        passes += [_pass("fp16", seed, 1, ("do", 2.0 ** k)), _pass("fp16", seed, 1, ("v", 2.0 ** k))]
    passes += [_pass("fp16", seed + 1, 0), _pass("fp16", seed, 1)]
    runs = _run(world, layout, True, Sl, passes, emulated)
    S = world * Sl

    def results(run):
        out32 = _assemble([c for r in range(world) for c in run[r]["out32"]], S)
        dq32 = _assemble([c for r in range(world) for c in run[r]["dq32"]], S)
        cat = lambda n: np.concatenate([run[r][n] for r in range(world)], axis=1)   # noqa: E731
        return dict(out=cat("out"), dq=cat("dq"), dk=cat("dk"), dv=cat("dv"), out32=out32, dq32=dq32,
                    dk32=cat("dk32"), dv32=cat("dv32"))

    base = results(runs[0])
    worst_dq = 0.0
    for p, run in zip(passes[1:], runs[1:]):
        got = results(run)
        which, f = p["scale"] if p["scale"] is not None else (None, 1.0)
        if p["seed"] != seed:
            continue
        want_f = dict(out=1.0 if which in ("do", None) else f, dk=f, dv=1.0 if which in ("v", None) else f, dq=f)
        for name in ("out", "dk", "dv", "out32", "dk32", "dv32"):
            want = base[name] * want_f[name.replace("32", "")]
            assert np.array_equal(got[name], want), (p["scale"], name, float(np.abs(got[name] - want).max()))
        e = float(np.linalg.norm(got["dq32"] - base["dq32"] * f) / np.linalg.norm(base["dq32"] * f))
        worst_dq = max(worst_dq, e)
        assert e < 1e-6, (p["scale"], e)
        assert _dq_close(base["dq"] * f, got["dq"], bf16=True), p["scale"]     # the bf16 dq: its rounding of that
    print("(d) dq rel err vs the scaled base run: worst %.2e" % worst_dq)


# ------------------------------------------------------------------------------------------------ (e)
def test_peer_fallback_runs_this_executor_with_fp32_inputs(emulated, monkeypatch):
    """LWM_RING_TRANSPORT=peer, and the peer heaps cannot be set up: the real _peer_transport marks every rank's group
    broken, fp32 inputs of the fp16 mode take the bf16 detour through this executor in the forward, and the backward
    follows the switched transport. The fp32 results equal the bf16 run of the same values after .float(): out, dk, dv
    bit for bit; dq is summed with fp32 atomics in no fixed order and then rounded to bf16, so a sum that lands on the
    other side of a rounding boundary moves an element by one bf16 unit (_dq_close)."""
    from lwm_b200 import ring_peer as rp, ringattention as ra
    world, Sl, layout = 4, 512, "zigzag"
    monkeypatch.setenv("LWM_RING_TRANSPORT", "peer")
    monkeypatch.setattr(ra, "_PEER_BROKEN", {})
    lock, asked = threading.Lock(), []

    def no_heaps(cls, group, device):
        with lock:
            asked.append(group.rank)
        raise rp.PeerTransportUnavailable("peer heaps cannot be mapped")

    monkeypatch.setattr(rp.CudaPeerTransport, "get", classmethod(no_heaps))
    q, k, v, do, bias, seg = _global_inputs(world, Sl, 900, True)
    bias_d, seg_d = bias.to(DEV), seg.to(DEV)
    emu = EmuP2P(world)
    groups = [EmuGroup(emu, r) for r in range(world)]

    def rank_fn(rank):
        torch.cuda.set_device(DEV)
        assert torch.cuda.current_stream() == torch.cuda.default_stream()
        grp = groups[rank]
        sl = slice(rank * Sl, (rank + 1) * Sl)
        got = {}
        for i, dt in enumerate((torch.float32, torch.bfloat16)):
            _TLS.made, _TLS.conversions = [], 0
            ql, kl, vl, dl = [t[:, sl].to(DEV, dt).contiguous() for t in (q, k, v, do)]
            grp.tag = (i, "fwd")
            out, res = ra.ring_forward(ql, kl, vl, bias_d, seg_d, True, grp, rank, world, layout, "fp16")
            assert id(grp) in ra._PEER_BROKEN and ra._transport(grp) == "nccl"
            n_asked = asked.count(rank)
            grp.tag = (i, "bwd")
            dq, dk, dv = ra.ring_backward(res, kl, vl, dl, bias_d, seg_d, True, grp, rank, world, layout, "fp16")
            assert all(t.dtype == dt for t in (out, dq, dk, dv))
            assert asked.count(rank) == n_asked == 1      # asked once, in the first forward; never in a backward
            got[dt] = [_np(t) for t in (out, dq, dk, dv)]
            emu.end_pass(rank)
        return got

    results = run_threads(world, emu, rank_fn)
    assert sorted(asked) == list(range(world))            # once per rank, in the first forward
    assert set(ra._PEER_BROKEN) == {id(g) for g in groups}
    # both passes ran on this executor: the dK/dV partial returns (channel 1) of the backward are in the log
    assert {m.tag for m in emu.log if m.channel == 1} == {(0, "bwd"), (1, "bwd")}
    ref = _reference(world, Sl, 900, True, True)
    worst = 0.0
    for r in range(world):
        f32, b16 = results[r][torch.float32], results[r][torch.bfloat16]
        for j, name in enumerate(("out", "dq", "dk", "dv")):
            if name == "dq":
                assert _dq_close(b16[j], f32[j], bf16=True)
            else:
                assert np.array_equal(f32[j], b16[j]), name
            e = _rel(f32[j], ref[j][:, r * Sl:(r + 1) * Sl], r == 0 and j in (0, 1))
            worst = max(worst, e / TOL_BF16_RESULT)
    print("(e) fallback worst err/tol=%.3f" % worst)
    assert worst <= 1.0


# ------------------------------------------------------------------------------------------------ (f)
_CLEAN = {}


def _nonfinite_run(world, tensors, precision):
    """ring_forward -> ring_backward on this executor (bf16 inputs), zigzag, causal -> global out, dq, dk, dv"""
    from lwm_b200 import ringattention as ra
    emu = EmuP2P(world)

    def rank_fn(rank):
        torch.cuda.set_device(DEV)
        _TLS.made, _TLS.conversions = [], 0
        grp = EmuGroup(emu, rank)
        sl = slice(rank * SL_RING, (rank + 1) * SL_RING)
        ql, kl, vl, dl = [t[:, sl].to(DEV).contiguous() for t in tensors]
        out, res = ra.ring_forward(ql, kl, vl, None, None, True, grp, rank, world, "zigzag", precision)
        dq, dk, dv = ra.ring_backward(res, kl, vl, dl, None, None, True, grp, rank, world, "zigzag", precision)
        emu.end_pass(rank)
        return [t.detach().float().cpu().numpy() for t in (out, dq, dk, dv)]

    results = run_threads(world, emu, rank_fn)
    return {name: np.concatenate([results[r][n] for r in range(world)], axis=1)
            for n, name in enumerate(("out", "dq", "dk", "dv"))}


@pytest.mark.parametrize("bad", list(BADS))
@pytest.mark.parametrize("which", ["k", "do"])
@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("world", [2, 4])
def test_nonfinite_inputs(emulated, monkeypatch, world, precision, which, bad):
    """tests/test_nonfinite_gpu.py::test_peer_ring on this executor: one bad element in rank 1's shard. Every q chunk
    and K/V block has its own fp16 scale here, from its largest finite |x|, so the bad element changes none of them.
    Inputs are bf16 only: fp32 inputs reach this executor as bf16."""
    from oracle.attn_dense import attention_visible
    monkeypatch.setenv("LWM_RING_TRANSPORT", "nccl")
    tensors, row = _ring_inputs(world, "bf16")
    key = (world, precision)
    if key not in _CLEAN:
        _CLEAN[key] = _nonfinite_run(world, tensors, precision)
    clean = _CLEAN[key]
    names = ("q", "k", "v", "do")
    dirty_t = list(tensors)
    t = dirty_t[names.index(which)].clone()
    t[BAD_B, row, BAD_H, BAD_COL] = BADS[bad]
    dirty_t[names.index(which)] = t
    dirty = _nonfinite_run(world, dirty_t, precision)
    S = world * SL_RING
    vis = np.tril(np.ones((S, S), bool))
    sl = [x.float().numpy()[BAD_B:BAD_B + 1, :, BAD_H:BAD_H + 1] for x in dirty_t]
    out, _, dq, dk, dv = attention_visible(*sl[:3], vis[None, None], sl[3])
    ref = dict(out=out[0, :, 0], dq=dq[0, :, 0], dk=dk[0, :, 0], dv=dv[0, :, 0])
    same = _same_sets(which, row, BAD_COL, vis, S, S)
    worst = 0.0
    for name in ("out", "dq", "dk", "dv"):
        if same[name] is None:
            continue
        _check_other_slices(name, clean[name], dirty[name], BAD_B, BAD_H, tol_dq=name == "dq", bf16=True)
        err = _check(name, clean[name][BAD_B, :, BAD_H], dirty[name][BAD_B, :, BAD_H], ref[name], same[name],
                     TOL[precision], same_tol=name == "dq", bf16=True, strict=name == "out" or which == "do")
        worst = max(worst, err / TOL[precision])
    print("(f) world=%d %s bad %s=%s worst err/tol=%.3f" % (world, precision, which, bad, worst))


# ------------------------------------------------------------------------------------------------ the conversion cache
def test_f16_cache_tells_views_at_one_address_apart(emulated):
    """CudaOpsF16 keys its conversions by address AND shape: with B = 1 a row slice of a shard is a view at the shard's
    own address, and must get its own fp16 copy and scale (the executor's B = 2 slices are copies, which never share
    an address within a pass)"""
    from lwm_b200 import ringattention as ra
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 512, 2, D, generator=g)
    x[:, 256:] *= 64.0
    x = x.to(DEV, torch.bfloat16)
    head = x[:, :256]
    assert head.data_ptr() == x.data_ptr() and head.is_contiguous()
    _TLS.conversions = 0
    ops = ra.CudaOpsF16()
    (x16, sx), (h16, sh) = ops._f16(x), ops._f16(head)
    assert ops._f16(x)[0] is x16 and ops._f16(head)[0] is h16 and _TLS.conversions == 2
    w16, ws = ra.to_f16(head.clone())
    assert h16.shape == head.shape and sh[0].item() == ws[0].item() != sx[0].item()
    assert torch.equal(h16.view(torch.int16), w16.view(torch.int16))
