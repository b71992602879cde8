"""The peer-memory ring executor (lwm_b200/ring_peer.py) with the REAL CUDA step functions, P ranks on one GPU.

The ranks are threads of one process; their heaps live on the device and flags on the host (tests/peer_emulation.py
explains why that ordering is sound without any device-side wait). What this adds to the CPU protocol tests
(tests/test_ring_peer_cpu.py) is the kernels' own bookkeeping across launches: every rank's shards of q, k, v and dO
carry a magnitude of their own, so every owner has its own power-of-two scales in the fp16 operand mode, and
  * forward carries are merged across launches whose K/V owners have different scale_k / scale_v,
  * dQ is summed over K/V owners with different scale_k (and scale_v, through dS),
  * dK / dV are summed over Q chunks with different scale_q / scale_do, the first visit writing (init) instead of adding,
with zigzag chunk offsets, per-batch launches (B = 2), and the heap regions of both pass parities reused by the passes
that follow. Results are compared on the global tensors with the float64 dense oracle (oracle/attn_dense.py).

Inputs and tolerances: tests/ring_emulated_inputs.py."""
import threading

import numpy as np
import pytest
import torch

from ring_emulated_inputs import NPAD, TOL_BF16_MODE, TOL_BF16_RESULT, TOL_F32_READOUT, _passes

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("world,layout,causal,Sl", [(2, "zigzag", True, 512), (4, "zigzag", True, 512),
                                                    (8, "zigzag", True, 256), (4, "contiguous", True, 512),
                                                    (3, "contiguous", False, 512)])
def test_peer_executor_with_cuda_kernels(world, layout, causal, Sl):
    from lwm_b200 import ring_peer as rp, ring_schedule as rs
    from lwm_b200.ringattention import PeerOpsBf16, PeerOpsF16
    from oracle.attn_dense import attention_dense, attention_dense_grads
    from peer_emulation import EmuTransport, EmuWorld
    dev = torch.device("cuda", 0)
    emu = EmuWorld(world, device=dev)
    passes = _passes(world, Sl)
    dev_masks = [(None if bias is None else bias.to(dev), None if seg is None else seg.to(dev))
                 for (_, _, _, (_, _, _, _, bias, seg)) in passes]
    results, fails = {}, []

    def worker(rank):
        try:
            torch.cuda.set_device(dev)
            # the emulation's ordering argument: every rank enqueues on the same (default) stream
            assert torch.cuda.current_stream(dev) == torch.cuda.default_stream(dev)
            tr = EmuTransport(emu, rank)
            plan = rs.make_peer_plan(world, rank, Sl, Sl, causal, layout)
            sl = slice(rank * Sl, (rank + 1) * Sl)
            mine = []
            for i, (prec, in_dtype, _, (q, k, v, do, _, _)) in enumerate(passes):
                ops = PeerOpsF16 if prec == "fp16" else PeerOpsBf16
                want_f32 = in_dtype == torch.float32
                ql, kl, vl, dl = [t[:, sl].to(dev, in_dtype).contiguous() for t in (q, k, v, do)]
                bias, seg = dev_masks[i]
                out, res = rp.run_forward(plan, ql, kl, vl, bias, seg, causal, ops, tr, want_f32)
                dq, dk, dv = rp.run_backward(plan, res, kl, vl, dl, bias, seg, causal, ops, tr, want_f32)
                assert out.dtype == in_dtype and dq.dtype == in_dtype and dk.dtype == in_dtype and dv.dtype == in_dtype
                mine.append([t.double().cpu().numpy() for t in (out, dq, dk, dv)])
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

    refs = {}
    worst = 0.0
    for i, (prec, in_dtype, m, (q, k, v, do, bias, seg)) in enumerate(passes):
        if m not in refs:
            kw = dict(causal=causal)
            if bias is not None:
                kw.update(attn_bias=bias.numpy(), segment_ids=seg.numpy())
            n = [t.double().numpy() for t in (q, k, v, do)]
            refs[m] = (attention_dense(*n[:3], **kw),) + tuple(attention_dense_grads(*n, **kw))
        if prec == "bf16":
            tol = TOL_BF16_MODE
        else:
            tol = TOL_F32_READOUT if in_dtype == torch.float32 else TOL_BF16_RESULT
        for r in range(world):
            sl = slice(r * Sl, (r + 1) * Sl)
            errs = []
            for j, (got, ref) in enumerate(zip(results[r][i], refs[m])):
                ref = ref[:, sl]
                if m and r == 0 and j in (0, 1):      # padded query rows (batch 0) are arbitrary in the oracle
                    got, ref = got.copy(), ref.copy()
                    got[0, :NPAD], ref[0, :NPAD] = 0, 0
                errs.append(float(np.linalg.norm(got - ref) / max(np.linalg.norm(ref), 1e-300)))
            print("world=%d %s pass %d precision=%s in=%s masks=%d rank %d errs(out,dq,dk,dv)=%s tol=%.0e" % (
                world, layout, i, prec, str(in_dtype).split(".")[-1], m, r, ["%.2e" % e for e in errs], tol))
            assert all(np.isfinite(errs)), (i, r, errs)
            worst = max(worst, max(errs) / tol)
    assert worst <= 1.0, "worst err/tol = %.3f" % worst
