"""torchrun worker: the sequence-parallel attention op on N GPUs against the float64 dense ORACLE (oracle/attn_dense.py)
evaluated on the same seeded inputs — forward and all three gradients, both work assignments, with and without
padding bias + packed segments, for float32 inputs (fp32 read-out of the result: the north_star 1e-3 bound applies
as is) and bfloat16 inputs (results additionally carry their bf16 rounding), plus the decode op.
Launched by tests/test_ring_multi_gpu.py, and by hand:
  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tests/ring_multi_gpu_worker.py
Environment: LWM_RING_TRANSPORT (peer|nccl), LWM_ATTN_PRECISION (fp16|bf16), RING_TEST_S (global sequence length)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TOL_F32_READOUT = 1e-3      # north_star bound, default (fp16 operand) precision mode
TOL_BF16_RESULT = 3e-3      # + bf16 rounding of out / gradients (8 significant bits)
TOL_BF16_MODE = 5e-3        # legacy bf16 operand mode: P / dS rounded to 8 bits


def main():
    import lwm_b200.ringattention as ra
    from lwm_b200.ringattention import ringattention, ringattention_inference
    from oracle.attn_dense import attention_dense, attention_dense_grads, attention_inference_dense, finfo_min
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dev = torch.device("cuda", torch.cuda.current_device())
    dist.init_process_group("nccl", device_id=dev)
    if os.environ.get("RING_TEST_MODE", "dense") == "sampled":
        return sampled(rank, world, dev)
    S = int(os.environ.get("RING_TEST_S", str(min(1024 * world, 4096))))
    B, H, D = 1, 4, 128
    npad = 50
    g = torch.Generator().manual_seed(99)
    q, k, v, do = [torch.randn(B, S, H, D, generator=g).to(torch.bfloat16).float() for _ in range(4)]
    bias = torch.zeros(B, 1, 1, S)
    bias[..., :npad] = finfo_min("bf16")
    seg = torch.zeros(B, S, dtype=torch.int32)
    seg[:, S // 2 + 7:] = 1
    kw = dict(axis_name="sp", float32_logits=True, cache_idx=None,
              blockwise_kwargs=dict(causal_block_size=1, deterministic=True, attn_pdrop=0.0, query_chunk_size=256,
                                    key_chunk_size=256))
    Sl = S // world
    sl = slice(rank * Sl, (rank + 1) * Sl)
    n = lambda t: t.detach().double().cpu().numpy()   # noqa: E731
    fp16_mode = ra._DEFAULT_PRECISION == "fp16"
    native_f32 = fp16_mode and ra._transport() == "peer"
    worst_ratio = 0.0
    for masks in (False, True):
        dol = do.clone()
        okw = dict(causal=True)
        if masks:
            dol[:, :npad] = 0
            okw.update(attn_bias=bias.reshape(B, S).numpy(), segment_ids=seg.numpy())
        ref = attention_dense(n(q), n(k), n(v), **okw)
        rq, rk, rv = attention_dense_grads(n(q), n(k), n(v), n(dol), **okw)
        b_, s_ = (bias.to(dev), seg.to(dev)) if masks else (None, None)
        for layout in ("zigzag", "contiguous"):
            for in_dtype in (torch.float32, torch.bfloat16):
                ql, kl, vl = [t[:, sl].to(dev, in_dtype).contiguous().requires_grad_(True) for t in (q, k, v)]
                ol = ringattention(ql, kl, vl, b_, s_, layout=layout, **kw)
                ol.backward(dol[:, sl].to(dev, in_dtype).contiguous())
                torch.cuda.synchronize()
                assert ol.dtype == in_dtype and ql.grad.dtype == in_dtype

                def rel(a, r):
                    a, r = n(a), r[:, sl]
                    if masks and rank == 0:          # padded query rows are arbitrary in the reference: excluded
                        a, r = a[:, npad:], r[:, npad:]
                    return float(np.linalg.norm(a - r) / max(np.linalg.norm(r), 1e-30))
                errs = (rel(ol, ref), rel(ql.grad, rq), rel(kl.grad, rk), rel(vl.grad, rv))
                if not fp16_mode:
                    tol = TOL_BF16_MODE
                elif in_dtype == torch.float32 and native_f32:
                    tol = TOL_F32_READOUT
                else:
                    tol = TOL_BF16_RESULT
                worst_ratio = max(worst_ratio, max(errs) / tol)
                print("rank %d layout=%s masks=%s in=%s errs(out,dq,dk,dv)=%s tol=%.0e" % (
                    rank, layout, masks, str(in_dtype).split(".")[-1], ["%.2e" % e for e in errs], tol), flush=True)
    # decode path: every rank holds a KV-cache shard, the single query row is replicated
    g2 = torch.Generator().manual_seed(7)
    qd = torch.randn(B, 1, H, D, generator=g2).to(torch.bfloat16)
    maskd = torch.ones(B, 1, 1, S, dtype=torch.bool)
    maskd[..., :29] = False
    maskd[..., S - 5:] = False
    kb, vb = k.to(torch.bfloat16), v.to(torch.bfloat16)
    od = ringattention_inference(qd.to(dev), kb[:, sl].contiguous().to(dev), vb[:, sl].contiguous().to(dev),
                                 maskd.to(dev), axis_name="sp")
    torch.cuda.synchronize()
    od_ref = attention_inference_dense(n(qd), n(k), n(v), maskd.numpy())
    e = float(np.linalg.norm(n(od) - od_ref) / np.linalg.norm(od_ref))
    print("rank %d decode (ringattention_inference) err vs oracle = %.2e" % (rank, e), flush=True)
    worst_ratio = max(worst_ratio, e / TOL_BF16_RESULT)
    t = torch.tensor([worst_ratio], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    dist.destroy_process_group()
    if t.item() > 1.0:
        print("RING_MULTI_GPU FAIL worst err/tol=%.3f" % t.item())
        sys.exit(1)
    if rank == 0:
        print("RING_MULTI_GPU OK transport=%s precision=%s worst err/tol=%.3f" % (ra._transport(), ra._DEFAULT_PRECISION,
                                                                                 t.item()))


def sampled(rank, world, dev):
    """Benchmark-size parity (32K tokens over 2 GPUs; 128K over 8): sampled query rows and every
    key row against the float64 row-wise oracle — lwm_b200/selftest.py::sampled_parity."""
    from lwm_b200.ringattention import ringattention
    from lwm_b200.selftest import sampled_parity
    S = int(os.environ.get("RING_TEST_S", "32768"))
    kw = dict(axis_name="sp", float32_logits=True, cache_idx=None,
              blockwise_kwargs=dict(causal_block_size=1, deterministic=True, attn_pdrop=0.0, query_chunk_size=1024,
                                    key_chunk_size=1024))
    errs = sampled_parity(S, 4, [1, 3], lambda q, k, v: ringattention(q, k, v, None, None, **kw), dev, rank, world)
    print("rank %d sampled parity S=%d: %s" % (rank, S, {k2: ("%.2e" % v2 if isinstance(v2, float) else v2)
                                                         for k2, v2 in errs.items()}), flush=True)
    worst = max(errs[n_] for n_ in ("out", "dq", "dk", "dv"))
    bad = 1.0 if errs["dq_unsampled_abs"] != 0.0 else 0.0
    t = torch.tensor([worst, bad], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    dist.destroy_process_group()
    if t[0].item() > TOL_F32_READOUT or t[1].item() != 0.0:
        print("RING_MULTI_GPU FAIL sampled worst=%.3e" % t[0].item())
        sys.exit(1)
    if rank == 0:
        print("RING_MULTI_GPU OK sampled S=%d world=%d worst rel err=%.3e (tol %.0e)" % (S, world, t[0].item(),
                                                                                      TOL_F32_READOUT))


if __name__ == "__main__":
    main()
