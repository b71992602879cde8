"""World-size-2/4 CPU tests (gloo) of the q-sharded `ringattention_inference` backward: the real
lwm_b200.ringattention._infer_sharded (recording its residuals) and _infer_sharded_bwd with their collectives on
torch.distributed, and float64 numpy stand-ins for the kernels that follow their contracts (staging with a scale,
merge with lse, delta, the backward launch with P = 0 for masked entries and -inf rows, the rank-ordered dQ sum).
Every rank's dq, dk and dv are compared with the float64 VJP of the whole problem, on both sides of INFER_MIN_Q."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_attn_infer_ring_gloo import NumpyInferOps, _case, _free_port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))


class NumpyInferGradOps(NumpyInferOps):
    @staticmethod
    def partial(q, k, v, mask, row_any, tensor_cores, staged=None):
        if staged is not None:      # the kernel reads the staged copies and applies their scales
            q, k, v = (x * s for x, s in staged)
        return NumpyInferOps.partial(q, k, v, mask, row_any, tensor_cores)

    @staticmethod
    def stage(x):
        return x.double() / 4.0, torch.tensor([4.0], dtype=torch.float64)

    @staticmethod
    def stage_by(x, scale):
        return x.double() / scale

    @staticmethod
    def merge_lse(o, ml, n_part, out_shape):
        out = NumpyInferOps.merge(o, ml, n_part, out_shape, torch.float64)
        m, l = ml[..., 0].numpy(), ml[..., 1].numpy()
        mm = m.max(-1, keepdims=True)
        lse2 = mm[:, 0] + np.log2((np.exp2(m - mm) * l).sum(-1))
        return out, torch.from_numpy(lse2 * np.log(2.0))

    @staticmethod
    def delta(o32, do16, sdo):
        return torch.einsum("bqhd,bqhd->bhq", o32, do16 * sdo)

    @staticmethod
    def backward(q16, k16, v16, do16, scales, lse, delta, bits, row_any):
        sq, sk, sv, sdo = (float(s) for s in scales)
        q, k, v, g = (x.numpy() * s for x, s in ((q16, sq), (k16, sk), (v16, sv), (do16, sdo)))
        B, Q, H, D = q.shape
        Sk = k.shape[1]
        vis = np.ones((B, Q, Sk), dtype=bool) if bits is None else np.unpackbits(
            bits.numpy().view(np.uint8), axis=-1, bitorder="little")[..., :Sk].astype(bool)
        s = np.einsum("bqhd,bkhd->bhqk", q, k) / np.sqrt(D)
        lse = lse.numpy()[..., None]
        p = np.where(vis[:, None] & np.isfinite(lse), np.exp(s - np.where(np.isfinite(lse), lse, 0.0)), 0.0)
        dp = np.einsum("bqhd,bkhd->bhqk", g, v)
        ds = p * (dp - delta.numpy()[..., None])
        dq = np.einsum("bhqk,bkhd->bqhd", ds, k) / np.sqrt(D)
        dk = np.einsum("bhqk,bqhd->bkhd", ds, q) / np.sqrt(D)
        dv = np.einsum("bhqk,bqhd->bkhd", p, g)
        return tuple(torch.from_numpy(np.ascontiguousarray(x)) for x in (dq, dk, dv))

    @staticmethod
    def reduce_cast(srcs, dst):
        acc = srcs[0].clone()
        for s in srcs[1:]:
            acc += s
        dst.copy_(acc)

    @staticmethod
    def cast(x32, dtype):
        return x32.to(dtype)


def _worker(rank, world, port, Ql, B, broadcast, use_mask, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from lwm_b200 import ringattention as ra
        from infer_grad_model import attention_inference_vjp
        q, k, v, mask, Sl = _case(world, Ql, B, broadcast, 7)
        q, k, v = q.double(), k.double(), v.double()
        g = torch.randn(q.shape, generator=torch.Generator().manual_seed(9), dtype=torch.float64)
        rows, keys = slice(rank * Ql, (rank + 1) * Ql), slice(rank * Sl, (rank + 1) * Sl)
        m_loc = mask[:, :, rows].contiguous() if use_mask else None
        comm, saved = ra.TorchComm(None, world), {}
        ra._infer_sharded(q[:, rows].contiguous(), k[:, keys].contiguous(), v[:, keys].contiguous(), m_loc, comm,
                          NumpyInferGradOps, saved=saved)
        dq, dk, dv = ra._infer_sharded_bwd(saved, g[:, rows].contiguous(), comm, NumpyInferGradOps)
        full = np.broadcast_to(mask.numpy(), (B,) + mask.shape[1:]) if use_mask else None
        rq, rk, rv = attention_inference_vjp(q.numpy(), k.numpy(), v.numpy(), full, g.numpy())
        from helpers import rel_fro     # all-zero references (every row masked) must come out exactly zero
        ret[rank] = max(rel_fro(x.numpy(), r) for x, r in ((dq, rq[:, rows]), (dk, rk[:, keys]), (dv, rv[:, keys])))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("Ql,B,broadcast,use_mask", [
    (1, 1, False, True),       # world * Q_loc below INFER_MIN_Q: uint8 slabs, row statistics recomputed
    (2, 2, False, True),
    (37, 2, False, True),      # Q_loc not a multiple of 64
    (37, 2, True, True),       # batch-broadcast mask
    (130, 1, False, True),
    (5, 2, False, False),      # attn_mask=None
])
def test_q_sharded_backward_matches_float64_vjp(world, Ql, B, broadcast, use_mask):
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, _free_port(), Ql, B, broadcast, use_mask, ret), nprocs=world, join=True)
    assert len(ret) == world
    for r in range(world):
        assert ret[r] < 1e-10, (r, ret[r])
