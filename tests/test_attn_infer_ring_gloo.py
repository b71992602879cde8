"""World-size-2/4 CPU tests (gloo) of the q-sharded `ringattention_inference` protocol: the real
lwm_b200.ringattention._infer_sharded with its collectives on torch.distributed (all_gather_into_tensor,
all_to_all_single), and numpy stand-ins for the mask-packing, partial and merge kernels that follow the kernels'
contracts (mask bits, fully masked rows, log2-domain partials). Compared against the dense float64 oracle on the
whole query and cache, with Q_loc not a multiple of 128, fully masked rows, a left-padded decode mask and a
batch-broadcast mask, on both sides of INFER_MIN_Q. The replicated protocol of the generation call
(lwm_b200.ringattention._infer_replicated, Q = 1) runs the same way under the generation masks of
tests/test_attn_decode_ring_gpu.py: whole ranks unfilled or padded, a fully masked batch row, a broadcast mask."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASKED_LOG2 = -1.0e30     # the kernels' kMaskedLogit


class NumpyInferOps:
    @staticmethod
    def mask_pack(mask, B, n_slabs, ncols):
        m = np.broadcast_to(mask.numpy()[:, 0] != 0, (B, mask.shape[2], mask.shape[3]))[..., :n_slabs * ncols]
        kw = (ncols + 127) // 128 * 4
        m = m.reshape(B, m.shape[1], n_slabs, ncols).transpose(2, 0, 1, 3)
        pad = np.zeros(m.shape[:3] + (kw * 32,), dtype=bool)
        pad[..., :ncols] = m
        bits = np.packbits(pad, axis=-1, bitorder="little").view("<u4").view(np.int32)
        return torch.from_numpy(bits.copy()), torch.from_numpy(m.any(axis=(0, 3)).astype(np.int32))

    @staticmethod
    def partial(q, k, v, mask, row_any, tensor_cores):
        B, Q, H, D = q.shape
        Sk = k.shape[1]
        if mask is None:
            vis = np.ones((B, Q, Sk), dtype=bool)
        elif tensor_cores:
            vis = np.unpackbits(mask.numpy().view(np.uint8), axis=-1, bitorder="little")[..., :Sk].astype(bool)
        else:
            vis = mask.numpy() != 0
        s = np.einsum("bqhd,bkhd->bqhk", q.double().numpy(), k.double().numpy()) / np.sqrt(D) * np.log2(np.e)
        vis = np.broadcast_to(vis[:, :, None, :], s.shape)
        if tensor_cores and row_any is not None:
            # a row fully masked over the whole ring visits every tile with the masked logit
            dead = (row_any.numpy() == 0)[:, :, None, None]
            s = np.where(vis, s, np.where(dead, MASKED_LOG2, -np.inf))
        else:
            s = np.where(vis, s, MASKED_LOG2)
        m = s.max(-1)
        p = np.where(np.isfinite(m)[..., None], np.exp2(s - np.where(np.isfinite(m), m, 0)[..., None]), 0.0)
        o = np.einsum("bqhk,bkhd->bqhd", p, v.double().numpy())
        ml = np.stack([m, p.sum(-1)], -1)
        return torch.from_numpy(o.reshape(-1, D)), torch.from_numpy(ml.reshape(-1, 2))

    @staticmethod
    def merge(o, ml, n_part, out_shape, dtype):
        o, ml = o.numpy(), ml.numpy()
        mm = ml[..., 0].max(-1, keepdims=True)
        c = np.where(np.isfinite(ml[..., 0]), np.exp2(ml[..., 0] - np.where(np.isfinite(mm), mm, 0)), 0.0)
        num = (c[..., None] * o).sum(1)
        den = (c * ml[..., 1]).sum(1)
        return torch.from_numpy((num / den[:, None]).reshape(out_shape))


def _case(world, Ql, B, broadcast, seed):
    """q [B,Q,H,D], k/v [B,K,H,D], mask [Bm,1,Q,K]: left padding, decode-style causal rows, fully masked rows"""
    H, D, Sl = 2, 16, 200
    Q, K = world * Ql, world * Sl
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, n, H, D, generator=g) for n in (Q, K, K))
    cache_index = K - Q - 30
    mask = (torch.arange(K)[None, :] <= (torch.arange(Q) + cache_index)[:, None])[None, None].repeat(B, 1, 1, 1)
    mask[0, :, :, :23] = False                     # left-padded prompt
    mask[..., min(3, Q - 2), :] = False             # fully masked rows
    mask[..., Q - 1, :] = False
    if B > 1:
        mask[1, :, :, 40:300] = False
    if broadcast:
        mask = mask[:1]
    return q, k, v, mask, Sl


def _worker(rank, world, port, Ql, B, broadcast, use_mask, ret):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from lwm_b200 import ringattention as ra
        from oracle.attn_dense import attention_inference_dense
        q, k, v, mask, Sl = _case(world, Ql, B, broadcast, 7)
        rows, keys = slice(rank * Ql, (rank + 1) * Ql), slice(rank * Sl, (rank + 1) * Sl)
        m_loc = mask[:, :, rows].contiguous() if use_mask else None
        out = ra._infer_sharded(q[:, rows].contiguous(), k[:, keys].contiguous(), v[:, keys].contiguous(), m_loc,
                                ra.TorchComm(None, world), NumpyInferOps)
        full = np.broadcast_to(mask.numpy(), (B,) + mask.shape[1:]) if use_mask else None
        ref = attention_inference_dense(q.numpy(), k.numpy(), v.numpy(), full)[:, rows]
        err = float(np.linalg.norm(out.numpy() - ref) / np.linalg.norm(ref))
        ret[rank] = err
    finally:
        dist.destroy_process_group()


def _replicated_worker(rank, world, port, ret):
    """the replicated (Q = 1, generation) protocol under every generation mask of the GPU test"""
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from lwm_b200 import ringattention as ra
        from oracle.attn_dense import attention_inference_dense
        from test_attn_decode_ring_gpu import MASK_KINDS, generation_mask
        B, H, D, Sl = 2, 2, 16, 50
        K = world * Sl
        g = torch.Generator().manual_seed(11)
        q = torch.randn(B, 1, H, D, generator=g)
        # every rank's shard has its own magnitudes: keys 2^-r, values 2^(6r), 2^(-6r) alternately
        r_of = torch.arange(K) // Sl
        k = torch.randn(B, K, H, D, generator=g) * (2.0 ** -r_of)[None, :, None, None]
        v = torch.randn(B, K, H, D, generator=g) * (2.0 ** (6 * r_of * (-1) ** r_of))[None, :, None, None]
        keys = slice(rank * Sl, (rank + 1) * Sl)
        for kind in MASK_KINDS:
            mask = generation_mask(kind, B, Sl, world)
            out = ra._infer_replicated(q, k[:, keys].contiguous(), v[:, keys].contiguous(), mask, rank,
                                       ra.TorchComm(None, world), NumpyInferOps).numpy()
            full = None if mask is None else np.broadcast_to(mask.numpy(), (B,) + mask.shape[1:])
            ref = attention_inference_dense(q.numpy(), k.numpy(), v.numpy(), full)
            ret[(rank, kind)] = float((np.linalg.norm(out - ref, axis=-1) / np.linalg.norm(ref, axis=-1)).max())
    finally:
        dist.destroy_process_group()


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("Ql,B,broadcast,use_mask", [
    (1, 1, False, True),       # world * Q_loc below INFER_MIN_Q: the GEMV kernel and uint8 mask slabs
    (37, 2, False, True),      # Q_loc not a multiple of 128
    (37, 2, True, True),       # batch-broadcast mask
    (130, 1, False, True),
    (5, 2, False, False),      # attn_mask=None
])
def test_q_sharded_protocol_matches_dense_oracle(world, Ql, B, broadcast, use_mask):
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, _free_port(), Ql, B, broadcast, use_mask, ret), nprocs=world, join=True)
    assert len(ret) == world
    for r in range(world):
        assert ret[r] < 1e-12, (r, ret[r])


@pytest.mark.parametrize("world", [2, 4])
def test_replicated_protocol_matches_dense_oracle(world):
    """Q = 1 replicated along the ring: each rank's partial over its shard, all-gathered and merged in rank order,
    under masks that leave whole ranks unfilled, padded or fully masked"""
    from test_attn_decode_ring_gpu import MASK_KINDS
    ret = mp.Manager().dict()
    mp.spawn(_replicated_worker, args=(world, _free_port(), ret), nprocs=world, join=True)
    assert len(ret) == world * len(MASK_KINDS)
    for (r, kind), err in sorted(ret.items()):
        assert err < 1e-12, (r, kind, err)
