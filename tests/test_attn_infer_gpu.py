"""GPU tests of `ringattention_inference` on the tensor-core path (Q >= INFER_MIN_Q), in fp32 and bf16, against the
dense float64 oracle: parity over query/key lengths that are not multiples of 128 with decode, block-sparse,
batch-broadcast and absent masks; exact power-of-two scaling; large shapes; the fp32 decode kernel; the q-sharded
ring protocol emulated on one GPU with threads; and a prefill + decode generation loop on a KV cache."""
import os

import numpy as np
import pytest
import torch

from helpers import rel_fro, to_np
from thread_comm import run_ranks

pytestmark = pytest.mark.gpu

TOL = {torch.float32: 1e-3, torch.bfloat16: 3e-3}


def _qkv(B, Q, K, H, dtype, seed, mags=(1.0, 1.0, 1.0)):
    g = torch.Generator().manual_seed(seed)
    t = [torch.randn(B, n, H, 128, generator=g) * m for n, m in zip((Q, K, K), mags)]
    return [x.to(dtype).cuda() for x in t]


def _mask(kind, B, Q, K, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "none":
        return None
    if kind == "decode":      # left-padded prompt, cache_index > 0 (the generation call site)
        from lwm_b200.ringattention import decode_attention_mask
        pad = torch.ones(B, K, dtype=torch.int32)
        pad[0, :19] = 0
        if B > 1:
            pad[1, :141] = 0
        return decode_attention_mask(pad, Q, max(0, K - Q - 5), K)
    if kind == "blocks":      # whole-false and whole-true 128x128 tiles, random elsewhere, one fully masked row
        nq, nk = (Q + 127) // 128, (K + 127) // 128
        kind_t = torch.randint(0, 3, (B, nq, nk), generator=g)
        rnd = torch.rand(B, Q, K, generator=g) < 0.5
        t = kind_t.repeat_interleave(128, 1).repeat_interleave(128, 2)[:, :Q, :K]
        m = torch.where(t == 0, torch.zeros_like(rnd), torch.where(t == 1, torch.ones_like(rnd), rnd))
        m[:, min(2, Q - 1)] = False
        return m[:, None]
    if kind == "broadcast":   # one causal mask for the whole batch, with a fully masked row
        m = (torch.arange(K)[None, :] <= (torch.arange(Q) + K - Q)[:, None])[None, None].clone()
        m[..., Q // 2, :] = False
        return m
    raise ValueError(kind)


def _ref(q, k, v, mask):
    from oracle.attn_dense import attention_inference_dense
    B = q.shape[0]
    m = None if mask is None else np.broadcast_to(mask.numpy(), (B,) + tuple(mask.shape[1:]))
    return attention_inference_dense(to_np(q), to_np(k), to_np(v), m)


def _check(out, ref, dtype, mask):
    o = to_np(out)
    assert out.dtype == dtype
    assert np.isfinite(o).all()
    assert rel_fro(o, ref) < TOL[dtype], rel_fro(o, ref)


CASES = [(Q, K) for Q in (8, 128, 200, 1000) for K in (Q, Q + 77, 4096)]   # 8 = INFER_MIN_Q


@pytest.mark.parametrize("Q,K", CASES)
@pytest.mark.parametrize("B,H", [(1, 1), (2, 3)])
@pytest.mark.parametrize("kind", ["decode", "blocks", "broadcast", "none"])
def test_tensor_core_path_matches_oracle_fp32(Q, K, B, H, kind):
    from lwm_b200.ringattention import ringattention_inference, INFER_MIN_Q
    assert Q >= INFER_MIN_Q
    q, k, v = _qkv(B, Q, K, H, torch.float32, Q * 7 + K)
    mask = _mask(kind, B, Q, K, Q + K)
    out = ringattention_inference(q, k, v, None if mask is None else mask.cuda())
    torch.cuda.synchronize()
    _check(out, _ref(q, k, v, mask), torch.float32, mask)


@pytest.mark.parametrize("Q,K", [(8, 81), (200, 4096), (1000, 1077)])
@pytest.mark.parametrize("kind", ["decode", "blocks"])
def test_tensor_core_path_matches_oracle_bf16(Q, K, kind):
    from lwm_b200.ringattention import ringattention_inference
    q, k, v = _qkv(2, Q, K, 3, torch.bfloat16, Q + K)
    mask = _mask(kind, 2, Q, K, K)
    out = ringattention_inference(q, k, v, mask.cuda())
    torch.cuda.synchronize()
    _check(out, _ref(q, k, v, mask), torch.bfloat16, mask)


def test_fully_masked_rows_average_all_values():
    from lwm_b200.ringattention import ringattention_inference
    Q, K = 200, 333
    q, k, v = _qkv(1, Q, K, 2, torch.float32, 1)
    mask = torch.ones(1, 1, Q, K, dtype=torch.bool)
    mask[..., 5, :] = False
    mask[..., 150:, :] = False
    out = to_np(ringattention_inference(q, k, v, mask.cuda()))
    mean = to_np(v).mean(axis=1)
    for r in [5] + list(range(150, Q)):
        assert rel_fro(out[0, r], mean[0]) < 1e-3     # V enters as its scaled fp16 copy


@pytest.mark.parametrize("e", [-20, 0, 20])
def test_scaling_v_scales_the_output_exactly(e):
    from lwm_b200.ringattention import ringattention_inference
    q, k, v = _qkv(1, 300, 1000, 2, torch.float32, 3)
    mask = _mask("blocks", 1, 300, 1000, 4).cuda()
    a = ringattention_inference(q, k, v, mask)
    b = ringattention_inference(q, k, v * 2.0 ** e, mask)
    torch.cuda.synchronize()
    assert torch.equal(b, a * 2.0 ** e)


def test_large_causal_prefill_on_sampled_rows():
    from lwm_b200.ringattention import ringattention_inference
    S, H = 32768, 4
    q, k, v = _qkv(1, S, S, H, torch.bfloat16, 11)
    mask = torch.ones(S, S, dtype=torch.bool, device="cuda").tril_()[None, None]
    out = ringattention_inference(q, k, v, mask)
    torch.cuda.synchronize()
    rows = torch.tensor([0, 1, 127, 128, 4095, 20000, S - 129, S - 1])
    ref = _ref(q[:, rows].cpu(), k.cpu(), v.cpu(), mask[:, :, rows].cpu())
    assert rel_fro(to_np(out[:, rows]), ref) < 3e-3


def test_query_longer_than_the_grid_limit_runs():
    from lwm_b200.ringattention import ringattention_inference
    Q, K = 65664, 256
    q, k, v = _qkv(1, Q, K, 1, torch.float32, 13)
    mask = torch.ones(1, 1, Q, K, dtype=torch.bool)
    mask[..., :K // 2, K // 2:] = False
    out = ringattention_inference(q, k, v, mask.cuda())
    torch.cuda.synchronize()
    rows = torch.tensor([0, 100, 40000, Q - 1])
    ref = _ref(q[:, rows].cpu(), k.cpu(), v.cpu(), mask[:, :, rows])
    assert rel_fro(to_np(out[:, rows]), ref) < 1e-3


@pytest.mark.parametrize("K", [4096, 131072])
def test_fp32_decode_matches_float64(K):
    from lwm_b200.ringattention import ringattention_inference
    q, k, v = _qkv(1, 1, K, 4, torch.float32, K)
    mask = torch.ones(1, 1, 1, K, dtype=torch.bool)
    mask[..., :33] = False
    out = ringattention_inference(q, k, v, mask.cuda())
    torch.cuda.synchronize()
    assert out.dtype == torch.float32
    assert rel_fro(to_np(out), _ref(q, k, v, mask)) < 1e-5


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("Ql,dtype", [(37, torch.float32), (130, torch.float32), (37, torch.bfloat16)])
def test_q_sharded_ring_emulated_with_threads(world, Ql, dtype):
    """the protocol through a thread fake comm and the real kernels; every rank's q, k, v has its own magnitude"""
    from lwm_b200 import ringattention as ra
    B, H, Sl = 2, 3, 300
    Q, K = world * Ql, world * Sl
    parts = [_qkv(B, Ql, Sl, H, torch.float32, 100 + r, mags=(2.0 ** -r, 2.0 ** -r, 2.0 ** (6 * r)))
             for r in range(world)]
    q = torch.cat([p[0] for p in parts], 1).to(dtype)
    k = torch.cat([p[1] for p in parts], 1).to(dtype)
    v = torch.cat([p[2] for p in parts], 1).to(dtype)
    mask = _mask("decode", B, Q, K, 0)
    mask[..., 1, :] = False
    mask[..., Q - 2, :] = False
    mask_d = mask.cuda()

    def rank_fn(r, comm):
        rows, keys = slice(r * Ql, (r + 1) * Ql), slice(r * Sl, (r + 1) * Sl)
        return ra._infer_sharded(q[:, rows].contiguous(), k[:, keys].contiguous(), v[:, keys].contiguous(),
                                 mask_d[:, :, rows].contiguous(), comm)
    outs = run_ranks(world, rank_fn)
    torch.cuda.synchronize()
    out = torch.cat(outs, 1)
    ref = _ref(q, k, v, mask)
    _check(out, ref, dtype, mask)


def test_generation_loop_on_fp32_kv_cache():
    """prefill a left-padded 300-token prompt (Q > 1), then 5 decode steps (Q = 1), each against the oracle"""
    from lwm_b200.kv_cache import ShardedKVCache
    from lwm_b200.ringattention import ringattention_inference, decode_attention_mask
    B, H, P, steps = 2, 3, 300, 5
    L = P + steps
    pad = torch.ones(B, L, dtype=torch.int32)
    pad[0, :37] = 0
    cache = ShardedKVCache(B, L, H, 128, dtype=torch.float32, device="cuda")
    g = torch.Generator().manual_seed(5)
    keys = []
    for t in range(steps + 1):
        n = P if t == 0 else 1
        q, kn, vn = (torch.randn(B, n, H, 128, generator=g).cuda() for _ in range(3))
        keys.append(kn)
        ck, cv = cache.concatenate(kn, vn)
        idx = cache.cache_index - n
        mask = decode_attention_mask(pad.cuda(), n, idx, L)
        out = ringattention_inference(q, ck, cv, mask)
        torch.cuda.synchronize()
        assert torch.equal(ck[:, :cache.cache_index], torch.cat(keys, 1))
        # the whole cache, empty slots included: the prompt's padded rows average V over every slot, as in the reference
        ref = _ref(q, ck, cv, mask.cpu())
        assert out.dtype == torch.float32
        assert rel_fro(to_np(out), ref) < (1e-3 if n > 1 else 1e-5), (t, rel_fro(to_np(out), ref))


def _nccl_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        from lwm_b200.ringattention import ringattention_inference
        B, H, Ql, Sl = 1, 2, 100, 256
        g = torch.Generator().manual_seed(0)
        q = torch.randn(B, world * Ql, H, 128, generator=g)
        k = torch.randn(B, world * Sl, H, 128, generator=g)
        v = torch.randn(B, world * Sl, H, 128, generator=g)
        mask = torch.ones(1, 1, world * Ql, world * Sl, dtype=torch.bool).tril_(world * Sl - world * Ql)
        rows, keys = slice(rank * Ql, (rank + 1) * Ql), slice(rank * Sl, (rank + 1) * Sl)
        out = ringattention_inference(q[:, rows].cuda(), k[:, keys].cuda(), v[:, keys].cuda(),
                                      mask[:, :, rows].cuda())
        ret[rank] = rel_fro(to_np(out), _ref(q, k, v, mask)[:, rows])
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_q_sharded_ring_on_two_gpus():
    import socket
    import torch.multiprocessing as mp
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ret = mp.Manager().dict()
    mp.spawn(_nccl_worker, args=(2, port, ret), nprocs=2, join=True)
    assert max(ret.values()) < 1e-3
