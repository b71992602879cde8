"""GPU tests of generation-time decode attention: one query row against a KV cache sharded over an `sp` ring, where
every rank reduces its shard with the GEMV kernel (`decode_partial_kernel`) and the per-rank (o, max, sum) partials
are merged by `decode_merge_kernel`. The reference is a float64 restatement of
oracle.attn_dense.attention_inference_dense computed on the device (checked against the numpy oracle first), with
its natural-log lse:
  * the replicated protocol `_infer_replicated` emulated with threads at world 2, 4 and 8: per-rank operand
    magnitudes, generation masks that leave whole ranks unfilled or padded, a fully masked batch row, a
    batch-broadcast mask, and peaked logits whose rank maxima lie more than 126 apart in log2;
  * caches of 131072 and 2^20 + 3 keys, where each CTA of the GEMV kernel takes more than 2048 keys;
  * the kernel's split and warp edges: key counts around 16 keys per iteration and 2048 keys per split, and rows
    whose only visible key sits in the last, short split, at the mask offsets of ranks 1 and 3 of a 4-way ring;
  * the lse that decode_merge(..., with_lse=True) returns.
Every output row is checked: relative Frobenius error <= 1e-5 (fp32) or 3e-3 (bf16, 8 significant bits), lse within
1e-5 * max(1, |lse|) for rows with a visible key."""
import math
import threading

import numpy as np
import pytest
import torch

from thread_comm import run_ranks

pytestmark = pytest.mark.gpu

TOL = {torch.float32: 1e-5, torch.bfloat16: 3e-3}
FINFO_MIN = -3.3895313892515355e38        # the reference's finfo(bfloat16).min, as in oracle.attn_dense
D = 128


def generation_mask(kind, B, Sl, world):
    """The mask of one generation step (decode_attention_mask, Q = 1) over a cache of world * Sl slots:
      in_rank0    cache_index inside rank 0: ranks 1.. hold only unfilled slots
      boundary    cache_index on the last slot of rank 0: rank 1 and later see nothing
      boundary1   cache_index on the first slot of rank 1: rank 1 sees one key
      left_pad    batch 0 padded over all of rank 0 and half of rank 1
      dead_row    batch 1 padded everywhere: no visible key on any rank
      broadcast   one [1,1,1,K] mask for the whole batch
      none        no mask
    -> bool [B or 1, 1, 1, K] (CPU) or None"""
    from lwm_b200.ringattention import decode_attention_mask
    K = world * Sl
    pad = torch.ones(B, K, dtype=torch.int32)
    idx = K - 4
    if kind == "none":
        return None
    if kind == "in_rank0":
        idx = Sl // 3
    elif kind == "boundary":
        idx = Sl - 1
    elif kind == "boundary1":
        idx = Sl
    elif kind == "left_pad":
        pad[0, :Sl + Sl // 2] = 0
    elif kind == "dead_row":
        pad[1, :] = 0
    elif kind == "broadcast":
        pad = pad[:1].clone()
        pad[0, :Sl // 2 + 5] = 0
    else:
        raise ValueError(kind)
    pad[0, :7] = 0
    return decode_attention_mask(pad, 1, idx, K)


MASK_KINDS = ["in_rank0", "boundary", "boundary1", "left_pad", "dead_row", "broadcast", "none"]


def ref_attention(q, k, v, mask, chunk=1 << 18):
    """float64 `ringattention_inference` on the device: q [B,Q,H,D], k/v [B,K,H,D] (the whole cache), mask bool or
    uint8 [Bm,1,Q,K] or None; s = where(mask, q.k / sqrt(D), finfo.min), out = softmax(s) v.
    -> (out [B,Q,H,D], lse [B,Q,H] natural log), float64. Chunked over keys so a 2^20-key cache stays small."""
    B, Q, H, _ = q.shape
    K = k.shape[1]
    qd = q.double()
    s = torch.empty(B, H, Q, K, dtype=torch.float64, device=q.device)
    for j in range(0, K, chunk):
        s[..., j:j + chunk] = torch.einsum("bqhd,bkhd->bhqk", qd, k[:, j:j + chunk].double())
    s /= math.sqrt(D)
    if mask is not None:
        s.masked_fill_(mask.to(s.device) == 0, FINFO_MIN)
    m = s.amax(-1, keepdim=True)
    p = torch.exp(s - m)
    den = p.sum(-1, keepdim=True)
    p /= den
    out = torch.zeros(B, Q, H, D, dtype=torch.float64, device=q.device)
    for j in range(0, K, chunk):
        out += torch.einsum("bhqk,bkhd->bqhd", p[..., j:j + chunk], v[:, j:j + chunk].double())
    return out, (m + torch.log(den))[..., 0].transpose(1, 2)


def visible_rows(mask, B, Q, H):
    """[B,Q,H] bool: rows with at least one visible key (all rows when mask is None)"""
    if mask is None:
        return torch.ones(B, Q, H, dtype=torch.bool)
    return (mask.cpu() != 0).any(-1)[:, 0].expand(B, Q)[..., None].expand(B, Q, H)


def check_rows(out, ref, dtype):
    """every row [.., D] finite and within TOL[dtype] relative Frobenius error -> the worst row's error"""
    assert out.dtype == dtype
    o = out.double().reshape(-1, D)
    r = ref.reshape(-1, D)
    assert torch.isfinite(o).all()
    err = ((o - r).norm(dim=-1) / r.norm(dim=-1).clamp_min(1e-300)).max().item()
    assert err < TOL[dtype], err
    return err


def check_lse(lse, ref_lse, rows):
    """lse [B*Q*H] against the float64 lse on the rows that see a key -> the worst error in units of max(1, |lse|)"""
    got = lse.double().reshape(ref_lse.shape)[rows.to(lse.device)]
    want = ref_lse[rows.to(ref_lse.device)]
    assert torch.isfinite(got).all()
    err = ((got - want).abs() / want.abs().clamp_min(1.0)).max().item() if want.numel() else 0.0
    assert err <= 1e-5, err
    return err


def _randn(shape, seed, scale=1.0, dtype=torch.float32):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


def _ring_cache(world, B, H, Sl, dtype, seed):
    """K and V of a world-rank cache, rank r's shard with its own magnitudes: keys 2^-r (so the logits of rank r
    scale as 2^-r), values 2^(6r), 2^(-6r) alternately"""
    k = torch.cat([_randn((B, Sl, H, D), seed + 2 * r, 2.0 ** -r) for r in range(world)], 1)
    v = torch.cat([_randn((B, Sl, H, D), seed + 2 * r + 1, 2.0 ** (6 * r * (-1) ** r)) for r in range(world)], 1)
    return k.to(dtype), v.to(dtype)


def _run_replicated(q, k, v, mask, world):
    """_infer_replicated on `world` threads over shards of k/v, with the real kernels
    -> (per-rank outputs, per-rank lse of the merge)"""
    from lwm_b200 import ringattention as ra
    Sl = k.shape[1] // world
    lses = [None] * world
    local = threading.local()

    class LseOps(ra.InferOps):
        @staticmethod
        def merge(o, ml, n_part, out_shape, dtype):
            out, lses[local.rank] = ra.decode_merge(o, ml, n_part, out_shape, dtype, with_lse=True)
            return out

    def rank_fn(r, comm):
        local.rank = r
        keys = slice(r * Sl, (r + 1) * Sl)
        return ra._infer_replicated(q, k[:, keys].contiguous(), v[:, keys].contiguous(), mask, r, comm, LseOps)

    outs = run_ranks(world, rank_fn)
    torch.cuda.synchronize()
    return outs, lses


def test_device_reference_matches_numpy_oracle():
    from oracle.attn_dense import attention_inference_dense
    B, Q, H, K = 2, 3, 2, 77
    q = _randn((B, Q, H, D), 41, 1.5, torch.float64)
    k = _randn((B, K, H, D), 42, 1.5, torch.float64)
    v = _randn((B, K, H, D), 43, 1.0, torch.float64)
    mask = torch.rand(B, 1, Q, K, generator=torch.Generator().manual_seed(0)) < 0.4
    mask[0, 0, 1] = False                  # a fully masked row: uniform average over every key
    mask[1, 0, 2, :-1] = False             # only the last key
    out, lse = ref_attention(q, k, v, mask.cuda(), chunk=32)
    want = attention_inference_dense(q.cpu().numpy(), k.cpu().numpy(), v.cpu().numpy(), mask.numpy())
    np.testing.assert_allclose(out.cpu().numpy(), want, rtol=1e-12, atol=1e-12)
    s = np.einsum("bqhd,bkhd->bqhk", q.cpu().numpy(), k.cpu().numpy()) / np.sqrt(D)
    s = np.where(mask.numpy()[:, 0, :, None, :], s, FINFO_MIN)
    mx = s.max(-1)
    want_lse = mx + np.log(np.exp(s - mx[..., None]).sum(-1))
    np.testing.assert_allclose(lse.cpu().numpy(), want_lse, rtol=1e-12)


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("kind", MASK_KINDS)
def test_replicated_ring_generation_step(world, dtype, kind):
    """a generation step on an emulated ring == the float64 reference on the whole cache == the single-GPU call on
    the concatenated cache; every rank returns the same bits"""
    from lwm_b200.ringattention import ringattention_inference
    B, H, Sl = 2, 3, 2500                  # 2 key splits per rank, 1250 keys each: not a multiple of 16
    seed = 1000 * world + 10 * MASK_KINDS.index(kind) + (dtype == torch.float32)
    q = _randn((B, 1, H, D), seed, 1.0, dtype)
    k, v = _ring_cache(world, B, H, Sl, dtype, seed + 1)
    mask = generation_mask(kind, B, Sl, world)
    mask_d = None if mask is None else mask.cuda()
    outs, lses = _run_replicated(q, k, v, mask_d, world)
    ref, ref_lse = ref_attention(q, k, v, mask_d)
    for r in range(1, world):
        assert torch.equal(outs[r], outs[0]) and torch.equal(lses[r], lses[0]), r
    err = check_rows(outs[0], ref, dtype)
    lse_err = check_lse(lses[0], ref_lse, visible_rows(mask, B, 1, H))
    whole = ringattention_inference(q, k, v, mask_d)
    torch.cuda.synchronize()
    check_rows(whole, ref, dtype)
    check_rows(outs[0], whole.double(), dtype)
    print("ring world=%d %s %s: out %.2e lse %.2e" % (world, str(dtype)[6:], kind, err, lse_err))


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_replicated_ring_peaked_logits(world, dtype):
    """q x 16 and one planted key per (batch, head) whose logit beats every other by more than 126 in log2: each
    row is one-hot on a key that sits on a different rank per head, and the other ranks' partial maxima fall more
    than 126 below it (their merge weight ex2(m_r - m) underflows to 0)"""
    B, H, Sl = 2, 3, 2500
    seed = 77 * world + (dtype == torch.float32)
    q = _randn((B, 1, H, D), seed, 16.0)
    k, v = _ring_cache(world, B, H, Sl, torch.float32, seed + 1)
    for b in range(B):
        for h in range(H):
            r = (h + 2 * b) % world
            j = r * Sl + (97 * (h + 1) + 13 * b) % Sl
            k[b, j, h] = q[b, 0, h] / q[b, 0, h].norm() * 12.0     # logit ~ 16 * 11.3 * 12 / 11.3 = 192
    q, k, v = q.to(dtype), k.to(dtype), v.to(dtype)
    ref, ref_lse = ref_attention(q, k, v, None)
    s = torch.einsum("bqhd,bkhd->bqhk", q.double(), k.double()) / math.sqrt(D) * math.log2(math.e)
    top2 = s.topk(2, dim=-1).values
    assert (top2[..., 0] - top2[..., 1] > 126).all()                # the setup really is peaked
    outs, lses = _run_replicated(q, k, v, None, world)
    err = check_rows(outs[0], ref, dtype)
    lse_err = check_lse(lses[0], ref_lse, visible_rows(None, B, 1, H))
    print("peaked world=%d %s: out %.2e lse %.2e" % (world, str(dtype)[6:], err, lse_err))


@pytest.mark.parametrize("K", [131072, 2 ** 20 + 3])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("masked", [True, False], ids=["pad", "nomask"])
def test_long_cache_decode(K, dtype, masked):
    """Q = 1 on one GPU at 128K and 1M keys: 64 and 256 key splits, the latter more than 2048 keys per CTA"""
    from lwm_b200 import ringattention as ra
    B, H = 2, 2
    seed = K + 2 * (dtype == torch.float32) + masked
    q = _randn((B, 1, H, D), seed, 1.0, dtype)
    k = _randn((B, K, H, D), seed + 1, 1.0, dtype)
    v = _randn((B, K, H, D), seed + 2, 1.0, dtype)
    mask = None
    if masked:
        pad = torch.ones(B, K, dtype=torch.int32, device="cuda")
        pad[0, :1000] = 0
        pad[1, :K // 3 + 1] = 0
        mask = ra.decode_attention_mask(pad, 1, K - 9, K)          # left padding and 8 unfilled slots
    out = ra.ringattention_inference(q, k, v, mask)
    o, ml = ra.decode_partial(q, k, v, None if mask is None else mask.to(torch.uint8), 0)
    out2, lse = ra.decode_merge(o, ml, 1, (B, 1, H, D), dtype, with_lse=True)
    torch.cuda.synchronize()
    assert torch.equal(out2, out)
    ref, ref_lse = ref_attention(q, k, v, mask)
    err = check_rows(out, ref, dtype)
    lse_err = check_lse(lse, ref_lse, visible_rows(mask, B, 1, H))
    print("long K=%d %s %s: out %.2e lse %.2e" % (K, str(dtype)[6:], "pad" if masked else "nomask", err, lse_err))


ROW_KINDS = ["last", "dead", "random", "all", "first", "last_split", "split_edge"]


def _row_mask(kind, Sk, gen):
    """one row's mask over a shard of Sk keys, in terms of decode_partial's key splits"""
    splits = max(1, min(256, (Sk + 2047) // 2048))
    per = (Sk + splits - 1) // splits
    m = torch.zeros(Sk, dtype=torch.uint8)
    if kind == "last":                  # the only visible key is the shard's last: the last, short split
        m[-1] = 1
    elif kind == "random":
        m = (torch.rand(Sk, generator=gen) < 0.3).to(torch.uint8)
    elif kind == "all":
        m[:] = 1
    elif kind == "first":
        m[0] = 1
    elif kind == "last_split":          # only the last split's keys, every third one
        m[(splits - 1) * per::3] = 1
    elif kind == "split_edge":          # the last key of split 0 and the first of split 1
        m[min(per, Sk) - 1] = 1
        m[min(per, Sk - 1)] = 1
    return m


SPLIT_SKS = [1, 3, 4, 15, 16, 17, 2047, 2048, 2049, 4097, 6145, 256 * 2048 + 1]


@pytest.mark.parametrize("Sk", SPLIT_SKS)
@pytest.mark.parametrize("Q", [1, 3, 7])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_split_and_warp_edges(Sk, Q, dtype):
    """decode_partial + decode_merge at the mask offsets k_pos0 of ranks 1 and 3 of a 4-way ring (the mask columns
    of the other ranks hold noise): each rank's partial alone, and the two merged, against the float64 reference"""
    from lwm_b200 import ringattention as ra
    B, H, W = 2, 2, 4
    gen = torch.Generator().manual_seed(Sk * 10 + Q)
    kinds = ROW_KINDS[:Q]
    mask = (torch.rand(B, 1, Q, W * Sk, generator=gen) < 0.5).to(torch.uint8)
    for r in (1, 3):
        for b in range(B):
            for i in range(Q):          # batch 1 takes the row kinds rotated by one
                mask[b, 0, i, r * Sk:(r + 1) * Sk] = _row_mask(kinds[(i + b) % Q], Sk, gen)
    mask = mask.cuda()
    seed = 3 * Sk + Q + (dtype == torch.float32)
    q = _randn((B, Q, H, D), seed, 1.0, dtype)
    shards, parts = {}, {}
    errs = []
    for r in (1, 3):
        k = _randn((B, Sk, H, D), seed + 10 * r, 2.0 ** -r, dtype)
        v = _randn((B, Sk, H, D), seed + 10 * r + 1, 2.0 ** (6 * r), dtype)
        cols = mask[..., r * Sk:(r + 1) * Sk]
        o, ml = ra.decode_partial(q, k, v, mask, r * Sk)
        out, lse = ra.decode_merge(o, ml, 1, (B, Q, H, D), dtype, with_lse=True)
        ref, ref_lse = ref_attention(q, k, v, cols)
        errs.append((check_rows(out, ref, dtype), check_lse(lse, ref_lse, visible_rows(cols, B, Q, H))))
        shards[r], parts[r] = (k, v, cols), (o, ml)
    o = torch.stack([parts[1][0], parts[3][0]], 1).contiguous()
    ml = torch.stack([parts[1][1], parts[3][1]], 1).contiguous()
    out, lse = ra.decode_merge(o, ml, 2, (B, Q, H, D), dtype, with_lse=True)
    k, v, cols = (torch.cat([shards[1][i], shards[3][i]], 1 if i < 2 else -1) for i in range(3))
    ref, ref_lse = ref_attention(q, k, v, cols)
    errs.append((check_rows(out, ref, dtype), check_lse(lse, ref_lse, visible_rows(cols, B, Q, H))))
    print("split Sk=%d Q=%d %s: out %.2e lse %.2e" % (Sk, Q, str(dtype)[6:], max(e[0] for e in errs),
                                                     max(e[1] for e in errs)))
