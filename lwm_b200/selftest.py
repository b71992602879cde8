"""On-GPU self-check used by __graft_entry__.smoke(): one small invocation of each hot path,
compared against the CPU oracle (the oracle is only ever the checker — see oracle/__init__.py)."""
import math

import numpy as np
import torch


def _rel(x, ref):
    x = np.asarray(x, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.linalg.norm(x - ref) / max(np.linalg.norm(ref), 1e-30))


def sampled_parity(S_total, H, check_heads, op, device, rank=0, world=1, base_seed=1234, shards=None, do_scale=1.0):
    """Parity of the attention op at 32K .. 128K tokens, where the dense oracle does not fit: this
    rank's shards of the seeded synthetic q/k/v (lwm_b200/synthetic.py) go through `op` (forward + backward) with a dO
    that is zero outside one sampled query row per 128-row tile (+ the last 128 rows of the sequence); the float64
    row-wise oracle (oracle/attn_rows.py) then gives, for each head in `check_heads`, the exact out / dq of the sampled
    rows and dk / dv of EVERY key row. Inputs are float32 tensors holding bf16-representable values, so `op` returns
    its un-rounded fp32 results. Returns {name: relative Frobenius error over this rank's rows}.
    op(q, k, v) -> out must be differentiable (the public ringattention op bound to the caller's process group).
    shards: optional dict(q, k, v, do) of this rank's DEVICE tensors [1, S_total/world, H, 128] already built with
    synthetic.shard(name, rank, ...) and the same base_seed (bench.py passes its timed inputs).
    do_scale: a power of two that multiplies dO (exactly, in both the op's input and the oracle's), to check the
    gradients at the magnitudes a loss averaged over many tokens produces; the relative errors are unchanged by it."""
    if do_scale <= 0 or math.frexp(do_scale)[0] != 0.5:
        raise ValueError("do_scale must be a power of two")
    from oracle.attn_rows import attention_rows, sample_rows
    from . import synthetic as syn
    D = 128
    Sl = S_total // world
    rows = sample_rows(S_total, seed=base_seed)
    lo, hi = rank * Sl, (rank + 1) * Sl
    mine = rows[(rows >= lo) & (rows < hi)]
    if shards is None:
        shards = {n_: syn.shard(n_, rank, Sl, H, D, base_seed, torch.bfloat16).to(device) for n_ in ("q", "k", "v", "do")}
    keep = torch.zeros(Sl, dtype=torch.bool)
    keep[mine - lo] = True
    do = shards["do"].float() * do_scale
    do[0, (~keep).to(device)] = 0
    qd, kd, vd = [shards[n_].float().requires_grad_(True) for n_ in ("q", "k", "v")]
    out = op(qd, kd, vd)
    out.backward(do)
    torch.cuda.synchronize()
    got = dict(out=out.detach()[0].double().cpu(), dq=qd.grad[0].double().cpu(), dk=kd.grad[0].double().cpu(),
               dv=vd.grad[0].double().cpu())
    errs = {}
    for h in check_heads:
        kg, vg = syn.head_global("k", world, h, Sl, D, base_seed), syn.head_global("v", world, h, Sl, D, base_seed)
        qg, dg = syn.head_global("q", world, h, Sl, D, base_seed), syn.head_global("do", world, h, Sl, D, base_seed) * do_scale
        ref = attention_rows(qg[rows], rows, kg, vg, dg[rows], causal=True)
        sel = (rows >= lo) & (rows < hi)
        pairs = dict(out=(got["out"][mine - lo, h], ref["out"][sel]), dq=(got["dq"][mine - lo, h], ref["dq"][sel]),
                     dk=(got["dk"][:, h], ref["dk"][lo:hi]), dv=(got["dv"][:, h], ref["dv"][lo:hi]))
        for name, (a, r) in pairs.items():
            e = float((a - r).norm() / r.norm().clamp_min(1e-300))
            errs[name] = max(errs.get(name, 0.0), e)
        # query rows whose dO is zero must get exactly zero dq
        dq_other = got["dq"][:, h].clone()
        dq_other[mine - lo] = 0
        errs["dq_unsampled_abs"] = max(errs.get("dq_unsampled_abs", 0.0), float(dq_other.abs().max()))
    errs["rows"] = int(len(mine))
    errs["keys"] = int(Sl)
    return errs


def smoke(verbose=True):
    from oracle.attn_dense import attention_dense, attention_dense_grads
    from oracle import vqgan_ref as vr
    from . import ringattention as ra
    from .vqgan import Ops, PackedConv
    res = {}
    # ---- ring attention, forward + backward through the reference-signature op (ring size 1), default precision
    # mode; inputs are bf16-representable values handed over as float32, so the results are the un-rounded fp32
    # read-out and the north_star bound (1e-3 relative Frobenius vs the float64 oracle) applies as is
    g = torch.Generator().manual_seed(0)
    B, S, H, D = 1, 512, 2, 128
    q, k, v, do = [torch.randn(B, S, H, D, generator=g).to(torch.bfloat16).float().cuda() for _ in range(4)]
    q.requires_grad_(True); k.requires_grad_(True); v.requires_grad_(True)
    kw = dict(axis_name="sp", float32_logits=True, cache_idx=None,
              blockwise_kwargs=dict(causal_block_size=1, deterministic=True, attn_pdrop=0.0,
                                    query_chunk_size=256, key_chunk_size=256))
    out = ra.ringattention(q, k, v, None, None, **kw)
    out.backward(do)
    torch.cuda.synchronize()
    n = lambda t: t.detach().float().cpu().numpy()  # noqa: E731
    ref = attention_dense(n(q), n(k), n(v), causal=True)
    rq, rk, rv = attention_dense_grads(n(q), n(k), n(v), n(do), causal=True)
    res["attn_precision_mode"] = ra._DEFAULT_PRECISION
    res["attn_fwd_rel_err"] = _rel(n(out), ref)
    res["attn_dq_rel_err"] = _rel(n(q.grad), rq)
    res["attn_dk_rel_err"] = _rel(n(k.grad), rk)
    res["attn_dv_rel_err"] = _rel(n(v.grad), rv)
    assert max(res["attn_fwd_rel_err"], res["attn_dq_rel_err"], res["attn_dk_rel_err"], res["attn_dv_rel_err"]) < 1e-3, res
    # the same op on bf16 tensors returns bf16 results: their own rounding (8 significant bits) is all that is added
    qb, kb, vb = [t.detach().to(torch.bfloat16).requires_grad_(True) for t in (q, k, v)]
    ob = ra.ringattention(qb, kb, vb, None, None, **kw)
    ob.backward(do.to(torch.bfloat16))
    torch.cuda.synchronize()
    res["attn_bf16_out_rel_err"] = _rel(n(ob), ref)
    res["attn_bf16_dq_rel_err"] = _rel(n(qb.grad), rq)
    assert res["attn_bf16_out_rel_err"] < 3e-3 and res["attn_bf16_dq_rel_err"] < 3e-3, res
    # ---- VQGAN: GroupNorm+SiLU prep -> wgmma conv, and the nearest-code search (bit-exact)
    ops = Ops("bf16x3")
    x = torch.randn(1, 16, 16, 128, generator=g)
    gn = vr._gn_p(g, 128)
    cp = vr._conv_p(g, 3, 128, 128)
    y = ops.conv(ops.prep(x.cuda(), {"scale": gn["scale"].cuda(), "bias": gn["bias"].cuda()}),
                 PackedConv(cp, torch.device("cuda")))
    yref = vr.conv2d(vr.silu(vr.group_norm(x, gn)), cp)
    res["vqgan_conv_rel_err"] = _rel(n(y), yref.numpy())
    assert res["vqgan_conv_rel_err"] < 1e-3, res
    emb = torch.randn(8192, 64, generator=g)
    z = torch.randn(256, 64, generator=g)
    _, idx = ops.vq_argmin(z.cuda(), emb.cuda())
    _, ref_idx = vr.vector_quantize(z.numpy(), emb.numpy())
    torch.cuda.synchronize()
    res["vq_indices_bit_exact"] = bool(np.array_equal(idx.cpu().numpy().astype(np.int32), ref_idx))
    assert res["vq_indices_bit_exact"], "VQ indices differ from the oracle"
    if verbose:
        print("smoke:", {k2: (("%.2e" % v2) if isinstance(v2, float) else v2) for k2, v2 in res.items()})
    return res
