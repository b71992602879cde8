"""Dense float64 attention oracle with the reference's mask semantics.

Follows the call-site contract lwm/llama.py:525-570 (additive `attn_bias` [B,1,1,S] built from
the mask as 0 / finfo(dtype).min at llama.py:533-537, optional segment ids, token-level causal
mask: causal_block_size=1 at llama.py:546) and SURVEY.md Appendix A `chunk_bias`: the three masks
are combined with `minimum`, never summed, and then ADDED to the scaled logits.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).
"""
import numpy as np


def finfo_min(dtype_name):
    """jnp.finfo(dtype).min for the dtypes the reference runs with (llama.py:536)."""
    if dtype_name in ("bf16", "bfloat16"):
        return -3.3895313892515355e38
    if dtype_name in ("fp32", "float32"):
        return float(np.finfo(np.float32).min)
    raise ValueError(dtype_name)


def dense_bias(B, Sq, Sk, q_pos0=0, k_pos0=0, attn_bias=None, segment_ids=None, causal=True, mask_value=None):
    """[B,1,Sq,Sk] additive bias = min(bias, segment mask, causal mask) on GLOBAL positions."""
    if mask_value is None:
        mask_value = finfo_min("bf16")
    q_pos = q_pos0 + np.arange(Sq)
    k_pos = k_pos0 + np.arange(Sk)
    b = np.zeros((B, 1, Sq, Sk), dtype=np.float64)
    if attn_bias is not None:
        ab = np.asarray(attn_bias, dtype=np.float64).reshape(B, -1)  # [B, S_global]
        b = b + ab[:, None, None, k_pos]                             # bias broadcast over queries
    if segment_ids is not None:
        seg = np.asarray(segment_ids).reshape(B, -1)
        neq = seg[:, q_pos][:, :, None] != seg[:, k_pos][:, None, :]
        b = np.minimum(b, neq[:, None].astype(np.float64) * mask_value)
    if causal:
        c = (q_pos[:, None] < k_pos[None, :]).astype(np.float64) * mask_value
        b = np.minimum(b, c[None, None])
    return b


def attention_dense(q, k, v, attn_bias=None, segment_ids=None, causal=True, q_pos0=0, k_pos0=0,
                    mask_value=None, return_lse=False):
    """q [B,Sq,H,D], k/v [B,Sk,H,D] (any float dtype) -> out [B,Sq,H,D] float64.

    The logits are evaluated in float32 before the mask is added, mirroring the reference's
    fp32 absorption of the logit by finfo.min (s + finfo.min == finfo.min in fp32), so that a row
    whose keys are all masked averages them uniformly instead of following the tiny logit gaps.
    """
    q = np.asarray(q, dtype=np.float64)
    k = np.asarray(k, dtype=np.float64)
    v = np.asarray(v, dtype=np.float64)
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    s = np.einsum("bqhd,bkhd->bhqk", q, k) / np.sqrt(D)
    b = dense_bias(B, Sq, Sk, q_pos0, k_pos0, attn_bias, segment_ids, causal, mask_value)
    mv = finfo_min("bf16") if mask_value is None else mask_value
    masked = b <= mv * 0.5
    s = np.where(masked, b, s + b)           # fp32 absorption: masked logits are exactly the mask value
    m = s.max(axis=-1, keepdims=True)
    p = np.exp(s - m)
    den = p.sum(axis=-1, keepdims=True)
    out = np.einsum("bhqk,bkhd->bqhd", p / den, v)
    if return_lse:
        return out, (m + np.log(den))[..., 0]  # [B,H,Sq]
    return out


def attention_dense_grads(q, k, v, dout, **kw):
    """Closed-form float64 gradients (dq, dk, dv) of attention_dense w.r.t. q, k, v."""
    q = np.asarray(q, dtype=np.float64)
    k = np.asarray(k, dtype=np.float64)
    v = np.asarray(v, dtype=np.float64)
    g = np.asarray(dout, dtype=np.float64)
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    s = np.einsum("bqhd,bkhd->bhqk", q, k) / np.sqrt(D)
    b = dense_bias(B, Sq, Sk, kw.get("q_pos0", 0), kw.get("k_pos0", 0), kw.get("attn_bias"),
                   kw.get("segment_ids"), kw.get("causal", True), kw.get("mask_value"))
    mv = finfo_min("bf16") if kw.get("mask_value") is None else kw["mask_value"]
    masked = b <= mv * 0.5
    s = np.where(masked, b, s + b)
    m = s.max(axis=-1, keepdims=True)
    p = np.exp(s - m)
    p = p / p.sum(axis=-1, keepdims=True)
    out = np.einsum("bhqk,bkhd->bqhd", p, v)
    dv = np.einsum("bhqk,bqhd->bkhd", p, g)
    dp = np.einsum("bqhd,bkhd->bhqk", g, v)
    delta = np.einsum("bqhd,bqhd->bhq", g, out)
    ds = p * (dp - delta[..., None])
    dq = np.einsum("bhqk,bkhd->bqhd", ds, k) / np.sqrt(D)
    dk = np.einsum("bhqk,bqhd->bkhd", ds, q) / np.sqrt(D)
    return dq, dk, dv


def visible_pairs(B, Sq, Sk, q_pos0=0, k_pos0=0, attn_bias=None, segment_ids=None, causal=True, mask_value=None):
    """[B,1,Sq,Sk] bool: the (q, k) pairs that dense_bias leaves unmasked"""
    mv = finfo_min("bf16") if mask_value is None else mask_value
    return dense_bias(B, Sq, Sk, q_pos0, k_pos0, attn_bias, segment_ids, causal, mask_value) > mv * 0.5


def _contract(w, x, vis, over_keys):
    """sum_j w[b,h,i,j] x[b,j,h,:] (over_keys) or sum_i w[b,h,i,j] x[b,i,h,:], w zero outside vis [B,1,Sq,Sk]: a
    non-finite entry of x enters only the products of the pairs in vis (0 * inf would make every pair NaN)"""
    fin = np.isfinite(x)
    r = np.einsum("bhqk,bkhd->bqhd" if over_keys else "bhqk,bqhd->bkhd", w, np.where(fin, x, 0.0))
    for b, n, h, d in zip(*np.nonzero(~fin)):
        col, vc = (w[b, h, :, n], vis[b, 0, :, n]) if over_keys else (w[b, h, n, :], vis[b, 0, n, :])
        r[b, :, h, d] += np.where(vc, col * x[b, n, h, d], 0.0)
    return r


def attention_visible(q, k, v, visible, dout=None, mask_value=None):
    """float64 attention over the pairs where visible [B or 1,1,Sq,Sk] holds, with the masked pairs kept out of every
    sum by np.where instead of an additive finfo.min, so that a NaN or inf operand reaches only the pairs that see it
    (NaN + finfo.min would be NaN). A row with no visible pair averages every key uniformly, as attention_dense's fully
    masked rows do; on finite inputs the results equal attention_dense / attention_dense_grads (and
    attention_inference_dense). -> (out [B,Sq,H,D], lse [B,H,Sq]), with dout also (dq, dk, dv)."""
    q, k, v = (np.asarray(t, dtype=np.float64) for t in (q, k, v))
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    mv = finfo_min("bf16") if mask_value is None else mask_value
    vis = np.broadcast_to(np.asarray(visible, dtype=bool), (B, 1, Sq, Sk))
    live = vis.any(-1, keepdims=True)                      # [B,1,Sq,1]
    vis = vis | ~live
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        s = np.einsum("bqhd,bkhd->bhqk", q, k) / np.sqrt(D)
        s = np.where(live, np.where(vis, s, -np.inf), 0.0)    # dead rows: equal logits, a uniform average
        m = s.max(axis=-1, keepdims=True)
        p = np.where(vis, np.exp(s - m), 0.0)
        den = p.sum(axis=-1, keepdims=True)
        p = p / den
        out = _contract(p, v, vis, True)
        lse = np.where(live[..., 0], (m + np.log(den))[..., 0], mv + np.log(Sk))
        if dout is None:
            return out, lse
        g = np.asarray(dout, dtype=np.float64)
        dv = _contract(p, g, vis, False)
        dp = np.einsum("bqhd,bkhd->bhqk", g, v)
        delta = np.einsum("bqhd,bqhd->bhq", g, out)
        ds = np.where(vis, p * (dp - delta[..., None]), 0.0)
        dq = _contract(ds, k, vis, True) / np.sqrt(D)
        dk = _contract(ds, q, vis, False) / np.sqrt(D)
    return out, lse, dq, dk, dv


def attention_inference_dense(q, k, v, attn_mask, mask_value=None):
    """`ringattention_inference` semantics (SURVEY.md Appendix A; call site lwm/llama.py:601-614):
    q [B,Q,H,D], k/v [B,K,H,D] (the whole, un-sharded cache), attn_mask bool [B,1,Q,K]:
    s = where(mask, q.k/sqrt(D), finfo.min); out = softmax(s) v. float64."""
    q = np.asarray(q, dtype=np.float64)
    k = np.asarray(k, dtype=np.float64)
    v = np.asarray(v, dtype=np.float64)
    mv = finfo_min("bf16") if mask_value is None else mask_value
    s = np.einsum("bqhd,bkhd->bhqk", q, k) / np.sqrt(q.shape[-1])
    if attn_mask is not None:
        s = np.where(np.asarray(attn_mask, dtype=bool), s, mv)
    m = s.max(axis=-1, keepdims=True)
    p = np.exp(s - m)
    return np.einsum("bhqk,bkhd->bqhd", p / p.sum(axis=-1, keepdims=True), v)
