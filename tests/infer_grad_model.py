"""Float64 VJP of `ringattention_inference` and a numpy model of its backward tile map (lwm_attn_infer_bwd_tilemap).

The VJP is that of oracle.attn_dense.attention_inference_dense, s = where(mask, q.k/sqrt(D), finfo.min),
out = softmax(s) v, under the project's fully-masked-row convention: a row with no true entry contributes nothing to
dq, dk or dv (its forward stays the uniform average). TEST INFRASTRUCTURE ONLY."""
import numpy as np


def attention_inference_vjp(q, k, v, attn_mask, dout):
    """q [B,Q,H,D], k/v [B,K,H,D], attn_mask bool [B,1,Q,K] or None, dout [B,Q,H,D] -> float64 (dq, dk, dv)"""
    q, k, v, g = (np.asarray(x, dtype=np.float64) for x in (q, k, v, dout))
    B, Q, H, D = q.shape
    K = k.shape[1]
    vis = np.ones((B, 1, Q, K), dtype=bool) if attn_mask is None else np.broadcast_to(
        np.asarray(attn_mask, dtype=bool), (B, 1, Q, K))
    s = np.einsum("bqhd,bkhd->bhqk", q, k) / np.sqrt(D)
    s = np.where(vis, s, -np.inf)
    live = vis.any(-1, keepdims=True)                        # [B,1,Q,1]
    m = np.where(live, s.max(-1, keepdims=True), 0.0)
    p = np.where(vis, np.exp(s - m), 0.0)
    p = p / np.where(live, p.sum(-1, keepdims=True), 1.0)   # fully masked rows: p = 0
    out = np.einsum("bhqk,bkhd->bqhd", p, v)
    dv = np.einsum("bhqk,bqhd->bkhd", p, g)
    dp = np.einsum("bqhd,bkhd->bhqk", g, v)
    delta = np.einsum("bqhd,bqhd->bhq", g, out)
    ds = p * (dp - delta[..., None])
    dq = np.einsum("bhqk,bkhd->bqhd", ds, k) / np.sqrt(D)
    dk = np.einsum("bhqk,bqhd->bkhd", ds, q) / np.sqrt(D)
    return dq, dk, dv


def pack_bits(vis, Sk):
    """bool [B,Q,Sk] -> int32 words [B,Q,ceil(Sk/128)*4] (bit j of word w <=> key 32 w + j), as lwm_attn_mask_pack"""
    B, Q = vis.shape[:2]
    kw = (Sk + 127) // 128 * 4
    pad = np.zeros((B, Q, kw * 32), dtype=bool)
    pad[..., :Sk] = vis[..., :Sk]
    return np.packbits(pad, axis=-1, bitorder="little").view("<u4").view(np.int32).reshape(B, Q, kw)


def bwd_tilemap_model(bits, row_any, B, Q, Sk):
    """The backward map from packed words: per (b, 128-key tile) the ascending 64-row Q tiles, entries t*2 + mixed.
    bits int32 [B,Q,kw] or None, row_any [B,Q] or None -> list (per b) of lists (per key tile) of entries."""
    n_kt, n_qt = (Sk + 127) // 128, (Q + 63) // 64
    live = np.ones((B, Q), dtype=bool) if row_any is None else np.asarray(row_any) != 0
    maps = []
    for b in range(B):
        per_kt = []
        for kt in range(n_kt):
            tail = (kt + 1) * 128 > Sk
            lst = []
            for t in range(n_qt):
                rows = [r for r in range(t * 64, min(Q, t * 64 + 64)) if live[b, r]]
                if not rows:
                    continue
                if bits is None:
                    any_t, all_t = True, True
                else:
                    w = bits[b, rows, kt * 4:kt * 4 + 4].view(np.uint32)
                    any_t = bool((w != 0).any())
                    all_t = bool((w == 0xFFFFFFFF).all())
                if any_t:
                    lst.append(t * 2 + int(tail or not all_t))
            per_kt.append(lst)
        maps.append(per_kt)
    return maps


def bwd_tilemap_brute(vis, B, Q, Sk):
    """The same classification element by element from the boolean mask [B,Q,Sk] (None: all visible): a pair is
    skipped when no entry of a live row (one with any true entry) is true, clean when every key of the 128-key tile
    exists and every live row sees all of them, mixed otherwise."""
    n_kt, n_qt = (Sk + 127) // 128, (Q + 63) // 64
    vis = np.ones((B, Q, Sk), dtype=bool) if vis is None else np.asarray(vis, dtype=bool)
    live = vis.any(-1)
    maps = []
    for b in range(B):
        per_kt = []
        for kt in range(n_kt):
            lst = []
            for t in range(n_qt):
                seen, full = False, True
                for r in range(t * 64, min(Q, t * 64 + 64)):
                    if not live[b, r]:
                        continue
                    for j in range(kt * 128, kt * 128 + 128):
                        e = j < Sk and vis[b, r, j]
                        seen |= e
                        full &= e
                if seen:
                    lst.append(t * 2 + int(not full))
            per_kt.append(lst)
        maps.append(per_kt)
    return maps
