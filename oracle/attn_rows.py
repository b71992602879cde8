"""Float64 oracle for SAMPLED query rows of a long causal sequence — the row-wise restatement of oracle/attn_dense.py
(same semantics: lwm/llama.py:525-570 call-site contract, SURVEY.md Appendix A), usable at 32K .. 128K tokens
(S = 32768 .. 131072) where the dense S x S oracle does not fit: a query row only needs its own logits row.

With a dO that is zero outside the sampled rows the gradients are exact too and cheap:
    dq_i = sum_j dS_ij k_j / sqrt(D)                      (i sampled; rows with dO_i = 0 have dq_i = 0 exactly)
    dk_j = sum_{i sampled} dS_ij q_i / sqrt(D),  dv_j = sum_{i sampled} P_ij dO_i       (ALL keys j)
so a GPU run with that dO is checked on every key row and on one query row of every 128-row tile.
TEST INFRASTRUCTURE ONLY (see oracle/__init__.py)."""
import math

import torch


def sample_rows(S, per_tile=1, tile=128, tail=128, seed=0):
    """one random row in every `tile`-row block plus the last `tail` rows (sorted, unique) — every tile of the
    kernels' grids contributes at least one checked row"""
    g = torch.Generator().manual_seed(seed)
    n_tiles = S // tile
    rows = (torch.arange(n_tiles).repeat_interleave(per_tile) * tile +
            torch.randint(0, tile, (n_tiles * per_tile,), generator=g))
    rows = torch.cat([rows, torch.arange(max(0, S - tail), S)])
    return torch.unique(rows)


def attention_rows(q_rows, row_pos, k, v, do_rows=None, causal=True, chunk=256, k_pos0=0):
    """q_rows [R,D], row_pos [R] (global positions), k/v [S,D] of ONE (batch, head), any float dtype.
    -> dict(out [R,D], lse [R]) and, with do_rows [R,D], also dq [R,D], dk [S,D], dv [S,D]. float64 throughout."""
    q = torch.as_tensor(q_rows, dtype=torch.float64)
    k = torch.as_tensor(k, dtype=torch.float64)
    v = torch.as_tensor(v, dtype=torch.float64)
    pos = torch.as_tensor(row_pos, dtype=torch.long)
    R, D = q.shape
    S = k.shape[0]
    scale = 1.0 / math.sqrt(D)
    out = torch.empty(R, D, dtype=torch.float64)
    lse = torch.empty(R, dtype=torch.float64)
    grads = do_rows is not None
    if grads:
        g = torch.as_tensor(do_rows, dtype=torch.float64)
        dq = torch.empty(R, D, dtype=torch.float64)
        dk = torch.zeros(S, D, dtype=torch.float64)
        dv = torch.zeros(S, D, dtype=torch.float64)
    kpos = k_pos0 + torch.arange(S)
    for a in range(0, R, chunk):
        b = min(R, a + chunk)
        s = (q[a:b] @ k.T) * scale
        if causal:
            s = s.masked_fill(pos[a:b, None] < kpos[None, :], float("-inf"))
        m = s.max(dim=1, keepdim=True).values
        p = torch.exp(s - m)
        den = p.sum(dim=1, keepdim=True)
        p = p / den
        out[a:b] = p @ v
        lse[a:b] = (m + torch.log(den))[:, 0]
        if grads:
            dp = g[a:b] @ v.T
            delta = (g[a:b] * out[a:b]).sum(dim=1, keepdim=True)
            ds = p * (dp - delta)
            dq[a:b] = (ds @ k) * scale
            dk += (ds.T @ q[a:b]) * scale
            dv += p.T @ g[a:b]
    res = dict(out=out, lse=lse)
    if grads:
        res.update(dq=dq, dk=dk, dv=dv)
    return res
