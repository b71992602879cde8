"""Reachable sets and checks of the non-finite input tests (tests/test_nonfinite_gpu.py explains the method), shared by
the one-GPU op, the peer-memory ring (tests/test_nonfinite_gpu.py) and the two-sided NCCL ring
(tests/test_ring_nccl_emulated_gpu.py)."""
import numpy as np
import torch

from helpers import rel_fro

BADS = {"nan": float("nan"), "+inf": float("inf"), "-inf": float("-inf")}
TOL = {"fp16": 3e-3, "bf16": 5e-3}       # dirty results vs the float64 oracle where both are finite
DTYPES = {"bf16": torch.bfloat16, "fp32": torch.float32}
D = 128
BAD_B, BAD_H, BAD_COL = 1, 1, 5          # batch entry, head and column of the bad element


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _dq_close(clean, dirty, bf16):
    """dQ of two runs: the order of its fp32 atomics only, i.e. within 1e-5 of max|dQ|, plus one bf16 unit in the last
    place of the element (at most 2^-7 of it) when the result is bf16: the fp32 sum may land on the other side of a
    rounding boundary"""
    lim = 1e-5 * np.abs(clean).max(initial=0.0) + (2.0 ** -7 * np.abs(clean) if bf16 else 0.0)
    return np.isfinite(dirty).all() and bool(np.all(np.abs(dirty - clean) <= lim))


def _check(name, clean, dirty, ref, same, tol, same_tol=False, bf16=False, strict=True):
    """clean / dirty: kernel results of one (b, h) slice; ref: the oracle on the dirty input; same: entries the bad
    element cannot reach (bit-identical, or as _dq_close with same_tol). Everything else is in reach: within tol of ref
    where both are finite, and (strict) non-finite wherever ref is. strict is off for the gradients of a bad q, k or v:
    a row whose forward met a NaN or +inf logit has lse = -inf, and the backward then gives it P = 0 at its finite
    logits (like a row that sees no key), where the oracle's P is NaN. -> the error where both are finite (0 if nowhere)"""
    same = np.broadcast_to(same, dirty.shape)
    if same_tol:
        assert _dq_close(clean[same], dirty[same], bf16), name
    else:
        n = int((_bits(clean)[same] != _bits(dirty)[same]).sum())
        assert n == 0, "%s: %d entries out of the bad element's reach changed" % (name, n)
    reach = ~same
    swallowed = reach & ~np.isfinite(ref) & np.isfinite(dirty)
    assert not (strict and swallowed.any()), "%s: %d non-finite oracle entries came out finite" % (
        name, int(swallowed.sum()))
    both = reach & np.isfinite(ref) & np.isfinite(dirty)
    err = 0.0
    if both.any():
        err = rel_fro(dirty[both], ref[both])
        assert err < tol, (name, err)
    return err


def _check_other_slices(name, clean, dirty, b, h, tol_dq=False, bf16=False):
    """[B,S,H,D] arrays: every (b', h') != (b, h) slice is bit-identical (dQ: _dq_close over the slice)"""
    for bb in range(clean.shape[0]):
        for hh in range(clean.shape[2]):
            if (bb, hh) == (b, h):
                continue
            c, d = clean[bb, :, hh], dirty[bb, :, hh]
            if tol_dq:
                assert _dq_close(c, d, bf16), (name, bb, hh)
            else:
                assert np.array_equal(_bits(c), _bits(d)), "%s: slice (b=%d, h=%d) changed" % (name, bb, hh)


def _rows_reaching(j, qt, n):
    """[n] bool: rows whose (qt-row) Q tile visits the K tile of key j under the causal rule"""
    r = np.arange(n)
    return (r // qt) * qt + qt - 1 >= (j // 128) * 128


def _keys_reached(i, qt, n):
    """[n] bool: keys in the K tiles that row i's (qt-row) Q tile visits under the causal rule"""
    kk = np.arange(n)
    return (kk // 128) * 128 <= (i // qt) * qt + qt - 1


def _same_sets(which, i, d, vis, n_q, n_k):
    """per result (out, lse, dq, dk, dv): bool arrays [rows, D] (lse: [rows]) of the entries the bad element at row
    i (column d) of `which` cannot reach; None = not compared (the result does not read the input)"""
    rows_q, cols = np.ones(n_q, bool), np.ones(D, bool)
    col_d = np.zeros(D, bool)
    col_d[d] = True
    if which == "q":
        other = np.arange(n_q) != i
        keys = ~_keys_reached(i, 64, n_k)
        return dict(out=other[:, None] & cols, lse=other, dq=other[:, None] & cols, dk=keys[:, None] & cols,
                    dv=keys[:, None] & cols)
    if which == "k":
        blind = ~vis[:, i]
        far = ~_rows_reaching(i, 64, n_q)
        return dict(out=blind[:, None] & cols, lse=blind, dq=far[:, None] & cols, dk=np.zeros((n_k, D), bool),
                    dv=np.zeros((n_k, D), bool))
    if which == "v":
        far_fwd = ~_rows_reaching(i, 128, n_q)
        far = ~_rows_reaching(i, 64, n_q)
        return dict(out=~col_d[None, :] | far_fwd[:, None], lse=rows_q, dq=far[:, None] & cols,
                    dk=np.zeros((n_k, D), bool), dv=np.ones((n_k, D), bool))
    assert which == "do"
    other = np.arange(n_q) != i
    keys = ~_keys_reached(i, 64, n_k)
    return dict(out=None, lse=None, dq=other[:, None] & cols, dk=keys[:, None] & cols,
                dv=keys[:, None] | ~col_d[None, :])


# ------------------------------------------------------------------------------------------------ ring inputs
B_RING, H_RING, SL_RING = 2, 2, 512


def _ring_inputs(world, dtype):
    g = torch.Generator().manual_seed(100 + world)
    S = world * SL_RING
    q, k, v, do = [torch.randn(B_RING, S, H_RING, D, generator=g) for _ in range(4)]
    row = SL_RING + 77                                      # on rank 1
    for t in (q, k, v, do):
        t[BAD_B, row, BAD_H, BAD_COL] = 0
    return [t.to(DTYPES[dtype]) for t in (q, k, v, do)], row
