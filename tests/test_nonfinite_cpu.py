"""oracle.attn_dense.attention_visible, the float64 oracle of tests/test_nonfinite_gpu.py: on finite inputs it equals
the dense oracles it stands in for, and a NaN or inf operand reaches only the pairs that see it."""
import numpy as np
import pytest

from oracle.attn_dense import (attention_dense, attention_dense_grads, attention_inference_dense, attention_visible,
                               finfo_min, visible_pairs)

B, S, H, D = 2, 96, 2, 128


def _inputs(seed):
    rng = np.random.default_rng(seed)
    q, k, v, do = (rng.standard_normal((B, S, H, D)) for _ in range(4))
    bias = np.zeros((B, S))
    bias[0, :11] = finfo_min("bf16")             # left padding: rows 0..10 of batch 0 see no key
    seg = np.zeros((B, S), dtype=np.int32)
    seg[1, 40:] = 1
    return q, k, v, do, dict(causal=True, attn_bias=bias, segment_ids=seg)


def _close(got, ref):
    assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()


def test_matches_attention_dense_on_finite_inputs():
    q, k, v, do, kw = _inputs(0)
    vis = visible_pairs(B, S, S, **kw)
    out, lse, dq, dk, dv = attention_visible(q, k, v, vis, do)
    ref, ref_lse = attention_dense(q, k, v, return_lse=True, **kw)
    _close(out, ref)
    _close(lse, ref_lse)
    for got, r in zip((dq, dk, dv), attention_dense_grads(q, k, v, do, **kw)):
        _close(got, r)


def test_matches_attention_inference_dense_on_finite_inputs():
    rng = np.random.default_rng(1)
    q = rng.standard_normal((B, 5, H, D))
    k, v = rng.standard_normal((B, 70, H, D)), rng.standard_normal((B, 70, H, D))
    mask = rng.random((B, 1, 5, 70)) < 0.6
    mask[0, 0, 2] = False                         # a row with no visible key
    _close(attention_visible(q, k, v, mask)[0], attention_inference_dense(q, k, v, mask))


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_a_bad_value_reaches_only_the_pairs_that_see_it(bad):
    q, k, v, do, kw = _inputs(2)
    vis = visible_pairs(B, S, S, **kw)
    j, d = 60, 7
    v2, k2 = v.copy(), k.copy()
    v2[1, j, 1, d] = bad
    out, _, dq, dk, dv = attention_visible(q, k, v2, vis, do)
    sees = vis[1, 0, :, j]
    assert not np.isfinite(out[1, sees, 1, d]).any()
    assert np.isfinite(out[1, ~sees, 1]).all() and np.isfinite(np.delete(out[1, :, 1], d, axis=-1)).all()
    assert np.isfinite(out[0]).all() and np.isfinite(out[:, :, 0]).all()
    # the same value in k: rows that get a -inf logit drop key j, as if it were masked for them
    k2[1, j, 1, d] = bad
    out, lse = attention_visible(q, k2, v, vis)
    logit = q[1, :, 1, d] * bad
    drop = sees & (logit == -np.inf)
    vis_drop = vis.copy()
    vis_drop[1, 0, drop, j] = False
    ref, ref_lse = attention_visible(q, k, v, vis_drop)
    assert drop.any() == bool(np.isinf(bad))
    if drop.any():
        _close(out[1, drop, 1], ref[1, drop, 1])
        _close(lse[1, 1, drop], ref_lse[1, 1, drop])
    assert not np.isfinite(out[1, sees & ~drop, 1]).any()
    assert np.isfinite(out[1, ~sees, 1]).all()
