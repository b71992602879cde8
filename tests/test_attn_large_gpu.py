"""Oracle parity at the benchmark sequence lengths (32K and 128K tokens, LWM-7B head
geometry) on one GPU: the public op in its default precision mode against the float64 row-wise oracle
(oracle/attn_rows.py) on one sampled query row of every 128-row tile plus the last 128 rows (out, dq) and on EVERY key
row (dk, dv) — see lwm_b200/selftest.py::sampled_parity. Tolerance: 1e-3 relative Frobenius (north_star) on the
un-rounded fp32 results, for unit-scale dO and for dO scaled by 2^-20 (the oracle's gradients are linear in dO, so
the same relative bound applies). The multi-GPU counterpart is tests/test_ring_multi_gpu.py (RING_TEST_MODE=sampled)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("S", [32768, 131072])
def test_sampled_oracle_parity_at_baseline_lengths(S):
    _check_sampled_parity(S, 1.0)


def test_sampled_oracle_parity_with_small_upstream_gradient():
    """dO x 2^-20: upstream gradients of the size a loss averaged over ~1M tokens produces, where P ~ 1/S is small
    too — the regime in which a dS rounded to fp16 in absolute units would lose its bits"""
    _check_sampled_parity(32768, 2.0 ** -20)


def _check_sampled_parity(S, do_scale):
    from lwm_b200 import ringattention as ra
    from lwm_b200.selftest import sampled_parity
    kw = dict(axis_name="sp", float32_logits=True, cache_idx=None,
              blockwise_kwargs=dict(causal_block_size=1, deterministic=True, attn_pdrop=0.0, query_chunk_size=1024,
                                    key_chunk_size=1024))
    errs = sampled_parity(S, 2, [1], lambda q, k, v: ra.ringattention(q, k, v, None, None, **kw), torch.device("cuda"),
                          do_scale=do_scale)
    print(S, do_scale, errs)
    assert errs["rows"] >= S // 128
    for name in ("out", "dq", "dk", "dv"):
        assert errs[name] < 1e-3, (name, errs)
    assert errs["dq_unsampled_abs"] == 0.0
