"""GPU parity of the backward tile kernel for the shapes its pipeline depends on: per-CTA Q-tile counts that
are odd or one (the Q/dO, dS^T and dQ staging buffers are double-buffered), a long loop over a single key tile
(the stages wrap around many times), B > 1 with an odd head count (coordinates of the fp32 dQ reduction), and
a non-zero dq_acc on entry (the reduction adds to it). Each case runs in both precision modes against the
float64 closed-form gradients of oracle/attn_dense.py; tolerances as in test_attn_bwd_gpu.py (bf16) and
test_attn_fp16_mode_gpu.py (fp16)."""
import numpy as np
import pytest
import torch

from helpers import make_qkv, rel_fro, to_np

pytestmark = pytest.mark.gpu
TOL = {"bf16": 3e-3, "fp16": 1e-3}


def _run(mode, q, k, v, do, causal, q_pos0=0, k_pos0=0, dq_init=None):
    from lwm_b200 import ringattention as ra
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    out = torch.empty_like(q)
    lse = torch.empty(B, H, Sq, dtype=torch.float32, device="cuda")
    delta = torch.empty_like(lse)
    dq = torch.zeros(B, Sq, H, D, dtype=torch.float32, device="cuda") if dq_init is None else dq_init.clone()
    dk = torch.zeros(B, Sk, H, D, dtype=torch.float32, device="cuda")
    dv = torch.zeros_like(dk)
    if mode == "bf16":
        ra.fwd_step(q, k, v, out, lse, None, None, None, q_pos0, k_pos0, causal, None, None, True, True)
        ra.bwd_prep(out, do, delta)
        ra.bwd_step(q, k, v, do, ra.lse_for_bwd(lse), delta, dq, dk, dv, q_pos0, k_pos0, causal, None, None)
    else:
        (q16, sq), (k16, sk), (v16, sv), (d16, sd) = [ra.to_f16(t) for t in (q, k, v, do)]
        out32 = torch.empty(B, Sq, H, D, dtype=torch.float32, device="cuda")
        ra.fwd_step(q16, k16, v16, out, lse, None, None, None, q_pos0, k_pos0, causal, None, None, True, True,
                    scales=(sq, sk, sv), out_f32=out32)
        ra.bwd_prep(out32, do, delta)
        ra.bwd_step(q16, k16, v16, d16, ra.lse_for_bwd(lse, f16=True), delta, dq, dk, dv, q_pos0, k_pos0, causal,
                    None, None, scales=(sq, sk, sv, sd))
    torch.cuda.synchronize()
    return to_np(dq), to_np(dk), to_np(dv)


def _check(mode, got, q, k, v, do, **kw):
    from oracle.attn_dense import attention_dense_grads
    ref = attention_dense_grads(to_np(q), to_np(k), to_np(v), to_np(do), **kw)
    for name, g, r in zip(("dq", "dk", "dv"), got, ref):
        assert np.isfinite(g).all(), name
        assert rel_fro(g, r) < TOL[mode], (name, rel_fro(g, r))


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
def test_odd_and_single_q_tile_counts(mode):
    # q_pos0 = 64: the three key tiles see 4, 3 and 1 Q tiles of 64 rows
    q, k, v, do = make_qkv(1, 256, 384, 2, n_extra=1, seed=101)
    got = _run(mode, q, k, v, do, True, q_pos0=64, k_pos0=0)
    _check(mode, got, q, k, v, do, causal=True, q_pos0=64, k_pos0=0)


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
def test_long_loop_over_one_key_tile(mode):
    # 128 Q tiles stream past one key tile: every double-buffered stage is reused 64 times
    q, k, v, do = make_qkv(1, 8192, 128, 1, n_extra=1, seed=102)
    got = _run(mode, q, k, v, do, False)
    _check(mode, got, q, k, v, do, causal=False)


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
def test_batch2_heads3(mode):
    q, k, v, do = make_qkv(2, 512, 512, 3, n_extra=1, seed=103)
    got = _run(mode, q, k, v, do, True)
    _check(mode, got, q, k, v, do, causal=True)


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
def test_dq_accumulates_onto_prior_value(mode):
    q, k, v, do = make_qkv(1, 512, 512, 2, n_extra=1, seed=104)
    g = torch.Generator(device="cpu").manual_seed(105)
    prior = torch.randn(1, 512, 2, 128, generator=g).cuda()
    dq, dk, dv = _run(mode, q, k, v, do, True, dq_init=prior)
    _check(mode, (dq - to_np(prior), dk, dv), q, k, v, do, causal=True)
