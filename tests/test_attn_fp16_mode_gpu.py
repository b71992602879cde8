"""fp16-internal precision mode of the attention kernels (precision='fp16'): every operand is an exact
power-of-two-scaled fp16 copy of the bf16 input and P / dS keep 11 significant bits. This is the mode that
meets the north_star tolerance — relative Frobenius error <= 1e-3 — on white-noise inputs, for the forward
fp32 readout AND for the fp32 gradient accumulators (bf16 mode: 1.3e-3 / 2.2e-3, see the other tests)."""
import numpy as np
import pytest
import torch

from helpers import make_qkv, rel_fro, to_np

pytestmark = pytest.mark.gpu
TOL = 1e-3


def _run(q, k, v, do, causal=True, bias=None, seg=None):
    from lwm_b200 import ringattention as ra
    B, S, H, D = q.shape
    (q16, sq), (k16, sk), (v16, sv), (d16, sd) = [ra.to_f16(t) for t in (q, k, v, do)]
    acc_o = torch.empty(B, S, H, D, dtype=torch.float32, device="cuda")
    acc_m = torch.empty(B, H, S, dtype=torch.float32, device="cuda")
    acc_l = torch.empty(B, H, S, dtype=torch.float32, device="cuda")
    ra.fwd_step(q16, k16, v16, None, None, acc_o, acc_m, acc_l, 0, 0, causal, bias, seg, True, False,
                scales=(sq, sk, sv))
    out = torch.empty_like(q)
    lse = torch.empty(B, H, S, dtype=torch.float32, device="cuda")
    out32 = torch.empty(B, S, H, D, dtype=torch.float32, device="cuda")
    ra.fwd_step(q16, k16, v16, out, lse, None, None, None, 0, 0, causal, bias, seg, True, True, scales=(sq, sk, sv),
                out_f32=out32)
    delta = torch.empty_like(lse)
    ra.bwd_prep(out32, do, delta)      # fp16 mode keeps the un-rounded output as the residual for delta
    dq = torch.zeros(B, S, H, D, dtype=torch.float32, device="cuda")
    dk, dv = torch.zeros_like(dq), torch.zeros_like(dq)
    ra.bwd_step(q16, k16, v16, d16, ra.lse_for_bwd(lse, f16=True), delta, dq, dk, dv, 0, 0, causal, bias, seg, scales=(sq, sk, sv, sd))
    torch.cuda.synchronize()
    o32 = to_np(acc_o) / to_np(acc_l).transpose(0, 2, 1)[..., None]
    return o32, to_np(out), to_np(lse), to_np(dq), to_np(dk), to_np(dv)


def test_to_f16_is_exact_and_scaled():
    from lwm_b200 import ringattention as ra
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(4, 256, 2, 128, generator=g) * 3e-5).to(torch.bfloat16).cuda()   # tiny magnitudes (gradients)
    x16, scale = ra.to_f16(x)
    torch.cuda.synchronize()
    s = float(scale[0])
    assert s > 0 and np.log2(s) == int(np.log2(s))                     # power of two
    back = x16.float() * s
    assert torch.equal(back, x.float())                                # exact round trip
    assert 4096 <= float(x16.float().abs().max()) < 8192               # |max| normalised into [2^12, 2^13)
    z16, zs = ra.to_f16(torch.zeros_like(x))
    assert float(zs[0]) == 1.0 and float(z16.abs().max()) == 0.0


@pytest.mark.parametrize("S,H,causal", [(512, 2, True), (2048, 2, True), (512, 2, False)])
def test_fp16_mode_meets_1e3_on_white_noise(S, H, causal):
    from oracle.attn_dense import attention_dense, attention_dense_grads
    q, k, v, do = make_qkv(1, S, S, H, n_extra=1, seed=41)
    o32, out, lse, dq, dk, dv = _run(q, k, v, do, causal)
    ref, ref_lse = attention_dense(to_np(q), to_np(k), to_np(v), causal=causal, return_lse=True)
    rq, rk, rv = attention_dense_grads(to_np(q), to_np(k), to_np(v), to_np(do), causal=causal)
    assert rel_fro(o32, ref) < TOL
    assert np.abs(lse - ref_lse).max() < 1e-3
    assert rel_fro(dv, rv) < TOL
    assert rel_fro(dq, rq) < TOL
    assert rel_fro(dk, rk) < TOL


def test_fp16_mode_scale_robustness():
    """operands far from unit scale (tiny upstream gradients, large keys, large or small values) must neither overflow
    nor lose bits: the V and dO scales vary independently, so their product ranges over 3e-10 .. 9e4"""
    from oracle.attn_dense import attention_dense_grads
    q0, k0, v0, do0 = make_qkv(1, 512, 512, 2, n_extra=1, seed=43)
    k = (k0.float() * 24.0).to(torch.bfloat16)
    q = (q0.float() / 24.0).to(torch.bfloat16)
    for v_scale in (1.0 / 300.0, 1.0, 300.0):
        for do_scale in (1e-7, 1.0, 300.0):
            v = (v0.float() * v_scale).to(torch.bfloat16)
            do = (do0.float() * do_scale).to(torch.bfloat16)
            o32, out, lse, dq, dk, dv = _run(q, k, v, do)
            rq, rk, rv = attention_dense_grads(to_np(q), to_np(k), to_np(v), to_np(do), causal=True)
            for name, got, ref in (("dq", dq, rq), ("dk", dk, rk), ("dv", dv, rv)):
                assert np.isfinite(got).all(), (v_scale, do_scale, name)
                assert rel_fro(got, ref) < TOL, (v_scale, do_scale, name, rel_fro(got, ref))


def test_fp16_mode_bias_segments_and_public_op():
    from lwm_b200.ringattention import ringattention
    from oracle.attn_dense import attention_dense, attention_dense_grads, finfo_min
    B, S, H = 1, 512, 2
    q, k, v, do = make_qkv(B, S, S, H, n_extra=1, seed=47)
    bias = torch.zeros(B, 1, 1, S)
    bias[..., :33] = finfo_min("bf16")
    seg = torch.zeros(B, S, dtype=torch.int32)
    seg[:, 301:] = 1
    do = do.clone()
    do[:, :33] = 0
    q.requires_grad_(True); k.requires_grad_(True); v.requires_grad_(True)
    out = ringattention(q, k, v, bias.cuda(), seg.cuda(), axis_name="sp", float32_logits=True, cache_idx=None,
                        blockwise_kwargs=dict(causal_block_size=1, deterministic=True, attn_pdrop=0.0,
                                              query_chunk_size=128, key_chunk_size=128), precision="fp16")
    out.backward(do)
    torch.cuda.synchronize()
    kw = dict(causal=True, attn_bias=bias.reshape(B, S).numpy(), segment_ids=seg.numpy())
    ref = attention_dense(to_np(q), to_np(k), to_np(v), **kw)
    rq, rk, rv = attention_dense_grads(to_np(q), to_np(k), to_np(v), to_np(do), **kw)
    assert np.isfinite(to_np(out)).all()
    assert rel_fro(to_np(out)[:, 33:], ref[:, 33:]) < 3e-3          # bf16 output rounding
    assert rel_fro(to_np(q.grad)[:, 33:], rq[:, 33:]) < 3e-3        # bf16 gradient rounding
    assert rel_fro(to_np(k.grad), rk) < 3e-3
    assert rel_fro(to_np(v.grad), rv) < 3e-3
