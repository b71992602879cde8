"""Gradients of the default precision mode (fp16 operands, power-of-two scales) at the magnitudes training feeds them.

A loss that is a mean over millions of tokens hands the attention backward an upstream gradient dO of 1e-6 .. 1e-10,
while V stays near unit scale; peaked attention with large V and dO pushes the other way. The fp16 operand copies are
normalised per tensor, so every quantity the kernels round to fp16 must be too: these tests sweep |dO| and |V| over
many octaves against the float64 oracle (oracle/attn_dense.py), and check at the kernel level that a power-of-two
factor on dO or V comes out of the gradients exactly (every scale is a power of two, so nothing else may change).

Tolerance: float32 inputs -> the un-rounded fp32 gradients, relative Frobenius error <= 1e-3 (the bound the default
mode meets at unit scale, tests/test_attn_public_op_gpu.py)."""
import numpy as np
import pytest
import torch

from helpers import make_qkv, rel_fro, to_np

pytestmark = pytest.mark.gpu
TOL = 1e-3
NPAD = 33


def _public_grads(q, k, v, do, causal=True, bias=None, seg=None, precision=None):
    """dq, dk, dv (numpy) of the public op, ring size 1"""
    from lwm_b200.ringattention import ringattention
    q, k, v = [t.detach().clone().requires_grad_(True) for t in (q, k, v)]
    out = ringattention(q, k, v, bias, seg, axis_name="sp", float32_logits=True, cache_idx=None,
                        blockwise_kwargs=dict(causal_block_size=1 if causal else None, deterministic=True,
                                              attn_pdrop=0.0, query_chunk_size=256, key_chunk_size=256),
                        precision=precision)
    out.backward(do)
    torch.cuda.synchronize()
    return to_np(q.grad), to_np(k.grad), to_np(v.grad)


def _check(label, got, q, k, v, do, tol=TOL, skip_q_rows=0, **okw):
    from oracle.attn_dense import attention_dense_grads
    ref = attention_dense_grads(to_np(q), to_np(k), to_np(v), to_np(do), **okw)
    errs = {}
    for name, g, r in zip(("dq", "dk", "dv"), got, ref):
        assert np.isfinite(g).all(), (label, name, "non-finite gradient")
        if name == "dq" and skip_q_rows:
            g, r = g[:, skip_q_rows:], r[:, skip_q_rows:]     # padded query rows are arbitrary in the oracle
        errs[name] = rel_fro(g, r)
    print("%s rel err dq=%.2e dk=%.2e dv=%.2e" % (label, errs["dq"], errs["dk"], errs["dv"]))
    for name, e in errs.items():
        assert e < tol, (label, name, errs)


def _randn(*shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).cuda()


@pytest.mark.parametrize("S", [512, 2048])
@pytest.mark.parametrize("log2_do", [-30, -20, -10, 0, 6])
def test_do_magnitude_sweep(S, log2_do):
    """dO = 2^k N(0,1) with q, k, v ~ N(0,1): the gradients are linear in dO, their relative error must not move"""
    H = 2
    q, k, v = [_randn(1, S, H, 128, seed=S + i) for i in range(3)]
    do = _randn(1, S, H, 128, seed=S + 3) * 2.0 ** log2_do
    _check("S=%d dO=2^%d" % (S, log2_do), _public_grads(q, k, v, do), q, k, v, do, causal=True)


@pytest.mark.parametrize("causal", [True, False])
def test_small_do_with_padding_bias_and_segments(causal):
    from oracle.attn_dense import finfo_min
    B, S, H = 1, 512, 2
    q, k, v = [_randn(B, S, H, 128, seed=70 + i) for i in range(3)]
    do = _randn(B, S, H, 128, seed=73) * 2.0 ** -20
    do[:, :NPAD] = 0
    bias = torch.zeros(B, 1, 1, S)
    bias[..., :NPAD] = finfo_min("bf16")
    seg = torch.zeros(B, S, dtype=torch.int32)
    seg[:, 301:] = 1
    got = _public_grads(q, k, v, do, causal, bias.cuda(), seg.cuda())
    _check("causal=%s masks dO=2^-20" % causal, got, q, k, v, do, skip_q_rows=NPAD, causal=causal,
           attn_bias=bias.reshape(B, S).numpy(), segment_ids=seg.numpy())


@pytest.mark.parametrize("log2_v", [-12, 0, 8])
def test_v_magnitude_sweep(log2_v):
    S, H = 2048, 2
    q, k = [_randn(1, S, H, 128, seed=80 + i) for i in range(2)]
    v = _randn(1, S, H, 128, seed=82) * 2.0 ** log2_v
    do = _randn(1, S, H, 128, seed=83)
    _check("V=2^%d" % log2_v, _public_grads(q, k, v, do), q, k, v, do, causal=True)


def test_peaked_attention_with_large_v_and_do():
    """q x 4 makes most rows nearly one-hot; V and dO x 2^6 make dP ~ 5e4: the magnitudes at which a dS rounded to fp16
    in absolute units overflows"""
    S, H = 2048, 2
    q = _randn(1, S, H, 128, seed=90) * 4.0
    k = _randn(1, S, H, 128, seed=91)
    v = _randn(1, S, H, 128, seed=92) * 64.0
    do = _randn(1, S, H, 128, seed=93) * 64.0
    _check("peaked, V and dO x 2^6", _public_grads(q, k, v, do), q, k, v, do, causal=True)


@pytest.mark.parametrize("log2_do", [-30, 6])
def test_bf16_mode_small_and_large_do(log2_do):
    """the bf16 operand mode keeps fp32's exponent range everywhere: it must stay within its own bound (5e-3)"""
    S, H = 512, 2
    q, k, v, do = [t.float() for t in make_qkv(1, S, S, H, n_extra=1, seed=95)]
    do = do * 2.0 ** log2_do
    _check("bf16 mode dO=2^%d" % log2_do, _public_grads(q, k, v, do, precision="bf16"), q, k, v, do, tol=5e-3,
           causal=True)


def _kernel_grads(q, k, v, do, causal=True):
    """dq, dk, dv (device fp32) of one forward + backward step of the fp16-operand kernels on bf16 inputs"""
    from lwm_b200 import ringattention as ra
    B, S, H, D = q.shape
    (q16, sq), (k16, sk), (v16, sv), (d16, sd) = [ra.to_f16(t) for t in (q, k, v, do)]
    out = torch.empty_like(q)
    lse = torch.empty(B, H, S, dtype=torch.float32, device="cuda")
    out32 = torch.empty(B, S, H, D, dtype=torch.float32, device="cuda")
    ra.fwd_step(q16, k16, v16, out, lse, None, None, None, 0, 0, causal, None, None, True, True, scales=(sq, sk, sv),
                out_f32=out32)
    delta = torch.empty_like(lse)
    ra.bwd_prep(out32, do, delta)
    dq = torch.zeros(B, S, H, D, dtype=torch.float32, device="cuda")
    dk, dv = torch.zeros_like(dq), torch.zeros_like(dq)
    ra.bwd_step(q16, k16, v16, d16, ra.lse_for_bwd(lse, f16=True), delta, dq, dk, dv, 0, 0, causal, None, None,
                scales=(sq, sk, sv, sd))
    torch.cuda.synchronize()
    return dq, dk, dv


@pytest.mark.parametrize("which", ["do", "v"])
@pytest.mark.parametrize("log2_f", [-20, 20])
def test_power_of_two_equivariance(which, log2_f):
    """dO -> 2^k dO must give exactly 2^k dk and 2^k dv; V -> 2^k V exactly 2^k dq and 2^k dk and the same dv. dq is
    summed with atomics in no fixed order, so it is compared to 1e-6 instead of bit for bit."""
    q, k, v, do = make_qkv(1, 512, 512, 2, n_extra=1, seed=61)
    f = 2.0 ** log2_f
    base = _kernel_grads(q, k, v, do)
    if which == "do":
        got = _kernel_grads(q, k, v, (do.float() * f).to(torch.bfloat16))
        want_f = dict(dq=f, dk=f, dv=f)
    else:
        got = _kernel_grads(q, k, (v.float() * f).to(torch.bfloat16), do)
        want_f = dict(dq=f, dk=f, dv=1.0)
    for name, g, b in zip(("dq", "dk", "dv"), got, base):
        want = b * want_f[name]
        assert torch.isfinite(g).all(), name
        if name == "dq":
            assert rel_fro(to_np(g), to_np(want)) < 1e-6, name
        else:
            assert torch.equal(g, want), (name, float((g - want).abs().max()), float(want.abs().max()))
