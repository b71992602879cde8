"""Float64 CPU model of the fp8 mode's forward (ringattention(..., precision='fp8'), include/lwm_b200.h:
lwm_attn_fwd_e4m3_step): the operands exactly as the kernel sees them, and exact attention over them.

  q, k  x8 = e4m3(x / s), s = 2^(e-7) with e the exponent of the tensor's largest finite |x| (clamped at -114; 1 when
        no element is finite and nonzero), rounded through torch.float8_e4m3fn; the kernel's logits are
        (q8 . k8) * s_q * s_k.
  v     the fp16 mode's copy: fp16(x / s), s = 2^(e-12) (exact for bf16 values, one rounding for fp32 ones).

Everything after that (the softmax, P V) is exact here. What the kernel adds to this model is the fp16 mode's own
error (P packed in fp16, fp32 accumulation), which the GPU tests measure on the same inputs with precision='fp16'.
TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np
import torch

from oracle.attn_dense import attention_dense


def pow2_scale(x, top):
    """2^(e - top), e the exponent of x's largest finite |x| clamped at -114; 1.0 when no element is finite and nonzero"""
    a = x.detach().float().abs().flatten()
    a = a[torch.isfinite(a)]
    m = float(a.max()) if a.numel() else 0.0
    if m == 0.0:
        return 1.0
    e = max(math.frexp(m)[1] - 1, -114)
    return 2.0 ** (e - top)


def e4m3_copy(x, scale=None):
    """-> (x8 float8_e4m3fn, scale): the staged copy of q or k"""
    s = pow2_scale(x, 7) if scale is None else scale
    return (x.detach().float() / s).to(torch.float8_e4m3fn), s


def f16_copy(x):
    """-> (x16 float16, scale): the fp16 mode's copy of v"""
    s = pow2_scale(x, 12)
    return (x.detach().float() / s).to(torch.float16), s


def model_operands(q, k, v):
    """q, k, v (CPU, any float dtype) -> the float64 values the fp8 kernel computes with"""
    (q8, sq), (k8, sk), (v16, sv) = e4m3_copy(q), e4m3_copy(k), f16_copy(v)
    return q8.double() * sq, k8.double() * sk, v16.double() * sv


def attention_e4m3_model(q, k, v, **kw):
    """-> (out [B,Sq,H,D], lse [B,H,Sq]) float64 numpy; kw as oracle.attn_dense.attention_dense's"""
    qm, km, vm = model_operands(q, k, v)
    return attention_dense(qm.numpy(), km.numpy(), vm.numpy(), return_lse=True, **kw)


def err_vs_max(a, ref):
    """max |a - ref| / max |ref|: the error measure of the fp8 mode's tests"""
    a, ref = np.asarray(a, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    return float(np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-300))
