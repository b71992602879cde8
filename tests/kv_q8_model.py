"""Torch restatement of the 8-bit KV-cache format (lwm_b200/csrc/kv_q8.cuh, DESIGN.md §5) and a float64 model of the
output error it causes. The CPU tests check the format against its definition with it, and the GPU tests compare the
kernels' bytes and errors against it. Runs on any device.

  e     = floor(log2(m)) - 6 for the group's largest finite |x| = m, clamped to [-126, 121]; 0 when m = 0
  code  = clamp(round_half_even(x / 2^e), -127, 127); -128 for NaN and +-inf
  value = code * 2^e (NaN for -128)"""
import math

import torch

GROUP = 32
EXP_MIN, EXP_MAX = -126, 121
NAN_CODE = -128


def _pow2(e):
    """2^e (float64) for an integer tensor e in [-126, 126], exact on every device (torch.pow is not on CUDA)"""
    table = torch.tensor([2.0 ** i for i in range(-126, 127)], dtype=torch.float64, device=e.device)
    return table[e.long() + 126]


def quantize_rows(x):
    """x [..., 128] (any float dtype) -> (codes int8 [..., 128], exps int8 [..., 4]) in row order"""
    xd = x.double().reshape(x.shape[:-1] + (4, GROUP))
    finite = torch.isfinite(xd)
    m = torch.where(finite, xd.abs(), torch.zeros_like(xd)).amax(-1)
    _, ex = torch.frexp(m)                                  # m = mant * 2^ex, mant in [0.5, 1): floor(log2 m) = ex - 1
    e = (ex.long() - 1 - 6).clamp(EXP_MIN, EXP_MAX)
    e = torch.where(m == 0, torch.zeros_like(e), e)
    scaled = xd * _pow2(-e)[..., None]                      # exact in float64
    codes = torch.round(torch.where(finite, scaled, torch.zeros_like(scaled))).clamp(-127, 127)   # half to even
    codes = torch.where(finite, codes, torch.full_like(codes, NAN_CODE))
    return codes.to(torch.int8).reshape(x.shape), e.to(torch.int8)


def dequantize_rows(codes, exps, dtype=torch.float64):
    """inverse of quantize_rows: code * 2^e, NaN for the NaN code"""
    c = codes.double().reshape(codes.shape[:-1] + (4, GROUP))
    val = c * _pow2(exps)[..., None]
    val = torch.where(c == NAN_CODE, torch.full_like(val, math.nan), val)
    return val.reshape(codes.shape).to(dtype)


def to_cache_layout(codes, exps):
    """row-order (codes [B,L,H,128], exps [B,L,H,4]) -> the cache's (data [B,L,H,128], exp [B,H,L,4])"""
    return codes.contiguous(), exps.permute(0, 2, 1, 3).contiguous()


def from_cache(data, exp):
    """the cache's (data [B,L,H,128], exp [B,H,L,4]) -> float64 values [B,L,H,128]"""
    return dequantize_rows(data, exp.permute(0, 2, 1, 3))


def attention_f64(q, k, v, mask=None, chunk=1 << 17):
    """softmax(where(mask, q.k / sqrt(D), finfo.min)) v in float64: q [B,Q,H,D], k/v [B,K,H,D], mask [Bm,1,Q,K] or
    None -> [B,Q,H,D]. Chunked over keys."""
    B, Q, H, D = q.shape
    K = k.shape[1]
    qd = q.double()
    s = torch.empty(B, H, Q, K, dtype=torch.float64, device=q.device)
    for j in range(0, K, chunk):
        s[..., j:j + chunk] = torch.einsum("bqhd,bkhd->bhqk", qd, k[:, j:j + chunk].double())
    s /= math.sqrt(D)
    if mask is not None:
        s.masked_fill_(mask.to(s.device) == 0, -3.3895313892515355e38)
    p = torch.softmax(s, -1)
    out = torch.zeros(B, Q, H, D, dtype=torch.float64, device=q.device)
    for j in range(0, K, chunk):
        out += torch.einsum("bhqk,bkhd->bqhd", p[..., j:j + chunk], v[:, j:j + chunk].double())
    return out


def row_error(out, ref):
    """the largest relative Frobenius error over the [.., D] rows"""
    o, r = out.double().reshape(-1, out.shape[-1]), ref.double().reshape(-1, ref.shape[-1])
    return ((o - r).norm(dim=-1) / r.norm(dim=-1).clamp_min(1e-300)).max().item()


def predicted_error(q, k, v, mask=None):
    """the format's own contribution: the error of float64 attention on the quantized k / v against float64 attention
    on k / v as given -> (error, float64 reference on the un-quantized cache)"""
    ref = attention_f64(q, k, v, mask)
    kq, vq = (dequantize_rows(*quantize_rows(t)) for t in (k, v))
    return row_error(attention_f64(q, kq, vq, mask), ref), ref
