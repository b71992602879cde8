"""GPU parity of the decode-time op `ringattention_inference` (lwm/llama.py:601-614) against the dense float64
oracle: q_len 1 (generation) and a short multi-row query, causal-style boolean masks incl. a left-padded
prompt, and the shard/merge path (two 'ranks' emulated on one GPU through the C ABI).
Tolerance: bf16 output (8 significant bits): relative Frobenius error <= 3e-3."""
import numpy as np
import pytest
import torch

from helpers import rel_fro, to_np

pytestmark = pytest.mark.gpu


def _mk(B, Q, K, H, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Q, H, 128, generator=g).to(torch.bfloat16).cuda()
    k = torch.randn(B, K, H, 128, generator=g).to(torch.bfloat16).cuda()
    v = torch.randn(B, K, H, 128, generator=g).to(torch.bfloat16).cuda()
    return q, k, v


@pytest.mark.parametrize("B,Q,K,H", [(1, 1, 4096, 4), (2, 1, 1000, 3), (1, 4, 2048, 2)])
def test_decode_matches_oracle(B, Q, K, H):
    from lwm_b200.ringattention import ringattention_inference
    from oracle.attn_dense import attention_inference_dense
    q, k, v = _mk(B, Q, K, H, 5)
    # decode-style mask: query row i (at cache position K-Q+i) sees keys <= its position, minus a padded prefix
    pos = torch.arange(K)[None, :] <= (K - Q + torch.arange(Q))[:, None]
    mask = pos[None, None].expand(B, 1, Q, K).clone()
    mask[0, :, :, :17] = False
    out = ringattention_inference(q, k, v, mask.cuda(), axis_name="sp")
    torch.cuda.synchronize()
    ref = attention_inference_dense(to_np(q), to_np(k), to_np(v), mask.numpy())
    assert np.isfinite(to_np(out)).all()
    assert rel_fro(to_np(out), ref) < 3e-3


def test_decode_shard_merge_equals_whole():
    """two ranks' partials merged == one rank holding the whole cache (the all-gather path, emulated)"""
    from lwm_b200 import ringattention as ra, _lib
    from oracle.attn_dense import attention_inference_dense
    B, Q, K, H = 1, 1, 4096, 4
    q, k, v = _mk(B, Q, K, H, 9)
    mask = torch.ones(B, 1, Q, K, dtype=torch.uint8)
    mask[..., 100:150] = 0
    mask = mask.cuda()
    half = K // 2
    parts = [ra.decode_partial(q, k[:, r * half:(r + 1) * half].contiguous(), v[:, r * half:(r + 1) * half].contiguous(),
                               mask, r * half) for r in range(2)]
    o = torch.stack([p[0] for p in parts], 1).contiguous()      # [row][rank][D]
    ml = torch.stack([p[1] for p in parts], 1).contiguous()
    out = torch.empty(B, Q, H, 128, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(B * Q * H, dtype=torch.float32, device="cuda")
    _lib.call("lwm_attn_decode_merge", _lib.ptr(o), _lib.ptr(ml), 2, _lib.ptr(out), 1, _lib.ptr(lse), B * Q * H,
              _lib.stream_ptr())
    torch.cuda.synchronize()
    ref = attention_inference_dense(to_np(q), to_np(k), to_np(v), mask.bool().cpu().numpy())
    assert rel_fro(to_np(out), ref) < 3e-3


def test_decode_fully_masked_row_is_finite():
    from lwm_b200.ringattention import ringattention_inference
    q, k, v = _mk(1, 1, 512, 2, 3)
    mask = torch.zeros(1, 1, 1, 512, dtype=torch.bool).cuda()
    out = ringattention_inference(q, k, v, mask)
    torch.cuda.synchronize()
    o = to_np(out)
    assert np.isfinite(o).all()
    # finfo.min on every key => uniform average of the values (reference semantics)
    assert rel_fro(o, to_np(v).mean(axis=1, keepdims=True)) < 5e-3
