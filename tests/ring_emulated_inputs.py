"""Inputs of the ring executors run with the real kernels on one GPU, their ranks as threads
(tests/test_ring_peer_emulated_gpu.py, tests/test_ring_nccl_emulated_gpu.py): every rank's shard of q, k, v and dO
carries a power-of-two magnitude of its own, so every owner (peer executor) and every chunk (NCCL executor) gets its
own fp16 operand scale. Values are bf16-representable.

Tolerances (those of tests/ring_multi_gpu_worker.py): 1e-3 for fp32 results of the default mode, 3e-3 for bf16
results (their own rounding), 5e-3 in the legacy bf16 operand mode. Padded query rows are excluded from out / dq."""
import torch

TOL_F32_READOUT, TOL_BF16_RESULT, TOL_BF16_MODE = 1e-3, 3e-3, 5e-3
B, H, D, NPAD = 2, 2, 128, 37


def _inputs(world, Sl, seed, masks):
    """global q, k, v, dO (float32 holding bf16 values) with per-rank magnitudes, and the masks"""
    from oracle.attn_dense import finfo_min
    S = world * Sl
    g = torch.Generator().manual_seed(seed)
    q, k, v, do = [torch.randn(B, S, H, D, generator=g) for _ in range(4)]
    for r in range(world):
        sl = slice(r * Sl, (r + 1) * Sl)
        q[:, sl] *= 2.0 ** -r * 1.3
        k[:, sl] *= 2.0 ** r * 0.7
        v[:, sl] *= 2.0 ** -r
        do[:, sl] *= 2.0 ** (r - 8)
    q, k, v, do = [t.to(torch.bfloat16).float() for t in (q, k, v, do)]
    bias = seg = None
    if masks:
        bias = torch.zeros(B, S)
        bias[0, :NPAD] = finfo_min("bf16")
        seg = torch.zeros(B, S, dtype=torch.int32)
        seg[B - 1, S // 2 + 5:] = 1
        do[0, :NPAD] = 0
    return q, k, v, do, bias, seg


def _passes(world, Sl):
    """every (precision mode, input dtype) pair, each once without and once with masks: consecutive passes never see
    the same inputs, so a read of a heap region left over from an earlier pass cannot go unnoticed"""
    sets = [_inputs(world, Sl, 500 + world, False), _inputs(world, Sl, 600 + world, True)]
    return [(prec, dt, m, sets[m]) for prec in ("fp16", "bf16") for dt in (torch.float32, torch.bfloat16) for m in (0, 1)]
