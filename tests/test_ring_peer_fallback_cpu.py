"""The peer-memory ring's fallback to the two-sided NCCL executor, without a GPU. When a group's peer heaps cannot be
mapped (`_peer_transport` returns None), fp32 inputs of the fp16 mode must reach the NCCL executor as bf16 operands
and come back as fp32, in the forward and in the backward, and a folded rotary embedding must not be dropped silently
on that path. The executors are replaced by recorders: only the host-side dispatch of ring_forward / ring_backward runs."""
import pytest
import torch

from lwm_b200 import _lib
from lwm_b200 import ringattention as ra

B, S, H, D, WORLD = 1, 256, 2, 128, 2


@pytest.fixture
def no_peer_heaps(monkeypatch):
    seen = {}

    def fwd(plan, q, k, v, bias, seg, causal, group, ops):
        seen["fwd"] = (q.dtype, k.dtype, v.dtype)
        return torch.zeros(q.shape, dtype=torch.bfloat16), dict(out_chunks=[])

    def bwd(plan, res, k, v, dout, bias, seg, causal, group, ops):
        seen["bwd"] = (k.dtype, v.dtype, dout.dtype)
        z = torch.zeros(k.shape, dtype=torch.bfloat16)
        return z, z.clone(), z.clone()

    monkeypatch.setenv("LWM_RING_TRANSPORT", "peer")
    monkeypatch.setattr(ra, "_peer_transport", lambda group, device, nbytes_hint=0: None)
    monkeypatch.setattr(ra, "_transport", lambda group=None: "nccl" if seen.get("broken") else "peer")
    monkeypatch.setattr(ra.rx, "run_forward", fwd)
    monkeypatch.setattr(ra.rx, "run_backward", bwd)
    return seen


def test_fp32_forward_falls_back_to_the_nccl_executor_with_bf16_operands(no_peer_heaps):
    q, k, v = [torch.zeros(B, S, H, D) for _ in range(3)]
    out, _ = ra.ring_forward(q, k, v, None, None, True, None, 0, WORLD, "contiguous", "fp16")
    assert no_peer_heaps["fwd"] == (torch.bfloat16,) * 3
    assert out.dtype == torch.float32 and out.shape == q.shape


def test_fp32_backward_after_the_fallback_gives_fp32_gradients(no_peer_heaps):
    no_peer_heaps["broken"] = True          # ring_backward follows the transport the forward switched the group to
    k, v, do = [torch.zeros(B, S, H, D) for _ in range(3)]
    dq, dk, dv = ra.ring_backward({}, k, v, do, None, None, True, None, 0, WORLD, "contiguous", "fp16")
    assert no_peer_heaps["bwd"] == (torch.bfloat16,) * 3
    assert dq.dtype == dk.dtype == dv.dtype == torch.float32


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_a_folded_rotation_is_refused_on_the_nccl_executor(no_peer_heaps, dtype):
    q, k, v = [torch.zeros(B, S, H, D, dtype=dtype) for _ in range(3)]
    rope = (torch.zeros(B, S, dtype=torch.int32), torch.zeros(64))
    with pytest.raises(_lib.LwmError, match="rotary embedding"):
        ra.ring_forward(q, k, v, None, None, True, None, 0, WORLD, "contiguous", "fp16", rope)
    assert "fwd" not in no_peer_heaps
