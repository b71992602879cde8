"""The fp8 mode (ringattention(..., precision='fp8')) without a GPU: its float64 error model against the dense oracle,
the argument validation of its C entry points and of the Python layer, and the machine code of its kernel instances."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import e4m3_attn_model as em

P = ctypes.c_void_p(0x1000)      # fake non-null pointer
N = None
SHAPE, ARG, DEVICE = 2, 3, 1


# ---------------------------------------------------------------------------------------------------- error model
def test_model_copies_follow_the_scale_rule():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(4, 256, 2, 128, generator=g) * 3.0
    x8, s = em.e4m3_copy(x)
    m = float(x8.float().abs().max())
    assert 128.0 <= m < 256.0 and s == 2.0 ** (np.frexp(float(x.abs().max()))[1] - 1 - 7)
    # x / s is exact (power of two), and the e4m3 rounding is round-to-nearest: within half an e4m3 ulp (2^-4 relative)
    y = x8.double() * s
    assert float(((y - x.double()).abs() / x.double().abs().clamp_min(2.0 ** -6 * s)).max()) <= 2.0 ** -4
    v16, sv = em.f16_copy(x.to(torch.bfloat16))
    assert torch.equal(v16.double() * sv, x.to(torch.bfloat16).double())     # bf16 values: the fp16 copy is exact


def test_model_scale_of_nonfinite_and_zero_tensors():
    assert em.pow2_scale(torch.zeros(8), 7) == 1.0
    assert em.pow2_scale(torch.tensor([float("inf"), float("nan"), 0.0]), 7) == 1.0
    assert em.pow2_scale(torch.tensor([float("inf"), 3.0]), 7) == 2.0 ** -6
    assert em.pow2_scale(torch.tensor([1e-38]), 7) == 2.0 ** (-114 - 7)      # clamped


@pytest.mark.parametrize("causal", [True, False])
def test_model_against_the_dense_oracle(causal):
    """the model is the dense oracle on rounded operands: close to the unrounded result, not equal to it"""
    from oracle.attn_dense import attention_dense
    g = torch.Generator().manual_seed(1)
    q, k, v = [torch.randn(1, 256, 2, 128, generator=g).to(torch.bfloat16) for _ in range(3)]
    out, lse = em.attention_e4m3_model(q, k, v, causal=causal)
    ref, ref_lse = attention_dense(q.double().numpy(), k.double().numpy(), v.double().numpy(), causal=causal,
                                   return_lse=True)
    e = em.err_vs_max(out, ref)
    assert 1e-4 < e < 5e-2, e
    assert float(np.abs(lse - ref_lse).max()) < 0.1       # nats; the early causal rows see a few keys only
    # with operands that e4m3 holds exactly, the model is the oracle
    qe, ke = [(t.float() * 4).round().clamp(-16, 16) / 4 for t in (q, k)]
    out_e, _ = em.attention_e4m3_model(qe, ke, v, causal=causal)
    ref_e = attention_dense(qe.double().numpy(), ke.double().numpy(), v.double().numpy(), causal=causal)
    assert np.allclose(out_e, ref_e, rtol=0, atol=1e-12)


# ---------------------------------------------------------------------------------------------------- C entry points
def _status(lib, name, *args):
    return getattr(lib, name)(*args), lib.lwm_last_error().decode()


def _fwd(**over):
    """the arguments of lwm_attn_fwd_e4m3_step for a well-formed one-step call, with `over` replaced"""
    names = ["q8", "k8", "v16", "sq", "sk", "sv", "out_f32", "out", "lse", "acc_o", "acc_m", "acc_l", "B", "H", "Sq", "Sk",
             "D", "q_pos0", "k_pos0", "causal", "bias", "bias_stride", "seg", "seg_stride", "softmax_scale", "first",
             "last", "tiles", "tile_count", "stream"]
    a = dict(q8=P, k8=P, v16=P, sq=P, sk=P, sv=P, out_f32=N, out=P, lse=P, acc_o=N, acc_m=N, acc_l=N, B=1, H=2, Sq=128,
             Sk=256, D=128, q_pos0=0, k_pos0=0, causal=1, bias=N, bias_stride=0, seg=N, seg_stride=0,
             softmax_scale=0.1, first=1, last=1, tiles=N, tile_count=N, stream=N)
    a.update(over)
    return tuple(a[n] for n in names)


BAD_CALLS = [
    ("lwm_attn_fwd_e4m3_step", _fwd(sk=N), ARG, "scales are required"),
    ("lwm_attn_fwd_e4m3_step", _fwd(sq=N, sk=N, sv=N), ARG, "scales are required"),
    ("lwm_attn_fwd_e4m3_step", _fwd(D=64), SHAPE, "head_dim must be 128"),
    ("lwm_attn_fwd_e4m3_step", _fwd(Sk=200), SHAPE, "multiples of 128"),
    ("lwm_attn_fwd_e4m3_step", _fwd(q8=N), ARG, "null q/k/v"),
    ("lwm_attn_fwd_e4m3_step", _fwd(lse=N), ARG, "out/lse required"),
    ("lwm_attn_fwd_e4m3_step", _fwd(last=0), ARG, "carry buffers"),
    ("lwm_attn_fwd_e4m3_step", _fwd(tiles=P), ARG, "both given or both null"),
    ("lwm_attn_fwd_e4m3_step", _fwd(tiles=P, tile_count=P), ARG, "needs bias or segment_ids"),
    ("lwm_attn_fwd_e4m3_step", _fwd(q_pos0=1 << 31), SHAPE, "int32"),
    ("lwm_attn_fwd_e4m3_step", _fwd(bias=P, bias_stride=128), SHAPE, "bias_stride"),
    ("lwm_attn_fwd_e4m3_step", _fwd(seg=P, seg_stride=128), SHAPE, "seg_stride"),
    ("lwm_attn_to_e4m3_scaled", (P, 1, P, P, 12, N), ARG, "n % 8"),
    ("lwm_attn_to_e4m3_scaled", (P, 2, P, P, 64, N), ARG, "bad arguments"),
    ("lwm_attn_to_e4m3_scaled", (P, 0, P, N, 64, N), ARG, "bad arguments"),
    ("lwm_attn_e4m3_scale_from_absmax", (P, 0, 1, P, N), ARG, "bad arguments"),
    ("lwm_attn_stage_rope", (P, 1, P, 0, P, P, P, 1, 8, 2, N), ARG, "dst dtype codes"),
    ("lwm_attn_stage_rope", (P, 1, P, 4, P, P, P, 1, 8, 2, N), ARG, "dst dtype codes"),
    ("lwm_attn_stage_rope", (P, 0, P, 3, N, P, P, 1, 8, 2, N), ARG, "needs a scale"),
]


@pytest.mark.parametrize("name,args,code,frag", BAD_CALLS, ids=["%s-%d" % (c[0], i) for i, c in enumerate(BAD_CALLS)])
def test_bad_arguments_are_rejected_with_a_message(lib, name, args, code, frag):
    status, msg = _status(lib, name, *args)
    assert status == code, (status, msg)
    assert frag in msg, msg


GOOD_CALLS = [
    ("lwm_attn_fwd_e4m3_step", _fwd()),
    ("lwm_attn_fwd_e4m3_step", _fwd(out_f32=P, first=0, last=0, acc_o=P, acc_m=P, acc_l=P, k_pos0=128)),
    ("lwm_attn_fwd_e4m3_step", _fwd(bias=P, bias_stride=256, seg=P, seg_stride=256, tiles=P, tile_count=P)),
    ("lwm_attn_to_e4m3_scaled", (P, 0, P, P, 64, N)),
    ("lwm_attn_to_e4m3_scaled", (P, 1, P, P, 64, N)),
    ("lwm_attn_e4m3_scale_from_absmax", (P, 4, 4, P, N)),
    ("lwm_attn_stage_rope", (P, 1, P, 3, P, P, P, 1, 8, 2, N)),
    ("lwm_attn_stage_rope", (P, 0, P, 3, P, P, P, 1, 8, 2, N)),
]


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: only meaningful where the device check fails")
@pytest.mark.parametrize("name,args", GOOD_CALLS, ids=["%s-%d" % (c[0], i) for i, c in enumerate(GOOD_CALLS)])
def test_well_formed_calls_fail_with_device_error_without_gpu(lib, name, args):
    status, msg = _status(lib, name, *args)
    assert status == DEVICE, (status, msg)


# ---------------------------------------------------------------------------------------------------- Python layer
def _qkv(requires_grad=False):
    return [torch.zeros(1, 128, 2, 128, dtype=torch.bfloat16, requires_grad=requires_grad) for _ in range(3)]


def test_fp8_needs_a_forward_without_gradient():
    from lwm_b200 import ringattention as ra
    q, k, v = _qkv(requires_grad=True)
    with pytest.raises(ValueError, match="without gradient"):
        ra.ringattention(q, k, v, precision="fp8")


def test_fp8_has_no_dropout():
    from lwm_b200 import ringattention as ra
    kw = dict(deterministic=False, attn_pdrop=0.1, dropout_rng=1)
    with torch.no_grad(), pytest.raises(ValueError, match="no attention dropout"):
        ra.ringattention(*_qkv(), blockwise_kwargs=kw, precision="fp8")


def test_fp8_is_not_on_the_nccl_executor(monkeypatch):
    from lwm_b200 import ringattention as ra
    monkeypatch.setenv("LWM_RING_TRANSPORT", "nccl")
    monkeypatch.setattr(ra, "_resolve_group", lambda axis_name: (None, 0, 2))
    with torch.no_grad(), pytest.raises(NotImplementedError, match="NCCL"):
        ra.ringattention(*_qkv(), precision="fp8")
    with pytest.raises(NotImplementedError, match="NCCL"):
        ra._ops_for("fp8")


def test_fp8_is_a_keyword_only_mode(monkeypatch):
    from lwm_b200 import ringattention as ra
    with pytest.raises(ValueError):
        ra.set_default_precision("fp8")
    monkeypatch.setattr(ra, "_DEFAULT_PRECISION", "fp8")     # what $LWM_ATTN_PRECISION=fp8 would set
    with torch.no_grad(), pytest.raises(ValueError, match="'bf16' or 'fp16'"):
        ra.ringattention(*_qkv())
    with pytest.raises(ValueError, match="'fp8'"):
        ra.ringattention(*_qkv(), precision="fp4")


def test_fp8_ops_have_no_backward():
    from lwm_b200 import ring_peer as rp
    from lwm_b200.ringattention import PeerOpsE4m3, PeerOpsF16
    for name in ("bwd_prep", "lse_for_bwd", "bwd_step", "reduce_cast", "reduce_cast_rope", "rope_conj"):
        with pytest.raises(NotImplementedError, match="forward-only"):
            getattr(PeerOpsE4m3, name)()
    # q and k in e4m3 inside the 2-byte operand regions; v staged by the fp16 mode's ops
    assert PeerOpsE4m3.op_itemsize == 2 and PeerOpsE4m3.op_dtype == torch.float8_e4m3fn
    assert rp.v_ops(PeerOpsE4m3) is PeerOpsF16 and rp.v_ops(PeerOpsF16) is PeerOpsF16


def test_narrow_operand_offsets_in_the_peer_layout():
    from lwm_b200.ring_peer import Layout
    lay = Layout(2, 256, 256, 4, 128, 2, 2, 2)
    assert lay.kv_row_off("kg", 1, 1, 300) == lay.kv_row_off("kg", 1, 1, 300, 2)
    assert lay.kv_row_off("kg", 1, 1, 300, 1) - lay.base(1) - lay.kg == (1 * 2 * 256 + 300) * 4 * 128


# ---------------------------------------------------------------------------------------------------- machine code
E4M3_INSTANCES = {
    "e4m3": "_ZN3lwm20attn_fwd_e4m3_kernelILb0EEEv14CUtensorMap_stS1_S1_NS_9FwdParamsE",
    "e4m3_map": "_ZN3lwm20attn_fwd_e4m3_kernelILb1EEEv14CUtensorMap_stS1_S1_NS_9FwdParamsE",
}


@pytest.mark.parametrize("instance", sorted(E4M3_INSTANCES))
def test_e4m3_exponentials_run_under_the_pv_gemm(monkeypatch, instance):
    """tests/test_attn_fwd_schedule_cpu.py's check on the fp8 instances, whose S GEMM is the e4m3 QGMMA"""
    import test_attn_fwd_schedule_cpu as sched
    tool = sched._cuobjdump()
    if tool is None or not os.path.exists(sched.LIB):
        pytest.skip("needs cuobjdump and the built liblwm_b200.so")
    r = subprocess.run([tool, "-sass", "-fun", E4M3_INSTANCES[instance], sched.LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    insns = [(int(m.group(1), 16), m.group(2)) for m in map(sched._INSN.search, r.stdout.splitlines()) if m]
    assert any("QGMMA.64x128x32.F32.E4M3.E4M3" in t for _, t in insns), "no e4m3 wgmma in %s" % instance
    monkeypatch.setattr(sched, "_HGMMA_SS", re.compile(r"QGMMA\.\S+\s+R\d+,\s+gdesc"))
    monkeypatch.setitem(sched.INSTANCES, instance, E4M3_INSTANCES[instance])
    sched.test_exponentials_run_under_the_pv_gemm({E4M3_INSTANCES[instance]: insns}, instance)
