"""The ordered dQ reduction without a GPU: argument validation of lwm_attn_bwd_step_ordered and
lwm_attn_infer_bwd_ordered (bad calls are rejected with a message before the device check, well-formed ones fail with
LWM_ERR_DEVICE), and the machine code of the five ordered attn_bwd_kernel instances: no local memory (warp 9's wait,
turn load and ticket fit the 24 registers it keeps after setmaxnreg.dec, and the consumers still fit theirs), a
backed-off wait in every ordered instance and in none of the others.
Pointers are fake non-null addresses: nothing dereferences them before the device check."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

from test_attn_fwd_schedule_cpu import _cuobjdump

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "lwm_b200", "lib", "liblwm_b200.so")
P = ctypes.c_void_p(0x1000)
N = None
SHAPE, ARG, DEVICE = 2, 3, 1


def _status(lib, name, *args):
    from lwm_b200 import _lib
    _lib.load()
    return getattr(lib, name)(*args), lib.lwm_last_error().decode()


def _step(scales=False, B=1, H=2, Sq=256, Sk=512, D=128, bias=None, tiles=None, counts=None, ws=P):
    """lwm_attn_bwd_step_ordered's arguments: (q, k, v, dout, scale_q, scale_k, scale_v, scale_do, lse, delta, dq_acc,
    dk_acc, dv_acc, B, H, Sq, Sk, D, q_pos0, k_pos0, causal, bias, bias_stride, segment_ids, seg_stride,
    softmax_scale, dkv_init, tiles, tile_count, order_ws, stream)"""
    s = P if scales else N
    return (P, P, P, P, s, s, s, s, P, P, P, P, P, B, H, Sq, Sk, D, 0, 0, 1, bias, 0 if bias is None else Sk, N, 0,
            0.1, 1, tiles, counts, ws, N)


def _infer(B=1, H=2, Q=72, Sk=300, D=128, ws=P, counts=P):
    """lwm_attn_infer_bwd_ordered's arguments: (q16, k16, v16, dout16, scale_q, scale_k, scale_v, scale_do, lse, delta,
    bits, tiles, tile_count, dq_acc, dk_acc, dv_acc, B, H, Q, Sk, D, softmax_scale, order_ws, stream)"""
    return (P, P, P, P, P, P, P, P, P, P, N, P, counts, P, P, P, B, H, Q, Sk, D, 0.1, ws, N)


BAD_CALLS = [
    ("null_workspace", "lwm_attn_bwd_step_ordered", _step(ws=N), ARG, "order_ws"),
    ("null_workspace_map", "lwm_attn_bwd_step_ordered", _step(bias=P, tiles=P, counts=P, ws=N), ARG, "order_ws"),
    ("map_without_counts", "lwm_attn_bwd_step_ordered", _step(bias=P, tiles=P), ARG, "tile_count"),
    ("map_without_mask", "lwm_attn_bwd_step_ordered", _step(tiles=P, counts=P), ARG, "bias or segment_ids"),
    ("partial_scales", "lwm_attn_bwd_step_ordered", _step()[:4] + (P, N, N, N) + _step()[8:], ARG, "scales"),
    ("seq_not_128", "lwm_attn_bwd_step_ordered", _step(Sq=192), SHAPE, "multiples of 128"),
    ("head_dim", "lwm_attn_bwd_step_ordered", _step(D=64), SHAPE, "head_dim"),
    ("semaphores_over_int32", "lwm_attn_bwd_step_ordered", _step(B=64, H=65535, Sq=65536), SHAPE, "int32"),
    ("infer_null_workspace", "lwm_attn_infer_bwd_ordered", _infer(ws=N), ARG, "order_ws"),
    ("infer_map_without_counts", "lwm_attn_infer_bwd_ordered", _infer(counts=N), ARG, "null"),
    ("infer_head_dim", "lwm_attn_infer_bwd_ordered", _infer(D=96), SHAPE, "head_dim"),
    ("infer_bad_shape", "lwm_attn_infer_bwd_ordered", _infer(Q=0), SHAPE, "bad shape"),
    ("infer_tickets_over_int32", "lwm_attn_infer_bwd_ordered", _infer(B=4096, H=4096, Q=64, Sk=128 * 200), SHAPE,
     "int32"),
]


@pytest.mark.parametrize("case,name,args,code,frag", BAD_CALLS, ids=[c[0] for c in BAD_CALLS])
def test_bad_arguments_are_rejected_with_a_message(lib, case, name, args, code, frag):
    status, msg = _status(lib, name, *args)
    assert status == code, (status, msg)
    assert frag in msg, msg


GOOD_CALLS = [
    ("bf16", "lwm_attn_bwd_step_ordered", _step()),
    ("f16", "lwm_attn_bwd_step_ordered", _step(scales=True)),
    ("bf16_map", "lwm_attn_bwd_step_ordered", _step(bias=P, tiles=P, counts=P)),
    ("f16_map", "lwm_attn_bwd_step_ordered", _step(scales=True, bias=P, tiles=P, counts=P)),
    ("infer", "lwm_attn_infer_bwd_ordered", _infer()),
]


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: only meaningful where the device check fails")
@pytest.mark.parametrize("case,name,args", GOOD_CALLS, ids=[c[0] for c in GOOD_CALLS])
def test_well_formed_calls_fail_with_device_error_without_gpu(lib, case, name, args):
    status, msg = _status(lib, name, *args)
    assert status == DEVICE, (status, msg)
    assert "no CPU fallback" in msg or "sm_90" in msg, msg


# attn_bwd_kernel<kF16, kMap, kBits, kOrdered>
_KERNEL = "_ZN3lwm15attn_bwd_kernelI%sEEv14CUtensorMap_stS1_S1_S1_S1_NS_9BwdParamsE"
_MODES = {"bf16": "Lb0ELb0ELb0E", "fp16": "Lb1ELb0ELb0E", "bf16_map": "Lb0ELb1ELb0E", "fp16_map": "Lb1ELb1ELb0E",
          "infer": "Lb1ELb1ELb1E"}
INSTANCES = {(m, o): _KERNEL % (t + ("Lb1E" if o else "Lb0E")) for m, t in _MODES.items() for o in (False, True)}
_INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")


@pytest.fixture(scope="module")
def sass():
    tool = _cuobjdump()
    if tool is None or not os.path.exists(LIB):
        pytest.skip("needs cuobjdump and the built liblwm_b200.so")
    r = subprocess.run([tool, "-sass", "-fun", ",".join(INSTANCES.values()), LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    fns, cur = {}, None
    for line in r.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = fns.setdefault(m.group(1), [])
            continue
        m = _INSN.search(line)
        if m and cur is not None:
            cur.append(m.group(2))
    return fns


@pytest.mark.parametrize("mode", sorted(_MODES))
def test_ordered_instance_keeps_everything_in_registers(sass, mode):
    insns = sass.get(INSTANCES[(mode, True)])
    assert insns, "ordered attn_bwd_kernel instance %s not in the library" % mode
    local = [t for t in insns if re.search(r"\b(LDL|STL)\b", t)]
    assert not local, "local-memory accesses (spills): %s" % local[:4]


@pytest.mark.parametrize("mode", sorted(_MODES))
def test_only_the_ordered_instance_waits_for_its_turn(sass, mode):
    ordered, plain = sass.get(INSTANCES[(mode, True)]), sass.get(INSTANCES[(mode, False)])
    assert ordered and plain
    assert any("NANOSLEEP" in t for t in ordered), "no backed-off turn wait in the ordered instance"
    assert not any("NANOSLEEP" in t or "GLOBALTIMER" in t for t in plain)
