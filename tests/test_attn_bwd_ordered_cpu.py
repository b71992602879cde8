"""The ordered dQ reduction without a GPU: argument validation of lwm_attn_bwd_step and lwm_attn_infer_bwd given an
order_ws (bad calls are rejected with a message before the device check, well-formed ones fail with LWM_ERR_DEVICE;
a null order_ws is the unordered call, to which the ordered limits do not apply), and the machine code of the five ordered attn_bwd_kernel instances: no local memory (warp 9's wait,
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


def _step(scales=False, B=1, H=2, Sq=256, Sk=512, D=128, q_pos0=0, bias=None, tiles=None, counts=None, ws=P, thr=0):
    """lwm_attn_bwd_step's arguments: (q, k, v, dout, scale_q, scale_k, scale_v, scale_do, lse, delta, dq_acc, dk_acc,
    dv_acc, B, H, Sq, Sk, D, q_pos0, k_pos0, causal, bias, bias_stride, segment_ids, seg_stride, softmax_scale,
    dkv_init, tiles, tile_count, order_ws, seed, drop_threshold, batch0, stream)"""
    s = P if scales else N
    return (P, P, P, P, s, s, s, s, P, P, P, P, P, B, H, Sq, Sk, D, q_pos0, 0, 1, bias, 0 if bias is None else Sk, N,
            0, 0.1, 1, tiles, counts, ws, 7, thr, 0, N)


def _infer(B=1, H=2, Q=72, Sk=300, D=128, ws=P, counts=P):
    """lwm_attn_infer_bwd's arguments: (q16, k16, v16, dout16, scale_q, scale_k, scale_v, scale_do, lse, delta, bits,
    tiles, tile_count, dq_acc, dk_acc, dv_acc, B, H, Q, Sk, D, softmax_scale, order_ws, stream)"""
    return (P, P, P, P, P, P, P, P, P, P, N, P, counts, P, P, P, B, H, Q, Sk, D, 0.1, ws, N)


# shapes whose ordered call is over the int32 limits of the workspace; the unordered call takes them (GOOD_CALLS)
_SEM_OVER = dict(B=64, H=65535, Sq=65536)
_TURNS_OVER = dict(H=100, Sq=2 ** 30, Sk=64 * 128, bias=P, tiles=P, counts=P)    # the block map's turns tip it over
_INFER_SEM_OVER = dict(H=65535, Q=64 * 40000, Sk=128)

BAD_CALLS = [
    ("map_without_counts", "lwm_attn_bwd_step", _step(bias=P, tiles=P), ARG, "tile_count"),
    ("map_without_mask", "lwm_attn_bwd_step", _step(tiles=P, counts=P), ARG, "bias or segment_ids"),
    ("partial_scales", "lwm_attn_bwd_step", _step()[:4] + (P, N, N, N) + _step()[8:], ARG, "scales"),
    ("seq_not_128", "lwm_attn_bwd_step", _step(Sq=192), SHAPE, "multiples of 128"),
    ("head_dim", "lwm_attn_bwd_step", _step(D=64), SHAPE, "head_dim"),
    ("semaphores_over_int32", "lwm_attn_bwd_step", _step(**_SEM_OVER), SHAPE, "int32"),
    ("turns_over_int32", "lwm_attn_bwd_step", _step(**_TURNS_OVER), SHAPE, "int32"),
    ("dropout_q_pos0", "lwm_attn_bwd_step", _step(q_pos0=64, thr=6554), SHAPE, "multiple of 128"),
    ("infer_map_without_counts", "lwm_attn_infer_bwd", _infer(counts=N), ARG, "null"),
    ("infer_head_dim", "lwm_attn_infer_bwd", _infer(D=96), SHAPE, "head_dim"),
    ("infer_bad_shape", "lwm_attn_infer_bwd", _infer(Q=0), SHAPE, "bad shape"),
    ("infer_tickets_over_int32", "lwm_attn_infer_bwd", _infer(B=4096, H=4096, Q=64, Sk=128 * 200), SHAPE,
     "int32"),
    ("infer_semaphores_over_int32", "lwm_attn_infer_bwd", _infer(**_INFER_SEM_OVER), SHAPE, "int32"),
]
# the general checks give the same verdict without the workspace and, on the training step, with dropout on
_GENERAL = ("map_without_counts", "map_without_mask", "partial_scales", "seq_not_128", "head_dim",
            "infer_map_without_counts", "infer_head_dim", "infer_bad_shape")
BAD_CALLS += [(c + "_unordered", n, a[:-2] + (N, N) if n == "lwm_attn_infer_bwd" else a[:29] + (N,) + a[30:], code, f)
              for c, n, a, code, f in BAD_CALLS if c in _GENERAL]
BAD_CALLS += [(c + "_dropout", n, a[:31] + (6554,) + a[32:], code, f)
              for c, n, a, code, f in BAD_CALLS if c in _GENERAL and n == "lwm_attn_bwd_step"]


@pytest.mark.parametrize("case,name,args,code,frag", BAD_CALLS, ids=[c[0] for c in BAD_CALLS])
def test_bad_arguments_are_rejected_with_a_message(lib, case, name, args, code, frag):
    status, msg = _status(lib, name, *args)
    assert status == code, (status, msg)
    assert frag in msg, msg


GOOD_CALLS = [
    ("bf16", "lwm_attn_bwd_step", _step()),
    ("f16", "lwm_attn_bwd_step", _step(scales=True)),
    ("bf16_map", "lwm_attn_bwd_step", _step(bias=P, tiles=P, counts=P)),
    ("f16_map", "lwm_attn_bwd_step", _step(scales=True, bias=P, tiles=P, counts=P)),
    ("infer", "lwm_attn_infer_bwd", _infer()),
    ("bf16_dropout", "lwm_attn_bwd_step", _step(thr=6554)),
    ("semaphores_over_int32_unordered", "lwm_attn_bwd_step", _step(ws=N, **_SEM_OVER)),
    ("turns_over_int32_unordered", "lwm_attn_bwd_step", _step(ws=N, **_TURNS_OVER)),
    ("turns_over_int32_without_map", "lwm_attn_bwd_step", _step(**dict(_TURNS_OVER, tiles=N, counts=N))),
    ("infer_semaphores_over_int32_unordered", "lwm_attn_infer_bwd", _infer(ws=N, **_INFER_SEM_OVER)),
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
