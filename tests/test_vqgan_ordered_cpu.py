"""The ordered (reproducible, batch-invariant) VQGAN entry points without a GPU: argument validation of
lwm_vq_gn_stats_ordered, lwm_vq_prep_f16_ordered and lwm_vq_conv2d_f16_ordered (bad calls, workspaces too small
included, are rejected with a message before the device check; well-formed ones fail with LWM_ERR_DEVICE), and the
machine code of the ordered conv instances: no local memory, and no atomic addition anywhere (the unordered instances
accumulate their statistics with atomic adds; the ordered ones only take an atomic max).
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


def _stats(x=P, st=P, ws=P, ws_bytes=None, n=2, h=16, w=16, c=128, groups=32):
    """lwm_vq_gn_stats_ordered(x, stats, workspace, workspace_bytes, N, H, W, C, groups, stream)"""
    need = n * -(-h * w // 128) * groups * 2 * 4
    return (x, st, ws, need if ws_bytes is None else ws_bytes, n, h, w, c, groups, N)


def _prep(gn=False, scale=P, amax=P, given=0, n=2, c=128, cpad=128):
    """lwm_vq_prep_f16_ordered(x, gn_stats, gamma, beta, out, scale_out, x_absmax, x_absmax_given, N, H, W, C, C_pad,
    groups, upsample2x, eps, stream)"""
    g = P if gn else N
    return (P, g, g, g, P, scale, amax, given, n, 8, 8, c, cpad, 32, 0, 1e-6, N)


def _conv(st=P, ws=P, ws_bytes=None, n=2, cout=128, cout_pad=128, w_scale_inv=0.25, groups=32, ho=16, wo=16):
    """lwm_vq_conv2d_f16_ordered(a, a_scale, w_stacked, bias, residual, out, gn_stats_out, workspace, workspace_bytes,
    absmax_out, N, Hin, Win, Cpad, Ho, Wo, Cout, Cout_pad, ksize, stride, pad, w_scale_inv, groups, clip, stream)"""
    need = n * (ho // 8) * (wo // 16) * 8 * groups * 2 * 4
    return (P, P, P, P, N, P, st, ws, need if ws_bytes is None else ws_bytes, P, n, ho, wo, 64, ho, wo, cout, cout_pad,
            3, 1, 1, w_scale_inv, groups, 0, N)


BAD_CALLS = [
    ("stats_null_x", "lwm_vq_gn_stats_ordered", _stats(x=N), ARG, "null pointer"),
    ("stats_null_workspace", "lwm_vq_gn_stats_ordered", _stats(ws=N), ARG, "null pointer"),
    ("stats_workspace_too_small", "lwm_vq_gn_stats_ordered", _stats(ws_bytes=2 * 2 * 32 * 2 * 4 - 4), SHAPE,
     "workspace too small"),
    ("stats_group_width", "lwm_vq_gn_stats_ordered", _stats(c=100), SHAPE, "C/groups"),
    ("stats_zero_groups", "lwm_vq_gn_stats_ordered", _stats(groups=0), SHAPE, "C/groups"),
    ("stats_empty", "lwm_vq_gn_stats_ordered", _stats(n=0), SHAPE, "non-empty"),
    ("prep_null_scale", "lwm_vq_prep_f16_ordered", _prep(scale=N), ARG, "null pointer"),
    ("prep_raw_without_absmax", "lwm_vq_prep_f16_ordered", _prep(amax=N), ARG, "x_absmax"),
    ("prep_channels", "lwm_vq_prep_f16_ordered", _prep(c=6, cpad=64), SHAPE, "C % 4"),
    ("prep_empty", "lwm_vq_prep_f16_ordered", _prep(n=0), SHAPE, "empty"),
    ("prep_batch_too_large", "lwm_vq_prep_f16_ordered", _prep(gn=True, n=1000), SHAPE, "too large"),
    ("conv_w_scale", "lwm_vq_conv2d_f16_ordered", _conv(w_scale_inv=0.0), ARG, "w_scale_inv"),
    ("conv_stats_without_workspace", "lwm_vq_conv2d_f16_ordered", _conv(ws=N), ARG, "workspace"),
    ("conv_workspace_too_small", "lwm_vq_conv2d_f16_ordered", _conv(ws_bytes=2 * 2 * 8 * 32 * 2 * 4 - 4), SHAPE,
     "workspace too small"),
    ("conv_group_straddles_n_tile", "lwm_vq_conv2d_f16_ordered", _conv(cout=768, cout_pad=768), SHAPE, "N tile"),
    ("conv_group_width_12", "lwm_vq_conv2d_f16_ordered", _conv(cout=384, cout_pad=384), SHAPE, "N tile"),
    ("conv_tile_shape", "lwm_vq_conv2d_f16_ordered", _conv(ho=12), SHAPE, "8 x 16"),
    ("conv_empty", "lwm_vq_conv2d_f16_ordered", _conv(n=0), SHAPE, "empty"),
]


@pytest.mark.parametrize("case,name,args,code,frag", BAD_CALLS, ids=[c[0] for c in BAD_CALLS])
def test_bad_arguments_are_rejected_with_a_message(lib, case, name, args, code, frag):
    status, msg = _status(lib, name, *args)
    assert status == code, (status, msg)
    assert frag in msg, msg


GOOD_CALLS = [
    ("stats", "lwm_vq_gn_stats_ordered", _stats()),
    ("stats_768", "lwm_vq_gn_stats_ordered", _stats(c=768, h=17, w=9)),
    ("prep_raw", "lwm_vq_prep_f16_ordered", _prep()),
    ("prep_raw_given", "lwm_vq_prep_f16_ordered", _prep(given=1)),
    ("prep_gn", "lwm_vq_prep_f16_ordered", _prep(gn=True, amax=N)),
    ("conv_stats", "lwm_vq_conv2d_f16_ordered", _conv()),
    ("conv_stats_512", "lwm_vq_conv2d_f16_ordered", _conv(cout=512, cout_pad=512)),
    ("conv_no_stats", "lwm_vq_conv2d_f16_ordered", _conv(st=N, ws=N, ws_bytes=0)),
    ("conv_no_stats_768", "lwm_vq_conv2d_f16_ordered", _conv(st=N, ws=N, ws_bytes=0, cout=768, cout_pad=768)),
]


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: only meaningful where the device check fails")
@pytest.mark.parametrize("case,name,args", GOOD_CALLS, ids=[c[0] for c in GOOD_CALLS])
def test_well_formed_calls_fail_with_device_error_without_gpu(lib, case, name, args):
    status, msg = _status(lib, name, *args)
    assert status == DEVICE, (status, msg)
    assert "no CPU fallback" in msg or "sm_90" in msg, msg


# conv_wgmma_kernel<NI, kF16 = true, kOrdered>
_KERNEL = "_ZN3lwm17conv_wgmma_kernelILi%dELb1ELb%dEEEv14CUtensorMap_stS1_S1_S1_NS_10ConvParamsE"
WIDTHS = [32, 64, 96, 128, 160, 192, 224, 256]
INSTANCES = {(ni, o): _KERNEL % (ni, o) for ni in WIDTHS for o in (0, 1)}
_INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
_ATOMIC_ADD = re.compile(r"\b(REDG?|ATOM[SG]?)\.\S*(ADD|CAS)")   # a float atomicAdd in shared memory is a CAS loop


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


@pytest.mark.parametrize("ni", WIDTHS)
def test_ordered_conv_keeps_everything_in_registers(sass, ni):
    insns = sass.get(INSTANCES[(ni, 1)])
    assert insns, "ordered conv_wgmma_kernel instance NI=%d not in the library" % ni
    local = [t for t in insns if re.search(r"\b(LDL|STL)\b", t)]
    assert not local, "local-memory accesses (spills): %s" % local[:4]


@pytest.mark.parametrize("ni", WIDTHS)
def test_only_the_unordered_conv_adds_atomically(sass, ni):
    ordered, plain = sass.get(INSTANCES[(ni, 1)]), sass.get(INSTANCES[(ni, 0)])
    assert ordered and plain
    assert any(_ATOMIC_ADD.search(t) for t in plain), "pattern check: the unordered instance has atomic adds"
    assert not [t for t in ordered if _ATOMIC_ADD.search(t)]
