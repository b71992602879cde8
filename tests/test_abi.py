"""The C-ABI library loads without a GPU and exports every symbol include/lwm_b200.h declares;
compute entry points refuse to run without an sm_90 device (no CPU fallback)."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "lwm_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(lwm_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol_and_no_folded_variant(lib):
    names = _declared()
    assert len(names) >= 13
    for n in names:
        assert hasattr(lib, n), "liblwm_b200.so does not export %s" % n
    # version 5: the attention passes take their options as nullable arguments of one entry point each
    # (lwm_attn_fwd_step: scales, block map, dropout; lwm_attn_bwd_step: the same and order_ws; lwm_attn_bwd_prep: out
    # dtype, scale_do; lwm_attn_decode_partial: dtype, the 8-bit cache's k_exp / v_exp, position_ids / inv_freq;
    # lwm_attn_infer_bwd: order_ws; lwm_attn_decode_merge: out dtype), and the per-option variants of them are neither
    # declared nor exported
    src = open(os.path.join(ROOT, "include", "lwm_b200.h")).read()
    assert re.search(r"#define LWM_B200_ABI_VERSION 5\b", src)
    assert lib.lwm_abi_version() == 5
    for gone in ("lwm_attn_fwd_step_dropout", "lwm_attn_bwd_step_dropout", "lwm_attn_bwd_step_ordered",
                 "lwm_attn_infer_bwd_ordered", "lwm_attn_decode_partial_q8"):
        assert gone not in names and not re.search(r"\b%s\b" % gone, src), gone
        assert not hasattr(lib, gone), "liblwm_b200.so still exports %s" % gone


def test_python_binding_covers_header():
    from lwm_b200 import _lib
    bound = set(_lib._SIGNATURES) | {"lwm_last_error", "lwm_ring_ctx_heap", "lwm_ring_ctx_heap_bytes"}
    assert set(_declared()) <= bound


def _prototypes():
    """name -> parameter type list of every function the header declares (comments removed)"""
    src = open(os.path.join(ROOT, "include", "lwm_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    protos = {}
    for m in re.finditer(r"\b(lwm_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", src):
        params = " ".join(m.group(2).split())
        protos[m.group(1)] = [] if params in ("", "void") else [p.strip() for p in params.split(",")]
    return protos


def _ctype_of(param):
    """the ctypes type that binds a C parameter declaration: any pointer is c_void_p, else its scalar type"""
    if "*" in param:
        return ctypes.c_void_p
    words = re.sub(r"\bconst\b", "", param).split()[:-1]       # drop the parameter name
    return {"int": ctypes.c_int, "long long": ctypes.c_longlong, "float": ctypes.c_float,
            "unsigned": ctypes.c_uint}[" ".join(words)]


def test_python_binding_matches_header_prototypes():
    """every bound entry point has argtypes of the same count and kind as the header's prototype, slot by slot: ctypes
    does not check a slip (an int passed where a pointer goes) and the call would only fail on the device"""
    from lwm_b200 import _lib
    protos = _prototypes()
    assert len(protos) >= len(_declared())
    for name, argtypes in _lib._SIGNATURES.items():
        assert name in protos, name
        assert argtypes == [_ctype_of(p) for p in protos[name]], name


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_compute_calls_fail_loudly_without_gpu(lib):
    from lwm_b200 import _lib
    with pytest.raises(_lib.LwmError):
        _lib.call("lwm_cast_f32_to_bf16", None, None, 4, None)
    assert b"no CPU fallback" in lib.lwm_last_error() or b"sm_90" in lib.lwm_last_error()
    from lwm_b200.ringattention import ringattention
    q = torch.zeros(1, 128, 1, 128, dtype=torch.bfloat16)
    with pytest.raises(_lib.LwmError):
        ringattention(q, q, q, None, None)


def test_no_product_import_of_oracle():
    """the product package must never import the oracle (parity claims depend on it)."""
    pkg = os.path.join(ROOT, "lwm_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py") and f != "selftest.py":
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, flags=re.M), f
