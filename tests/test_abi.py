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


def test_library_exports_every_declared_symbol_and_its_abi_version(lib):
    names = _declared()
    assert len(names) >= 13
    for n in names:
        assert hasattr(lib, n), "liblwm_b200.so does not export %s" % n
    # version 3: lwm_vq_prep_f16 writes a scaled fp16 plane (scale_out, x_absmax) and lwm_vq_conv2d_f16 reads its scale
    # (a_scale) and can return the output's |max| (absmax_out)
    src = open(os.path.join(ROOT, "include", "lwm_b200.h")).read()
    assert re.search(r"#define LWM_B200_ABI_VERSION 3\b", src)
    assert lib.lwm_abi_version() == 3


def test_python_binding_covers_header():
    from lwm_b200 import _lib
    bound = set(_lib._SIGNATURES) | {"lwm_last_error", "lwm_ring_ctx_heap", "lwm_ring_ctx_heap_bytes"}
    assert set(_declared()) <= bound


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
