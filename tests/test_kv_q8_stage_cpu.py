"""The operand passes that read the 8-bit KV cache directly (lwm_kv_q8_absmax, lwm_kv_q8_stage), without a GPU:
  * declared, exported and bound with matching argument counts, and the ABI version is still 5;
  * every bad argument is rejected with its error code and a message before the device check, and well-formed calls
    reach the device check;
  * QuantizedKV's batch-row view, and the ops classes routing a QuantizedKV to these calls (the bf16 mode's copy to
    lwm_kv_dequant_q8 into its destination) instead of dequantizing it."""
import ctypes
import os

import pytest
import torch

from helpers import abi_row_id

P = ctypes.c_void_p(0x1000)
P_ODD = ctypes.c_void_p(0x1001)
P_4 = ctypes.c_void_p(0x1004)        # 4-byte but not 8-byte aligned
N = None
SHAPE, ARG, DEVICE = 2, 3, 1
NEW_SYMBOLS = ("lwm_kv_q8_absmax", "lwm_kv_q8_stage")


def _prototype_params(name):
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(root, "include", "lwm_b200.h")).read(), flags=re.S)
    m = re.search(r"\bint %s\s*\(([^()]*)\)\s*;" % name, src)
    assert m, name
    return [p.strip() for p in " ".join(m.group(1).split()).split(",")]


def test_symbols_are_declared_exported_and_bound(lib):
    from lwm_b200 import _lib
    for name in NEW_SYMBOLS:
        params = _prototype_params(name)
        assert hasattr(lib, name)
        assert len(_lib._SIGNATURES[name]) == len(params), name
        for param, ct in zip(params, _lib._SIGNATURES[name]):
            assert (ct is ctypes.c_void_p) == ("*" in param), (name, param)
    assert lib.lwm_abi_version() == 5


# lwm_kv_q8_absmax(data, exp, B, L, H, D, out_bits, stream)
AB = (P, P, 2, 64, 4, 128, P, N)
# lwm_kv_q8_stage(data, exp, dst, dst_dtype, scale, B, L, H, D, stream)
ST = (P, P, P, 2, P, 2, 64, 4, 128, N)


def _with(args, **at):
    a = list(args)
    for k, val in at.items():
        a[int(k[1:])] = val
    return tuple(a)


BAD_CALLS = [
    ("lwm_kv_q8_absmax", _with(AB, a0=N), ARG, "null pointer"),
    ("lwm_kv_q8_absmax", _with(AB, a1=N), ARG, "null pointer"),
    ("lwm_kv_q8_absmax", _with(AB, a6=N), ARG, "null pointer"),
    ("lwm_kv_q8_absmax", _with(AB, a5=64), SHAPE, "head_dim"),
    ("lwm_kv_q8_absmax", _with(AB, a2=0), SHAPE, "bad sizes"),
    ("lwm_kv_q8_absmax", _with(AB, a3=0), SHAPE, "bad sizes"),
    ("lwm_kv_q8_absmax", _with(AB, a4=-1), SHAPE, "bad sizes"),
    ("lwm_kv_q8_absmax", _with(AB, a0=P_ODD), ARG, "aligned"),
    ("lwm_kv_q8_absmax", _with(AB, a1=P_ODD), ARG, "aligned"),
    ("lwm_kv_q8_stage", _with(ST, a0=N), ARG, "null pointer"),
    ("lwm_kv_q8_stage", _with(ST, a1=N), ARG, "null pointer"),
    ("lwm_kv_q8_stage", _with(ST, a2=N), ARG, "null pointer"),
    ("lwm_kv_q8_stage", _with(ST, a4=N), ARG, "null pointer"),
    ("lwm_kv_q8_stage", _with(ST, a8=64), SHAPE, "head_dim"),
    ("lwm_kv_q8_stage", _with(ST, a3=1), ARG, "dst dtype codes"),
    ("lwm_kv_q8_stage", _with(ST, a3=0), ARG, "dst dtype codes"),
    ("lwm_kv_q8_stage", _with(ST, a3=4), ARG, "dst dtype codes"),
    ("lwm_kv_q8_stage", _with(ST, a5=0), SHAPE, "bad sizes"),
    ("lwm_kv_q8_stage", _with(ST, a6=0), SHAPE, "bad sizes"),
    ("lwm_kv_q8_stage", _with(ST, a7=0), SHAPE, "bad sizes"),
    ("lwm_kv_q8_stage", _with(ST, a0=P_ODD), ARG, "aligned"),
    ("lwm_kv_q8_stage", _with(ST, a1=P_ODD), ARG, "aligned"),
    ("lwm_kv_q8_stage", _with(ST, a2=P_4), ARG, "aligned"),                 # fp16 copies: 8-byte aligned
    ("lwm_kv_q8_stage", _with(ST, a2=P_ODD, a3=3), ARG, "aligned"),         # e4m3 copies: 4-byte aligned
]


def _status(lib, name, *args):
    from lwm_b200 import _lib
    _lib.load()
    return getattr(lib, name)(*args), lib.lwm_last_error().decode()


@pytest.mark.parametrize("name,args,code,frag", BAD_CALLS,
                         ids=["%s-%d" % (abi_row_id(*c[:2]), i) for i, c in enumerate(BAD_CALLS)])
def test_bad_arguments_are_rejected_with_a_message(lib, name, args, code, frag):
    status, msg = _status(lib, name, *args)
    assert status == code, (status, msg)
    assert frag in msg, msg


GOOD_CALLS = [("lwm_kv_q8_absmax", AB), ("lwm_kv_q8_absmax", _with(AB, a2=1, a3=1, a4=1)),
              ("lwm_kv_q8_stage", ST), ("lwm_kv_q8_stage", _with(ST, a3=3, a2=P_4))]


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: only meaningful where the device check fails")
@pytest.mark.parametrize("name,args", GOOD_CALLS, ids=["%s-%d" % (abi_row_id(*c), i) for i, c in enumerate(GOOD_CALLS)])
def test_well_formed_calls_fail_with_device_error_without_gpu(lib, name, args):
    status, msg = _status(lib, name, *args)
    assert status == DEVICE, (status, msg)


# ------------------------------------------------------------------------------------------------
# the Python surface
# ------------------------------------------------------------------------------------------------
def _cache(B=3, L=5, H=2):
    from lwm_b200.kv_cache import QuantizedKV
    g = torch.Generator().manual_seed(0)
    return QuantizedKV(torch.randint(-127, 128, (B, L, H, 128), dtype=torch.int8, generator=g),
                       torch.randint(-20, 20, (B, H, L, 4), dtype=torch.int8, generator=g))


def test_batch_row_view():
    c = _cache()
    for b in (0, 2, -1):
        r = c[b]
        assert tuple(r.shape) == (1, 5, 2, 128) and tuple(r.exp.shape) == (1, 2, 5, 4)
        assert r.data.data_ptr() == c.data[b].data_ptr() and r.exp.data_ptr() == c.exp[b].data_ptr()
        assert torch.equal(r.data[0], c.data[b]) and torch.equal(r.exp[0], c.exp[b])
    with pytest.raises(IndexError):
        c[3]


@pytest.fixture
def calls(monkeypatch):
    """the C-ABI calls the ops make, recorded instead of run: [(name, args)]"""
    from lwm_b200 import _lib
    log = []
    monkeypatch.setattr(_lib, "call", lambda name, *args: log.append((name, args)))
    monkeypatch.setattr(_lib, "stream_ptr", lambda stream=None: None)

    def no_copy(self, dtype):
        raise AssertionError("the cache was dequantized")
    from lwm_b200.kv_cache import QuantizedKV
    monkeypatch.setattr(QuantizedKV, "dequantize", no_copy)
    return log


def _ptr(a):
    return a.value if isinstance(a, ctypes.c_void_p) else a


def test_ops_stage_the_cache_from_its_codes(calls):
    from lwm_b200 import ringattention as ra
    c = _cache()
    B, L, H, D = c.shape
    dst16 = torch.empty((B, L, H, D), dtype=torch.float16)
    dst8 = torch.empty((B, L, H, D), dtype=torch.float8_e4m3fn)
    dstb = torch.empty((B, L, H, D), dtype=torch.bfloat16)
    scale, bits = torch.ones(1), torch.zeros(1, dtype=torch.int32)
    ra.PeerOpsF16.absmax(c, bits)
    ra.PeerOpsF16.stage(c, dst16, scale)
    ra.PeerOpsE4m3.stage(c[1], dst8[1], scale)
    ra.PeerOpsBf16.stage(c, dstb, None)
    names = [n for n, _ in calls]
    assert names == ["lwm_kv_q8_absmax", "lwm_kv_q8_stage", "lwm_kv_q8_stage", "lwm_kv_dequant_q8"]
    a = [[_ptr(x) for x in args] for _, args in calls]
    assert a[0][:7] == [c.data.data_ptr(), c.exp.data_ptr(), B, L, H, D, bits.data_ptr()]
    assert a[1][:9] == [c.data.data_ptr(), c.exp.data_ptr(), dst16.data_ptr(), 2, scale.data_ptr(), B, L, H, D]
    assert a[2][:9] == [c.data[1].data_ptr(), c.exp[1].data_ptr(), dst8[1].data_ptr(), 3, scale.data_ptr(), 1, L, H, D]
    assert a[3][:8] == [c.data.data_ptr(), c.exp.data_ptr(), dstb.data_ptr(), 1, B, L, H, D]
    # the scales: the fp16 and e4m3 scale from the codes' |max|, with the existing scale kernels
    calls.clear()
    out = torch.empty(1)
    ra.PeerOpsF16.scale_of(c, out)
    ra.PeerOpsE4m3.scale_of(c, out)
    assert [n for n, _ in calls] == ["lwm_kv_q8_absmax", "lwm_attn_scale_from_absmax",
                                     "lwm_kv_q8_absmax", "lwm_attn_e4m3_scale_from_absmax"]
