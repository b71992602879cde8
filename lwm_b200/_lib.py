"""ctypes binding of liblwm_b200.so (the C ABI declared in include/lwm_b200.h).

The library is built in-tree by `__graft_entry__.build()`. A missing library is a hard error:
there is deliberately no eager/PyTorch fallback for any op."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "liblwm_b200.so")
_lib = None

c_void_p, c_int, c_ll, c_float = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float

# name -> argtypes ; every function returns int status except where noted
_SIGNATURES = {
    "lwm_abi_version": [],
    "lwm_attn_fwd_step": [c_void_p] * 12 + [c_int] * 5 + [c_ll, c_ll, c_int, c_void_p, c_ll, c_void_p, c_ll, c_float,
                                                         c_int, c_int, c_void_p, c_void_p, c_ll, ctypes.c_uint, c_int,
                                                         c_void_p],
    "lwm_attn_fwd_e4m3_step": [c_void_p] * 12 + [c_int] * 5 + [c_ll, c_ll, c_int, c_void_p, c_ll, c_void_p, c_ll,
                                                              c_float, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "lwm_attn_bwd_prep": [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "lwm_attn_bwd_lse": [c_void_p, c_void_p, c_ll, c_float, c_void_p],
    "lwm_attn_bwd_step": [c_void_p] * 13 + [c_int] * 5 + [c_ll, c_ll, c_int, c_void_p, c_ll, c_void_p, c_ll, c_float,
                                                         c_int, c_void_p, c_void_p, c_void_p, c_ll, ctypes.c_uint, c_int,
                                                         c_void_p],
    "lwm_attn_dropout_mask": [c_ll, ctypes.c_uint, c_int, c_int, c_ll, c_ll, c_int, c_int, c_void_p, c_void_p],
    "lwm_attn_to_f16": [c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_void_p],
    "lwm_attn_step_tilemap": [c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_int, c_ll, c_ll, c_int]
                             + [c_void_p] * 6,
    "lwm_attn_absmax": [c_void_p, c_int, c_ll, c_void_p, c_void_p],
    "lwm_attn_absmax_scale": [c_void_p, c_int, c_ll, c_void_p, c_void_p, c_void_p],
    "lwm_attn_scale_from_absmax": [c_void_p, c_int, c_int, c_void_p, c_void_p],
    "lwm_attn_to_f16_scaled": [c_void_p, c_int, c_void_p, c_void_p, c_ll, c_void_p],
    "lwm_attn_e4m3_scale_from_absmax": [c_void_p, c_int, c_int, c_void_p, c_void_p],
    "lwm_attn_to_e4m3_scaled": [c_void_p, c_int, c_void_p, c_void_p, c_ll, c_void_p],
    "lwm_reduce_cast_f32": [c_void_p, c_int, c_void_p, c_int, c_ll, c_void_p],
    "lwm_ring_ctx_create": [c_int, c_int, c_ll, c_int, c_void_p],
    "lwm_ring_ctx_get_handle": [c_void_p, c_void_p],
    "lwm_ring_ctx_open_peers": [c_void_p, c_void_p],
    "lwm_ring_copy": [c_void_p, c_void_p, c_ll, c_void_p],
    "lwm_ring_signal": [c_void_p, c_int, c_int, ctypes.c_uint, c_void_p],
    "lwm_ring_wait": [c_void_p, c_int, ctypes.c_uint, c_void_p],
    "lwm_ring_ctx_destroy": [c_void_p],
    "lwm_ring_plan": [c_int, c_int, c_ll, c_ll, c_int, c_int, c_int, c_void_p],
    "lwm_ring_layout": [c_int, c_ll, c_ll, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "lwm_attn_decode_partial": [c_void_p] * 3 + [c_int] + [c_void_p] * 6 + [c_int] * 5 + [c_ll, c_ll, c_ll, c_int, c_float]
                               + [c_void_p] * 3,
    "lwm_attn_decode_merge": [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_ll, c_void_p],
    "lwm_kv_cache_write_rope": [c_void_p, c_void_p, c_int] + [c_void_p] * 4 + [c_int, c_int, c_ll, c_int, c_int, c_ll,
                                                                               c_int, c_int, c_void_p],
    "lwm_kv_cache_write_q8": [c_void_p, c_void_p, c_int] + [c_void_p] * 6 + [c_int, c_int, c_ll, c_int, c_int, c_ll,
                                                                              c_int, c_int, c_void_p],
    "lwm_kv_dequant_q8": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "lwm_kv_q8_absmax": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p],
    "lwm_kv_q8_stage": [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "lwm_kv_cache_write_at": [c_void_p, c_void_p, c_int] + [c_void_p] * 6 + [c_int, c_void_p, c_ll] + [c_int] * 5
                             + [c_void_p, c_void_p],
    "lwm_rope_check_positions": [c_void_p, c_ll, c_int, c_void_p, c_void_p],
    "lwm_attn_mask_pack": [c_void_p, c_ll, c_ll, c_ll, c_int, c_int, c_ll, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "lwm_attn_infer_tilemap": [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "lwm_attn_infer_partial": [c_void_p] * 12 + [c_int] * 6 + [c_float, c_void_p],
    "lwm_attn_infer_bwd_tilemap": [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "lwm_attn_infer_bwd": [c_void_p] * 16 + [c_int] * 5 + [c_float, c_void_p, c_void_p],
    "lwm_cast_f32_to_bf16": [c_void_p, c_void_p, c_ll, c_void_p],
    "lwm_add_f32": [c_void_p, c_void_p, c_ll, c_void_p],
    "lwm_vq_gn_stats": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "lwm_vq_prep": [c_void_p] * 6 + [c_int] * 7 + [c_float, c_void_p],
    "lwm_vq_conv2d": [c_void_p] * 7 + [c_int] * 13 + [c_void_p],
    "lwm_vq_conv_cin3": [c_void_p] * 4 + [c_int] * 4 + [c_void_p],
    "lwm_vq_prep_f16": [c_void_p] * 7 + [c_int] * 8 + [c_float, c_void_p],
    "lwm_vq_conv2d_f16": [c_void_p] * 8 + [c_int] * 11 + [c_float, c_int, c_int, c_void_p],
    "lwm_vq_gn_stats_ordered": [c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "lwm_vq_prep_f16_ordered": [c_void_p] * 7 + [c_int] * 8 + [c_float, c_void_p],
    "lwm_vq_conv2d_f16_ordered": [c_void_p] * 8 + [c_ll, c_void_p] + [c_int] * 11 + [c_float, c_int, c_int, c_void_p],
    "lwm_vq_argmin": [c_void_p] * 5 + [c_int] * 3 + [c_void_p],
    "lwm_vq_gather": [c_void_p] * 3 + [c_ll, c_int, c_int, c_void_p],
    "lwm_attn_rope": [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p] + [c_int] * 6 + [c_void_p],
    "lwm_attn_absmax_rope": [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "lwm_attn_stage_rope": [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "lwm_reduce_cast_rope_f32": [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "lwm_vq_frame_tokens": [c_void_p] * 3 + [c_int] * 6 + [c_void_p],
    "lwm_vq_unframe_tokens": [c_void_p, c_void_p, c_ll, c_int, c_void_p],
    "lwm_vq_frames_prep": [c_void_p] + [c_int] * 4 + [c_void_p] * 2 + [c_int] * 2 + [c_void_p] * 2 + [c_int] * 6
                          + [c_void_p, c_void_p],
}


class LwmError(RuntimeError):
    pass


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LwmError(
            "liblwm_b200.so not found at %s — run `python __graft_entry__.py` (nvcc, sm_90a) first; "
            "lwm_b200 has no CPU/PyTorch fallback" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    lib.lwm_last_error.restype = ctypes.c_char_p
    lib.lwm_last_error.argtypes = []
    for name, argtypes in _SIGNATURES.items():
        fn = getattr(lib, name, None)
        if fn is None:
            continue  # exported-symbol coverage is asserted by tests/test_abi.py
        fn.restype = c_int
        fn.argtypes = argtypes
    lib.lwm_ring_ctx_heap.restype = c_void_p           # address (in this process) of a rank's heap payload
    lib.lwm_ring_ctx_heap.argtypes = [c_void_p, c_int]
    lib.lwm_ring_ctx_heap_bytes.restype = c_ll
    lib.lwm_ring_ctx_heap_bytes.argtypes = [c_void_p]
    _lib = lib
    return lib


_n_calls = 0


def launch_count():
    """number of C-ABI compute calls made by this process so far (each launches at least one kernel)"""
    return _n_calls


_NOT_COMPUTE = ("lwm_ring_",)      # transport / bootstrap calls launch no kernel of ours


def call(name, *args):
    global _n_calls
    lib = load()
    if not name.startswith(_NOT_COMPUTE):
        _n_calls += 1
    status = getattr(lib, name)(*args)
    if status != 0:
        raise LwmError("%s failed (status %d): %s" % (name, status, lib.lwm_last_error().decode()))


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream_ptr(stream=None):
    import torch
    s = stream if stream is not None else torch.cuda.current_stream()
    return ctypes.c_void_p(s.cuda_stream)
