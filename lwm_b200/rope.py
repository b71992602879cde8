"""Rotary position embedding of the attention prologue — host mirror of lwm/llama.py:344-375
(`precompute_freqs_cis`, `apply_rotary_emb`; used at llama.py:515-519) over the CUDA kernel `lwm_attn_rope`.

The reference precomputes a complex64 table [max_position, 64] on the host and gathers it by position_ids; the kernel
rebuilds the same float32 angles on the fly, so only the 64 inverse frequencies are kept on the device.
Differentiable: the VJP of a rotation is the rotation by the conjugate, done by the same kernel (conj=1).
No CPU path: tensors must live on an H100."""
import numpy as np
import torch

from . import _lib

_DT = {torch.float32: 0, torch.bfloat16: 1}


def precompute_inv_freq(dim, theta=10000.0, dtype=np.float32):
    """The `freqs` vector of precompute_freqs_cis (llama.py:345), same numpy expression and dtype."""
    return (1.0 / (theta ** (np.arange(0, dim, 2)[: (dim // 2)].astype(dtype) / dim))).astype(np.float32)


class RotaryTable:
    """Stands in for the reference's `freqs_cis` table: holds dim/theta (and max positions for range checks)."""

    def __init__(self, dim, max_position_embedding, theta=10000.0, device="cuda"):
        if dim != 128:
            raise _lib.LwmError("lwm_attn_rope is built for head_dim 128 (LWM-7B), got %d" % dim)
        self.dim, self.max_position, self.theta = dim, int(max_position_embedding), float(theta)
        self.inv_freq = torch.from_numpy(precompute_inv_freq(dim, theta)).to(device)


def precompute_freqs_cis(dim, max_position_embedding, theta=10000.0, dtype=np.float32, device="cuda"):
    """Same call shape as the reference (llama.py:344); returns a RotaryTable instead of a 512 MB complex array."""
    return RotaryTable(dim, max_position_embedding, theta, device)


def _launch(xq, xk, position_ids, table, out_dtype, conj):
    if not xq.is_cuda:
        raise _lib.LwmError("apply_rotary_emb: tensors must be CUDA tensors (no CPU path)")
    B, S, Hq, D = xq.shape
    Hk = xk.shape[2]
    if xk.shape[0] != B or xk.shape[1] != S or xk.shape[3] != D or xq.dtype != xk.dtype:
        raise _lib.LwmError("apply_rotary_emb: xq %s and xk %s disagree" % (tuple(xq.shape), tuple(xk.shape)))
    if xq.dtype not in _DT or out_dtype not in _DT:
        raise _lib.LwmError("apply_rotary_emb: dtypes must be float32 or bfloat16")
    if tuple(position_ids.shape) != (B, S):
        raise _lib.LwmError("apply_rotary_emb: position_ids must be [B,S]")
    xq, xk = xq.contiguous(), xk.contiguous()
    pos = position_ids.to(device=xq.device, dtype=torch.int32).contiguous()
    oq = torch.empty(xq.shape, dtype=out_dtype, device=xq.device)
    ok = torch.empty(xk.shape, dtype=out_dtype, device=xq.device)
    _lib.call("lwm_attn_rope", _lib.ptr(xq), _lib.ptr(xk), _DT[xq.dtype], _lib.ptr(oq), _lib.ptr(ok), _DT[out_dtype],
              _lib.ptr(pos), _lib.ptr(table.inv_freq), B, S, Hq, Hk, D, int(conj), _lib.stream_ptr())
    return oq, ok


class _Rope(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xq, xk, position_ids, table, out_dtype):
        ctx.table, ctx.in_dtype = table, xq.dtype
        ctx.save_for_backward(position_ids)
        return _launch(xq, xk, position_ids, table, out_dtype, conj=False)

    @staticmethod
    def backward(ctx, gq, gk):
        (position_ids,) = ctx.saved_tensors
        dq, dk = _launch(gq, gk, position_ids, ctx.table, ctx.in_dtype, conj=True)
        return dq, dk, None, None, None


def apply_rotary_emb(xq, xk, freqs_cis, dtype=torch.float32, *, position_ids):
    """apply_rotary_emb(xq, xk, freqs_cis, dtype) of llama.py:354-375 with the gather of llama.py:515 folded in:
    xq [B,S,Hq,128], xk [B,S,Hk,128] (head-split projections), freqs_cis = the RotaryTable from precompute_freqs_cis,
    position_ids [B,S] = the positions the reference gathers the table rows by. Returns (xq_out, xk_out) in `dtype`."""
    if not isinstance(freqs_cis, RotaryTable):
        raise _lib.LwmError("apply_rotary_emb: freqs_cis must come from lwm_b200.rope.precompute_freqs_cis")
    if int(position_ids.max()) >= freqs_cis.max_position or int(position_ids.min()) < 0:
        raise _lib.LwmError("apply_rotary_emb: position_ids outside [0, max_position_embedding)")
    return _Rope.apply(xq, xk, position_ids, freqs_cis, dtype)


def rotate(x, freqs_cis, dtype, *, position_ids):
    """apply_rotary_emb on one tensor: x [B,S,H,128] rotated at position_ids int32 [B,S] (same device, already checked
    by check_position_ids), in `dtype`; differentiable like apply_rotary_emb."""
    return _Rope.apply(x, x[:, :, :0], position_ids, freqs_cis, dtype)[0]


ERR_SLOT, ERR_POSITION = 1, 2        # bits of the device error word (LWM_DEVICE_ERR_* in include/lwm_b200.h)
_ERROR_WORDS = {}


def error_word(device):
    """The sticky int32 [1] error word of a GPU, shared by every check of the capturable decode step on it: the KV-cache
    write at the device cursor (ERR_SLOT: a slot past the cache, ERR_POSITION) and the position check of
    ringattention_inference while capturing (ERR_POSITION). take_errors reads and clears it. The word is created with the
    first cache cursor on the device (ShardedKVCache.cursor, or its first eager decode write), never inside a capture,
    where its zero-fill would be recorded and replayed."""
    device = torch.device(device)
    if device.index is None:
        device = torch.device(device.type, torch.cuda.current_device())
    word = _ERROR_WORDS.get(device)
    if word is None:
        if capturing():
            raise RuntimeError("the decode error word of %s does not exist yet: run the step once eagerly (the warm-up) "
                               "before capturing it" % device)
        word = _ERROR_WORDS[device] = torch.zeros(1, dtype=torch.int32, device=device)
    return word


def take_errors(device):
    """-> the error bits (ERR_SLOT | ERR_POSITION) the device checks have set on `device` since the last call, and clears
    them. One device->host synchronisation; 0 means every write and position since then was in range."""
    word = error_word(device)
    bits = int(word.item())
    if bits:
        word.zero_()
    return bits


def capturing():
    """whether the current CUDA stream is capturing a CUDA graph (False without a GPU)"""
    return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()


def check_positions_on_device(position_ids, max_position):
    """ERR_POSITION into the device's error word if any of position_ids (int32, contiguous, on a GPU) is outside
    [0, max_position): the range check without a device->host copy (lwm_rope_check_positions)"""
    _lib.call("lwm_rope_check_positions", _lib.ptr(position_ids), position_ids.numel(), int(max_position),
              _lib.ptr(error_word(position_ids.device)), _lib.stream_ptr())


def check_position_ids(who, freqs_cis, position_ids, shape, device, device_check=True):
    """The rotary-embedding keywords of the ops that rotate inside their own passes -> None (both None) or
    (position_ids int32 [shape] contiguous on `device`, inv_freq). Raises ValueError unless they come together, freqs_cis
    is a RotaryTable, position_ids has `shape` and every position is in [0, max_position). Device positions cost one
    device->host synchronisation (the range check); host positions none (the copy to the device is asynchronous).
    While the current stream is capturing a CUDA graph, position_ids must be a device tensor (a host tensor's copy would
    be recorded with the values it has now) and the range check runs on the device instead, without a synchronisation:
    an out-of-range position sets ERR_POSITION in error_word (device_check=False leaves the check to the caller's
    kernel)."""
    if freqs_cis is None and position_ids is None:
        return None
    if freqs_cis is None or position_ids is None:
        raise ValueError("%s: freqs_cis and position_ids go together (the rotary embedding needs both)" % who)
    if not isinstance(freqs_cis, RotaryTable):
        raise ValueError("%s: freqs_cis must come from lwm_b200.rope.precompute_freqs_cis" % who)
    if tuple(position_ids.shape) != tuple(shape):
        raise ValueError("%s: position_ids must be [B, S_loc] = %s, got %s" % (who, tuple(shape), tuple(position_ids.shape)))
    if capturing():
        if not position_ids.is_cuda:
            raise ValueError("%s: while capturing a CUDA graph position_ids must be a device tensor (the copy of a host "
                             "tensor would replay the values it has at capture)" % who)
        pos = position_ids.to(device=device, dtype=torch.int32).contiguous()
        if device_check and pos.numel():
            check_positions_on_device(pos, freqs_cis.max_position)
        return pos, freqs_cis.inv_freq
    if position_ids.numel():
        lo, hi = torch.stack(torch.aminmax(position_ids)).tolist()
        if lo < 0 or hi >= freqs_cis.max_position:
            raise ValueError("%s: position_ids outside [0, max_position_embedding)" % who)
    pos = position_ids.to(dtype=torch.int32)
    return pos.to(device=device, non_blocking=True).contiguous(), freqs_cis.inv_freq


def split_heads(x, num_heads, head_dim=128):
    """_split_heads (llama.py:376-377): [B,S,H*D] -> [B,S,H,D] — a view, never a copy."""
    return x.view(x.shape[0], x.shape[1], num_heads, head_dim)
