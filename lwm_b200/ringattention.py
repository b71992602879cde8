"""Host side of the H100 RingAttention operator — same call signature as the reference's
`ringattention(q, k, v, attn_bias, segment_ids, *, axis_name, float32_logits, cache_idx,
blockwise_kwargs)` bound with functools.partial at lwm/llama.py:540-557 and called at
lwm/llama.py:569 on per-device shards inside shard_map.

Translation of the execution model (SURVEY.md §8b):
  * shard_map over mesh axis 'sp'  ->  one process per GPU; `axis_name` resolves to a
    torch.distributed process group registered with `set_axis_group` (default: WORLD; a
    non-initialised process group means ring size 1).
  * lax.ppermute(k, v : i -> i+1)  ->  NCCL send/recv (batch_isend_irecv) on a side stream into
    the other half of a double buffer while the tile kernel consumes the current half.
  * the (numerator, denominator, max) scan carry -> fp32 carry buffers merged in the kernel's
    epilogue (include/lwm_b200.h: lwm_attn_fwd_step).

Everything numeric happens in liblwm_b200.so; this file only sequences launches and NCCL calls.
There is no fallback: without the library / an sm_90 GPU the op raises.
"""
import math
import os

import torch
import torch.distributed as dist

from . import _lib
from . import ring_exec as rx
from . import ring_peer as rp
from . import ring_schedule as rs

_AXIS_GROUPS = {}
_DEFAULT_PRECISION = os.environ.get("LWM_ATTN_PRECISION", "fp16")


def set_default_precision(precision: str) -> None:
    """'fp16' (default — the mode that meets the 1e-3 parity bound): every operand is converted once per pass to a
    power-of-two-scaled fp16 copy (exact for bf16 inputs, one rounding to 11 significant bits for fp32 inputs) and P / dS
    keep fp16's 11 bits; un-rounded fp32 output kept as the backward's residual. 'bf16': bf16 tensor-core operands,
    P / dS rounded to bf16 (8 bits) — the usual flash-attention numerics, 1.3e-3 .. 2.6e-3 on white-noise inputs."""
    global _DEFAULT_PRECISION
    if precision not in ("bf16", "fp16"):
        raise ValueError("precision must be 'bf16' or 'fp16'")
    _DEFAULT_PRECISION = precision


def set_axis_group(axis_name: str, group) -> None:
    """Bind a mesh-axis name (the reference's 'sp') to a torch.distributed process group. Call it on every rank of
    WORLD, in the same order, like torch.distributed.new_group itself."""
    _AXIS_GROUPS[axis_name] = group


def attention_bias_from_mask(attention_mask, dtype=torch.bfloat16):
    """The call site's mask -> bias transform (lwm/llama.py:526, 532-537): attention_mask [B,S_global] (>0 = attend)
    -> additive bias [B,1,1,S_global] in `dtype`: 0 where attended, finfo(dtype).min where not."""
    m = attention_mask[:, None, None, :]
    zero = torch.zeros((), dtype=dtype, device=m.device)
    low = torch.full((), torch.finfo(dtype).min, dtype=dtype, device=m.device)
    return torch.where(m > 0, zero, low)


def decode_attention_mask(attention_mask, query_length, cache_index, max_decoder_length=None):
    """Boolean mask [B,1,Q,K] for `ringattention_inference` while decoding from a KV cache (lwm/llama.py:574-591):
    causal_mask[i, j] = j <= i + cache_index over the cache length, combined (AND) with the padding mask
    attention_mask [B,K] (combine_masks)."""
    K = attention_mask.shape[-1] if max_decoder_length is None else int(max_decoder_length)
    dev = attention_mask.device
    causal = torch.arange(K, device=dev)[None, :] <= (torch.arange(query_length, device=dev) + int(cache_index))[:, None]
    return (attention_mask[:, None, None, :K] > 0) & causal[None, None]


def _resolve_group(axis_name):
    if not (dist.is_available() and dist.is_initialized()):
        return None, 0, 1
    group = _AXIS_GROUPS.get(axis_name, dist.group.WORLD)
    return group, dist.get_rank(group), dist.get_world_size(group)


def _check_blockwise_kwargs(kw, s_q, s_k):
    kw = dict(kw or {})
    cbs = kw.get("causal_block_size", None)
    if cbs not in (None, 1):
        raise NotImplementedError("causal_block_size must be None or 1 (lwm/llama.py:546 uses 1)")
    if not kw.get("deterministic", True) and float(kw.get("attn_pdrop", 0.0)) > 0.0:
        raise NotImplementedError("attention dropout is not supported (attn_pdrop is 0.0 in every LWM config)")
    for name, s in (("query_chunk_size", s_q), ("key_chunk_size", s_k)):
        c = kw.get(name)
        if c is not None and s % int(c) != 0 and s > int(c):
            raise ValueError("%s=%d must divide the per-device sequence length %d" % (name, c, s))
    # policy / precision / prevent_cse / dropout_rng / dtype are XLA-side knobs: accepted, unused.
    return cbs is not None


def _prep_bias(attn_bias, B):
    if attn_bias is None:
        return None
    b = attn_bias
    if b.dim() == 4:
        if b.shape[1] != 1 or b.shape[2] != 1:
            raise ValueError("attn_bias must be [B,1,1,S_global] (lwm/llama.py:527,563)")
        b = b.reshape(b.shape[0], b.shape[-1])
    if b.shape[0] != B:
        b = b.expand(B, b.shape[-1])
    return b.to(torch.float32).contiguous()


class _RingAttnFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, bias, seg, causal, axis_name, layout, precision):
        group, rank, world = _resolve_group(axis_name)
        out, res = ring_forward(q, k, v, bias, seg, causal, group, rank, world, layout, precision)
        # residuals stay in the schedule's compute layout (zigzag chunks, operand dtype), so the backward only has
        # to permute dout on entry and dq on exit
        ctx.n_chunks = len(res["q_chunks"])
        sc = [t for t in res.get("scales", ()) if t is not None]
        ctx.n_scales = len(sc)
        ctx.save_for_backward(k, v, bias, seg, *res["q_chunks"], *res["out_chunks"], *res["lse_chunks"], *sc)
        ctx.causal, ctx.axis_name, ctx.layout, ctx.precision = causal, axis_name, layout, precision
        return out

    @staticmethod
    def backward(ctx, dout):
        saved = ctx.saved_tensors
        k, v, bias, seg = saved[:4]
        n = ctx.n_chunks
        res = dict(q_chunks=list(saved[4:4 + n]), out_chunks=list(saved[4 + n:4 + 2 * n]),
                   lse_chunks=list(saved[4 + 2 * n:4 + 3 * n]))
        sc = list(saved[4 + 3 * n:4 + 3 * n + ctx.n_scales])
        res["scales"] = tuple(sc) if sc else (None,) * (n + 2)
        group, rank, world = _resolve_group(ctx.axis_name)
        dq, dk, dv = ring_backward(res, k, v, dout.contiguous(), bias, seg, ctx.causal, group, rank, world,
                                   ctx.layout, ctx.precision)
        return dq, dk, dv, None, None, None, None, None, None


def _check_mask_extent(bias, seg, rank, world, Sq, Sk):
    """attn_bias / segment_ids are indexed by GLOBAL token position (they are replicated along the ring,
    lwm/llama.py:563-564): a per-shard mask would be read out of bounds by the kernels."""
    if bias is not None and bias.shape[-1] < world * Sk:
        raise ValueError("attn_bias covers %d keys but the ring holds %d: pass the un-sharded [B,1,1,S_global] bias "
                         "(lwm/llama.py:563)" % (bias.shape[-1], world * Sk))
    if seg is not None and seg.shape[-1] < max(world * Sq, world * Sk):
        raise ValueError("segment_ids covers %d positions but the ring holds %d: pass the un-sharded [B,S_global] ids "
                         "(lwm/llama.py:564)" % (seg.shape[-1], max(world * Sq, world * Sk)))


def ringattention(q, k, v, attn_bias=None, segment_ids=None, *, axis_name="sp", float32_logits=True,
                  cache_idx=None, blockwise_kwargs=None, layout="auto", precision=None):
    """Drop-in for the reference op. q [B,Sq_loc,H,D], k/v [B,Sk_loc,H,D] CUDA shards of the contiguously
    sequence-sharded tensors (in_specs lwm/llama.py:559-565), all bfloat16 or all float32 (the dtype the reference's
    scripts run with); attn_bias [B,1,1,S_global] additive (0 / finfo.min), segment_ids [B,S_global] or None, both
    replicated along the ring. Returns the local output shard [B,Sq_loc,H,D] in the input dtype; differentiable w.r.t.
    q,k,v (gradients in the input dtype). With float32 inputs in the default precision mode nothing is rounded to bf16:
    the operands are rounded once to scaled fp16 (11 bits) and the output / gradients are the un-rounded fp32
    accumulators.

    float32_logits: logits/softmax/carries are always fp32 here (the reference default, True).
    layout: 'contiguous' = the reference's schedule; 'zigzag' = internally rebalance the causal
    work across ranks (same inputs/outputs); 'auto' picks zigzag when it applies.
    precision: None -> module default (set_default_precision / $LWM_ATTN_PRECISION): 'fp16' | 'bf16'."""
    precision = precision or _DEFAULT_PRECISION
    if precision not in ("bf16", "fp16"):
        raise ValueError("precision must be 'bf16' or 'fp16'")
    if cache_idx is not None:
        raise NotImplementedError("cache_idx is always None at the reference call site (lwm/llama.py:544)")
    if not q.is_cuda:
        raise _lib.LwmError("ringattention: tensors must live on an sm_90 GPU (no CPU fallback)")
    in_dtype = q.dtype
    if not (k.dtype == in_dtype and v.dtype == in_dtype and in_dtype in (torch.bfloat16, torch.float32)):
        raise TypeError("ringattention: q, k, v must all be bfloat16 or all float32 (fp32 logits and accumulation "
                        "are internal)")
    group, rank, world = _resolve_group(axis_name)
    native_f32 = in_dtype == torch.float32 and precision == "fp16" and (world == 1 or _transport(group) == "peer")
    if in_dtype == torch.float32 and not native_f32:
        # bf16 operand mode / NCCL transport: fp32 callers go through one rounding of q/k/v to bf16 (2^-9 relative)
        q, k, v = q.to(torch.bfloat16), k.to(torch.bfloat16), v.to(torch.bfloat16)
    B, Sq, H, D = q.shape
    causal = _check_blockwise_kwargs(blockwise_kwargs, Sq, k.shape[1])
    bias = _prep_bias(attn_bias, B)
    seg = None
    if segment_ids is not None:
        seg = segment_ids.to(torch.int32).contiguous()
    _check_mask_extent(bias, seg, rank, world, Sq, k.shape[1])
    out = _RingAttnFn.apply(q.contiguous(), k.contiguous(), v.contiguous(), bias, seg, causal, axis_name, layout,
                            precision)
    return out if out.dtype == in_dtype else out.to(in_dtype)


# ------------------------------------------------------------------------------------------------
# single-step wrappers over the C ABI
# ------------------------------------------------------------------------------------------------
def to_f16(x, stream=None):
    """bf16 tensor -> (exact scaled fp16 copy, device scalar scale) — include/lwm_b200.h: lwm_attn_to_f16."""
    x16 = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    scale = torch.empty(2, dtype=torch.float32, device=x.device)   # [scale, absmax-bits workspace]
    _lib.call("lwm_attn_to_f16", _lib.ptr(x), _lib.ptr(x16), _lib.ptr(scale), _lib.ptr(scale[1:]), x.numel(),
              _lib.stream_ptr(stream))
    return x16, scale


def step_tilemap(B, Sq, Sk, q_pos0, k_pos0, causal, bias, seg, fwd=True, bwd=True, stream=None):
    """Block map of one training step with a bias and/or segment ids (include/lwm_b200.h: lwm_attn_step_tilemap)
    -> (fwd_tiles, fwd_count, bwd_tiles, bwd_count); the maps not asked for are None."""
    dev = (bias if bias is not None else seg).device
    n_qt, n_q64, n_kt = Sq // 128, Sq // 64, Sk // 128
    ft = torch.empty((B, n_qt, n_kt), dtype=torch.int32, device=dev) if fwd else None
    fc = torch.empty((B, n_qt), dtype=torch.int32, device=dev) if fwd else None
    bt = torch.empty((B, n_kt, n_q64), dtype=torch.int32, device=dev) if bwd else None
    bc = torch.empty((B, n_kt), dtype=torch.int32, device=dev) if bwd else None
    ws = torch.empty(B * (n_q64 + n_kt) * 4, dtype=torch.int32, device=dev)
    _lib.call("lwm_attn_step_tilemap", _lib.ptr(bias), 0 if bias is None else bias.shape[1], _lib.ptr(seg),
              0 if seg is None else seg.shape[1], B, Sq, Sk, int(q_pos0), int(k_pos0), int(bool(causal)), _lib.ptr(ft),
              _lib.ptr(fc), _lib.ptr(bt), _lib.ptr(bc), _lib.ptr(ws), _lib.stream_ptr(stream))
    return ft, fc, bt, bc


def fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last,
             stream=None, scales=None, out_f32=None, tilemap=None):
    """tilemap: None, or the forward map (tiles, counts) of step_tilemap for these arguments: the tile kernel then
    visits only the KV tiles in it (same results, bit for bit)."""
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    if tilemap is not None:
        tail = (_lib.ptr(tilemap[0]), _lib.ptr(tilemap[1]), _lib.stream_ptr(stream))
        if scales is not None:
            _lib.call("lwm_attn_fwd_step_map_f16", _lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(scales[0]),
                      _lib.ptr(scales[1]), _lib.ptr(scales[2]), _lib.ptr(out_f32), _lib.ptr(out), _lib.ptr(lse),
                      _lib.ptr(acc_o), _lib.ptr(acc_m), _lib.ptr(acc_l), B, H, Sq, Sk, D, int(q_pos0), int(k_pos0),
                      int(bool(causal)), _lib.ptr(bias), 0 if bias is None else bias.shape[1], _lib.ptr(seg),
                      0 if seg is None else seg.shape[1], 1.0 / math.sqrt(D), int(first), int(last), *tail)
        else:
            _lib.call("lwm_attn_fwd_step_map", _lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(out), _lib.ptr(lse),
                      _lib.ptr(acc_o), _lib.ptr(acc_m), _lib.ptr(acc_l), B, H, Sq, Sk, D, int(q_pos0), int(k_pos0),
                      int(bool(causal)), _lib.ptr(bias), 0 if bias is None else bias.shape[1], _lib.ptr(seg),
                      0 if seg is None else seg.shape[1], 1.0 / math.sqrt(D), int(first), int(last), *tail)
        return
    if scales is not None:   # fp16-operand kernels: q/k/v are fp16 copies, scales = (sq, sk, sv) device scalars
        _lib.call("lwm_attn_fwd_step_f16", _lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(scales[0]),
                  _lib.ptr(scales[1]), _lib.ptr(scales[2]), _lib.ptr(out_f32), _lib.ptr(out), _lib.ptr(lse),
                  _lib.ptr(acc_o),
                  _lib.ptr(acc_m), _lib.ptr(acc_l), B, H, Sq, Sk, D, int(q_pos0), int(k_pos0), int(bool(causal)),
                  _lib.ptr(bias), 0 if bias is None else bias.shape[1], _lib.ptr(seg),
                  0 if seg is None else seg.shape[1], 1.0 / math.sqrt(D), int(first), int(last),
                  _lib.stream_ptr(stream))
        return
    _lib.call("lwm_attn_fwd_step", _lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(out), _lib.ptr(lse),
              _lib.ptr(acc_o), _lib.ptr(acc_m), _lib.ptr(acc_l), B, H, Sq, Sk, D, int(q_pos0), int(k_pos0),
              int(bool(causal)), _lib.ptr(bias), 0 if bias is None else bias.shape[1], _lib.ptr(seg),
              0 if seg is None else seg.shape[1], 1.0 / math.sqrt(D), int(first), int(last),
              _lib.stream_ptr(stream))


def bwd_prep(out, dout, delta, stream=None):
    B, Sq, H, D = out.shape
    if out.dtype == torch.float32:
        _lib.call("lwm_attn_bwd_prep_f32", _lib.ptr(out), _lib.ptr(dout), _lib.ptr(delta), B, H, Sq, D,
                  _lib.stream_ptr(stream))
        return
    _lib.call("lwm_attn_bwd_prep", _lib.ptr(out), _lib.ptr(dout), _lib.ptr(delta), B, H, Sq, D,
              _lib.stream_ptr(stream))


F16_P_BOOST_LOG2 = 14.0      # include/lwm_b200.h: LWM_ATTN_F16_P_BOOST_LOG2


def lse_for_bwd(lse, stream=None, f16=False):
    """-lse*log2(e) (masked-level rows -> -inf), computed once per backward: what bwd_step takes as `lse`.
    f16=True: for the fp16-operand kernel, which keeps P^T * 2^14 (the +14 rides on this array)."""
    out = torch.empty_like(lse)
    _lib.call("lwm_attn_bwd_lse", _lib.ptr(lse), _lib.ptr(out), lse.numel(), F16_P_BOOST_LOG2 if f16 else 0.0,
              _lib.stream_ptr(stream))
    return out


def bwd_step(q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg, stream=None,
             scales=None, init=False, tilemap=None):
    """`lse` is the PRE-SCALED array returned by lse_for_bwd. init=True: dk_acc/dv_acc rows are written, not accumulated.
    tilemap: None, or the backward map (tiles, counts) of step_tilemap for these arguments (dK, dV bit-identical; dQ
    up to the order of its reductions)."""
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    if tilemap is not None:
        tail = (_lib.ptr(tilemap[0]), _lib.ptr(tilemap[1]), _lib.stream_ptr(stream))
        if scales is not None:
            _lib.call("lwm_attn_bwd_step_map_f16", _lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(dout),
                      _lib.ptr(scales[0]), _lib.ptr(scales[1]), _lib.ptr(scales[2]), _lib.ptr(scales[3]), _lib.ptr(lse),
                      _lib.ptr(delta), _lib.ptr(dq_acc), _lib.ptr(dk_acc), _lib.ptr(dv_acc), B, H, Sq, Sk, D,
                      int(q_pos0), int(k_pos0), int(bool(causal)), _lib.ptr(bias), 0 if bias is None else bias.shape[1],
                      _lib.ptr(seg), 0 if seg is None else seg.shape[1], 1.0 / math.sqrt(D), int(bool(init)), *tail)
        else:
            _lib.call("lwm_attn_bwd_step_map", _lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(dout), _lib.ptr(lse),
                      _lib.ptr(delta), _lib.ptr(dq_acc), _lib.ptr(dk_acc), _lib.ptr(dv_acc), B, H, Sq, Sk, D,
                      int(q_pos0), int(k_pos0), int(bool(causal)), _lib.ptr(bias), 0 if bias is None else bias.shape[1],
                      _lib.ptr(seg), 0 if seg is None else seg.shape[1], 1.0 / math.sqrt(D), int(bool(init)), *tail)
        return
    if scales is not None:   # (sq, sk, sv, sdo)
        _lib.call("lwm_attn_bwd_step_f16", _lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(dout), _lib.ptr(scales[0]),
                  _lib.ptr(scales[1]), _lib.ptr(scales[2]), _lib.ptr(scales[3]), _lib.ptr(lse), _lib.ptr(delta),
                  _lib.ptr(dq_acc), _lib.ptr(dk_acc), _lib.ptr(dv_acc), B, H, Sq, Sk, D, int(q_pos0), int(k_pos0),
                  int(bool(causal)), _lib.ptr(bias), 0 if bias is None else bias.shape[1], _lib.ptr(seg),
                  0 if seg is None else seg.shape[1], 1.0 / math.sqrt(D), int(bool(init)), _lib.stream_ptr(stream))
        return
    _lib.call("lwm_attn_bwd_step", _lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(dout), _lib.ptr(lse),
              _lib.ptr(delta), _lib.ptr(dq_acc), _lib.ptr(dk_acc), _lib.ptr(dv_acc), B, H, Sq, Sk, D,
              int(q_pos0), int(k_pos0), int(bool(causal)), _lib.ptr(bias),
              0 if bias is None else bias.shape[1], _lib.ptr(seg), 0 if seg is None else seg.shape[1],
              1.0 / math.sqrt(D), int(bool(init)), _lib.stream_ptr(stream))


def _map_kw(q, k, q_pos0, k_pos0, causal, bias, seg, fwd):
    """{} without a bias and segment ids, else {"tilemap": this step's forward (fwd) or backward map}"""
    if bias is None and seg is None:
        return {}
    m = step_tilemap(q.shape[0], q.shape[1], k.shape[1], q_pos0, k_pos0, causal, bias, seg, fwd=fwd, bwd=not fwd)
    return {"tilemap": m[:2] if fwd else m[2:]}


def mapped_fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last, **kw):
    """fwd_step over the step's block map whenever a bias or segment ids are given: the step the ring executors run"""
    fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last, **kw,
             **_map_kw(q, k, q_pos0, k_pos0, causal, bias, seg, True))


def mapped_bwd_step(q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg, **kw):
    """bwd_step over the step's block map whenever a bias or segment ids are given"""
    bwd_step(q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg, **kw,
             **_map_kw(q, k, q_pos0, k_pos0, causal, bias, seg, False))


def cast_f32_to_bf16(src, dst, stream=None):
    _lib.call("lwm_cast_f32_to_bf16", _lib.ptr(src), _lib.ptr(dst), src.numel(), _lib.stream_ptr(stream))


# ------------------------------------------------------------------------------------------------
# ring drivers
# ------------------------------------------------------------------------------------------------
class CudaOps:
    """The injected step functions of ring_exec: thin calls into liblwm_b200.so."""
    fwd_step = staticmethod(mapped_fwd_step)
    bwd_prep = staticmethod(bwd_prep)
    lse_for_bwd = staticmethod(lse_for_bwd)
    bwd_step = staticmethod(mapped_bwd_step)
    cast = staticmethod(cast_f32_to_bf16)

    @staticmethod
    def accumulate(acc, start, length, buf):
        for b in range(acc.shape[0]):
            dst = acc[b, start:start + length]
            _lib.call("lwm_add_f32", _lib.ptr(dst), _lib.ptr(buf[b]), dst.numel(), _lib.stream_ptr())


class CudaOpsF16(CudaOps):
    """fp16-internal precision: the step functions convert each bf16 operand once (cached for the lifetime
    of one forward/backward pass, keyed by storage) and call the fp16-operand kernels."""

    def __init__(self):
        self._cache = {}
        self.out_f32 = {}     # bf16 out chunk (by address) -> fp32 copy, the residual the backward's delta uses

    def _f16(self, x):
        key = (x.data_ptr(), tuple(x.shape))
        hit = self._cache.get(key)
        if hit is None:
            x16, scale = to_f16(x)
            hit = (x16, scale, x)          # keep the source alive so its address cannot be recycled
            self._cache[key] = hit
        return hit[0], hit[1]

    def fwd_step(self, q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last):
        (q16, sq), (k16, sk), (v16, sv) = self._f16(q), self._f16(k), self._f16(v)
        o32 = None
        if last:
            o32 = torch.empty(out.shape, dtype=torch.float32, device=out.device)
            self.out_f32[out.data_ptr()] = o32
        mapped_fwd_step(q16, k16, v16, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last,
                        scales=(sq, sk, sv), out_f32=o32)

    @staticmethod
    def lse_for_bwd(lse):
        return lse_for_bwd(lse, f16=True)

    def bwd_step(self, q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg):
        (q16, sq), (k16, sk), (v16, sv), (d16, sd) = self._f16(q), self._f16(k), self._f16(v), self._f16(dout)
        mapped_bwd_step(q16, k16, v16, d16, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg,
                        scales=(sq, sk, sv, sd))


def _f32_residuals(ops, res):
    """fp16 precision mode: the backward's delta = rowsum(dO o O) is taken from the un-rounded fp32 output."""
    if isinstance(ops, CudaOpsF16):
        res["out_chunks"] = [ops.out_f32.get(o.data_ptr(), o) for o in res["out_chunks"]]
    return res


# ------------------------------------------------------------------------------------------------
# step functions in the form the peer-memory executor (ring_peer.py) and the single-GPU path take them
# ------------------------------------------------------------------------------------------------
def _dt(t):
    if t.dtype == torch.float32:
        return 0
    if t.dtype == torch.bfloat16:
        return 1
    raise TypeError("expected float32 or bfloat16, got %s" % t.dtype)


class PeerOpsF16:
    """fp16 operand mode: operands are power-of-two-scaled fp16 copies sharing ONE scale per sharded tensor."""
    op_dtype, op_itemsize, scaled = torch.float16, 2, True

    @staticmethod
    def absmax(x, bits):
        _lib.call("lwm_attn_absmax", _lib.ptr(x), _dt(x), x.numel(), _lib.ptr(bits), _lib.stream_ptr())

    @staticmethod
    def make_scale(table, col):
        s = torch.empty(1, dtype=torch.float32, device=table.device)
        _lib.call("lwm_attn_scale_from_absmax", _lib.ptr(table.view(-1)[col:]), table.shape[0], table.shape[1],
                  _lib.ptr(s), _lib.stream_ptr())
        return s

    @staticmethod
    def scale_of(x, out):
        """out[0] = 2^(e-12), e the exponent of |x|max (the power-of-two scale of the fp16 operand copy of x)"""
        bits = torch.empty(1, dtype=torch.int32, device=x.device)
        st = _lib.stream_ptr()
        _lib.call("lwm_attn_absmax_scale", _lib.ptr(x), _dt(x), x.numel(), _lib.ptr(bits), _lib.ptr(out), st)

    @staticmethod
    def stage(x, dst, scale):
        _lib.call("lwm_attn_to_f16_scaled", _lib.ptr(x), _dt(x), _lib.ptr(dst), _lib.ptr(scale), x.numel(),
                  _lib.stream_ptr())

    @staticmethod
    def fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last, scales, out_f32):
        mapped_fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last,
                        scales=scales, out_f32=out_f32)

    @staticmethod
    def bwd_prep(out, dout16, sdo, delta):
        B, Sq, H, D = out.shape
        _lib.call("lwm_attn_bwd_prep_f16", _lib.ptr(out), _dt(out), _lib.ptr(dout16), _lib.ptr(sdo), _lib.ptr(delta),
                  B, H, Sq, D, _lib.stream_ptr())

    @staticmethod
    def lse_for_bwd(lse):
        return lse_for_bwd(lse, f16=True)

    @staticmethod
    def bwd_step(q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg, scales, init):
        mapped_bwd_step(q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg,
                        scales=scales, init=init)

    @staticmethod
    def reduce_cast(srcs, dst):
        import ctypes
        arr = (ctypes.c_void_p * len(srcs))(*[t.data_ptr() for t in srcs])
        _lib.call("lwm_reduce_cast_f32", arr, len(srcs), _lib.ptr(dst), _dt(dst), dst.numel(), _lib.stream_ptr())

    cast = staticmethod(cast_f32_to_bf16)


class PeerOpsBf16(PeerOpsF16):
    """bf16 operand mode: staging is a plain copy (fp32 inputs are rounded to bf16 there), no scales."""
    op_dtype, op_itemsize, scaled = torch.bfloat16, 2, False

    @staticmethod
    def stage(x, dst, scale):
        dst.copy_(x)

    @staticmethod
    def fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last, scales, out_f32):
        mapped_fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last)
        if last and out_f32 is not None:
            out_f32.copy_(out)

    @staticmethod
    def bwd_prep(out, dout, sdo, delta):
        bwd_prep(out, dout, delta)

    @staticmethod
    def lse_for_bwd(lse):
        return lse_for_bwd(lse, f16=False)

    @staticmethod
    def bwd_step(q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg, scales, init):
        mapped_bwd_step(q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg, init=init)


_PEER_BROKEN = {}      # process group id -> reason: the peer-memory heaps could not be set up for this group


def _transport(group=None):
    """'peer' (default): copy-engine pulls/puts over peer-mapped heaps (ring_peer.py). 'nccl': the two-sided
    send/recv executor (ring_exec.py) — the portable alternative (and what the gloo CPU tests drive); also what a group
    is switched to, with a warning, when all its ranks agree that the peer heaps cannot be mapped on this box."""
    t = os.environ.get("LWM_RING_TRANSPORT", "peer")
    if t not in ("nccl", "peer"):
        raise ValueError("LWM_RING_TRANSPORT must be 'peer' or 'nccl'")
    if t == "peer" and (id(group) if group is not None else 0) in _PEER_BROKEN:
        return "nccl"
    return t


def _peer_transport(group, device, nbytes_hint=0):
    """the group's peer transport, or None (after a collective, loud switch to NCCL) when it cannot be set up"""
    import warnings
    try:
        tr = rp.CudaPeerTransport.get(group, device)
        if nbytes_hint:
            tr.ensure(nbytes_hint)
        return tr
    except rp.PeerTransportUnavailable as e:
        _PEER_BROKEN[id(group) if group is not None else 0] = str(e)
        warnings.warn("lwm_b200: peer-memory ring transport unavailable (%s): this process group now uses the two-sided "
                      "NCCL executor (LWM_RING_TRANSPORT=nccl)" % e)
        return None


def _ops_for(precision):
    return CudaOpsF16() if precision == "fp16" else CudaOps


def _peer_ops(precision):
    return PeerOpsF16 if precision == "fp16" else PeerOpsBf16


def _local_scales(ops, tensors):
    """single GPU: per-tensor scales from the local |max| (same kernels as the sharded exchange, world = 1)"""
    if not ops.scaled:
        return [None] * len(tensors)
    table = torch.zeros((1, 4), dtype=torch.int32, device=tensors[0].device)
    out = []
    for c, t in enumerate(tensors):
        ops.absmax(t, table[0, c:c + 1])
        out.append(ops.make_scale(table, c))
    return out


def _stage_local(ops, x, scale):
    if not ops.scaled and x.dtype == ops.op_dtype:
        return x
    y = torch.empty(x.shape, dtype=ops.op_dtype, device=x.device)
    ops.stage(x, y, scale)
    return y


def ring_forward(q, k, v, bias, seg, causal, group, rank, world, layout="auto", precision="bf16"):
    """-> (out, residuals). out is fp32 (un-rounded) for fp32 inputs, bf16 otherwise. world == 1 is the
    single-launch path (no carry buffers)."""
    B, Sq, H, D = q.shape
    want_f32 = q.dtype == torch.float32
    if world == 1:
        ops = _peer_ops(precision)
        sq, sk, sv = _local_scales(ops, (q, k, v))
        q16, k16, v16 = _stage_local(ops, q, sq), _stage_local(ops, k, sk), _stage_local(ops, v, sv)
        out = torch.empty((B, Sq, H, D), dtype=torch.bfloat16, device=q.device)
        out32 = torch.empty((B, Sq, H, D), dtype=torch.float32, device=q.device) if (ops.scaled or want_f32) else None
        lse = torch.empty((B, H, Sq), dtype=torch.float32, device=q.device)
        ops.fwd_step(q16, k16, v16, out, lse, None, None, None, 0, 0, causal, bias, seg, True, True, (sq, sk, sv), out32)
        res = dict(q_chunks=[q16], out_chunks=[out32 if ops.scaled else out], lse_chunks=[lse], scales=(sq, sk, sv))
        return (out32 if want_f32 else out), res
    lay = rs.choose_layout(world, Sq, k.shape[1], causal, layout)
    if _transport(group) == "peer":
        plan = rs.make_peer_plan(world, rank, Sq, k.shape[1], causal, lay)
        pops = _peer_ops(precision)
        tr = _peer_transport(group, q.device, rp._layout_for(plan, q.shape, k.shape[1], pops).total)
        if tr is not None:
            return rp.run_forward(plan, q, k, v, bias, seg, causal, pops, tr, want_f32)
        if want_f32:        # the NCCL executor takes bf16 operands (documented in ringattention())
            out, res = ring_forward(q.to(torch.bfloat16), k.to(torch.bfloat16), v.to(torch.bfloat16), bias, seg, causal,
                                    group, rank, world, layout, precision)
            return out.float(), res
    ops = _ops_for(precision)
    plan = rs.make_plan(world, rank, Sq, k.shape[1], causal, lay, n_sub_first=rs.auto_sub(world, k.shape[1], lay))
    out, res = rx.run_forward(plan, q, k, v, bias, seg, causal, group, ops)
    return out, _f32_residuals(ops, res)


def ring_backward(res, k, v, dout, bias, seg, causal, group, rank, world, layout="auto", precision="bf16"):
    B, Sk, H, D = k.shape
    dev = k.device
    want_f32 = k.dtype == torch.float32
    if world == 1:
        ops = _peer_ops(precision)
        q16, out, lse = res["q_chunks"][0], res["out_chunks"][0], res["lse_chunks"][0]
        sq, sk, sv = res["scales"]
        Sq = q16.shape[1]
        sdo = _local_scales(ops, (dout,))[0]
        k16, v16, d16 = _stage_local(ops, k, sk), _stage_local(ops, v, sv), _stage_local(ops, dout, sdo)
        delta = torch.empty((B, H, Sq), dtype=torch.float32, device=dev)
        ops.bwd_prep(out, d16, sdo, delta)
        nlse = ops.lse_for_bwd(lse)
        dq_acc = torch.zeros((B, Sq, H, D), dtype=torch.float32, device=dev)
        dk_acc = torch.empty((B, Sk, H, D), dtype=torch.float32, device=dev)     # written, not accumulated (init)
        dv_acc = torch.empty((B, Sk, H, D), dtype=torch.float32, device=dev)
        ops.bwd_step(q16, k16, v16, d16, nlse, delta, dq_acc, dk_acc, dv_acc, 0, 0, causal, bias, seg,
                     (sq, sk, sv, sdo), True)
        if want_f32:
            return dq_acc, dk_acc, dv_acc
        dq, dk, dv = [torch.empty(t.shape, dtype=torch.bfloat16, device=dev) for t in (dq_acc, dk_acc, dv_acc)]
        cast_f32_to_bf16(dq_acc, dq)
        cast_f32_to_bf16(dk_acc, dk)
        cast_f32_to_bf16(dv_acc, dv)
        return dq, dk, dv
    lay = rs.choose_layout(world, dout.shape[1], Sk, causal, layout)
    if _transport(group) == "peer":
        plan = rs.make_peer_plan(world, rank, dout.shape[1], Sk, causal, lay)
        return rp.run_backward(plan, res, k, v, dout, bias, seg, causal, _peer_ops(precision),
                               rp.CudaPeerTransport.get(group, dev), want_f32)
    if want_f32:            # forward fell back to the NCCL executor: bf16 operands in, fp32 gradients out
        dq, dk, dv = ring_backward(res, k.to(torch.bfloat16), v.to(torch.bfloat16), dout.to(torch.bfloat16), bias, seg,
                                   causal, group, rank, world, layout, precision)
        return dq.float(), dk.float(), dv.float()
    ops = _ops_for(precision)
    n_sub = rs.auto_sub(world, Sk, lay)
    plan = rs.make_plan(world, rank, dout.shape[1], Sk, causal, lay, n_sub_first=n_sub, n_sub_last=n_sub)
    return rx.run_backward(plan, res, k, v, dout, bias, seg, causal, group, ops)


# ------------------------------------------------------------------------------------------------
# inference path: ringattention_inference (lwm/llama.py:601-614)
# ------------------------------------------------------------------------------------------------
# Query rows at which the tensor-core kernel (attn_fwd_kernel's inference mode) takes over from the GEMV kernel, which
# streams K/V once per query row. From tools/perf_infer.py (H100, H = 32): at K = 131072 the tensor-core path is faster
# from Q = 8 in fp32 and bf16 (bf16 Q = 4: 3.6 vs 3.1 ms); with short caches the GEMV kernel stays ahead up to
# Q = 64, by at most 0.15 ms per call.
INFER_MIN_Q = 8


def _check_infer_dtypes(q, k, v):
    if not (q.dtype == k.dtype == v.dtype and q.dtype in (torch.bfloat16, torch.float32)):
        raise TypeError("ringattention_inference: q, k, v must all be bfloat16 or all float32")


def decode_partial(q, k, v, mask_u8, k_pos0, stream=None):
    """This rank's partial over its KV shard with the GEMV kernel (bf16 or fp32 q/k/v, read as they are)
    -> (o_part [B*Q*H,128] fp32, ml_part [B*Q*H,2] fp32)."""
    B, Q, H, D = q.shape
    Sk = k.shape[1]
    rows = B * Q * H
    splits = max(1, min(256, (Sk + 2047) // 2048))
    o_part = torch.empty(rows, D, dtype=torch.float32, device=q.device)
    ml_part = torch.empty(rows, 2, dtype=torch.float32, device=q.device)
    ws = torch.empty(splits * rows * (D + 2), dtype=torch.float32, device=q.device)
    sb = sq = 0
    if mask_u8 is not None:
        sb, sq = mask_u8.stride(0), mask_u8.stride(-2)
    fn = "lwm_attn_decode_partial_f32" if q.dtype == torch.float32 else "lwm_attn_decode_partial"
    _lib.call(fn, _lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(mask_u8), _lib.ptr(o_part),
              _lib.ptr(ml_part), _lib.ptr(ws), B, H, Q, Sk, D, int(k_pos0), int(sb), int(sq), splits,
              1.0 / math.sqrt(D), _lib.stream_ptr(stream))
    return o_part, ml_part


def decode_merge(o_parts, ml_parts, n_part, out_shape, dtype):
    """merge n_part partials per row ([rows][n_part][128], [rows][n_part][2]) into the normalised output"""
    out = torch.empty(out_shape, dtype=dtype, device=o_parts.device)
    rows = o_parts.shape[0]
    lse = torch.empty(rows, dtype=torch.float32, device=o_parts.device)
    fn = "lwm_attn_decode_merge_f32" if dtype == torch.float32 else "lwm_attn_decode_merge"
    _lib.call(fn, _lib.ptr(o_parts), _lib.ptr(ml_parts), n_part, _lib.ptr(out), _lib.ptr(lse), rows,
              _lib.stream_ptr())
    return out


def mask_pack(mask, B, n_slabs, ncols):
    """bool/uint8 mask [Bm,1,Q,K] (Bm in {1, B}; read through its strides) -> (bits [n_slabs,B,Q,kw] int32 for the
    key columns [s*ncols, (s+1)*ncols) of slab s, row_any [B,Q] int32)."""
    Q = mask.shape[2]
    m = mask.view(torch.uint8) if mask.dtype == torch.bool else mask
    if m.dtype != torch.uint8:
        m = (m != 0).view(torch.uint8)
    kw = (ncols + 127) // 128 * 4
    bits = torch.empty(n_slabs, B, Q, kw, dtype=torch.int32, device=m.device)
    row_any = torch.empty(B, Q, dtype=torch.int32, device=m.device)
    sb = m.stride(0) if m.shape[0] > 1 else 0
    _lib.call("lwm_attn_mask_pack", _lib.ptr(m), sb, m.stride(2), m.stride(3), B, Q, 0, ncols, n_slabs,
              _lib.ptr(bits), _lib.ptr(row_any), _lib.stream_ptr())
    return bits, row_any


def _scaled_f16(x):
    scale = torch.empty(1, dtype=torch.float32, device=x.device)
    PeerOpsF16.scale_of(x, scale)
    return _stage_local(PeerOpsF16, x, scale), scale


def infer_partial(q, k, v, bits, row_any):
    """This rank's partial with the tensor-core kernel: q [B,Q,H,128] against k/v [B,Sk,H,128] (bf16 or fp32, staged
    to scaled fp16 here), bits [B,Q,kw] / row_any [B,Q] (row_any over the whole ring) or None
    -> (o_part [B*Q*H,128], ml_part [B*Q*H,2])."""
    B, Q, H, D = q.shape
    Sk = k.shape[1]
    dev = q.device
    n_qt, n_kt = (Q + 127) // 128, (Sk + 127) // 128
    tiles = torch.empty(B, n_qt, n_kt, dtype=torch.int32, device=dev)
    counts = torch.empty(B, n_qt, dtype=torch.int32, device=dev)
    _lib.call("lwm_attn_infer_tilemap", _lib.ptr(bits), _lib.ptr(row_any), B, Q, Sk, _lib.ptr(tiles),
              _lib.ptr(counts), _lib.stream_ptr())
    (q16, sq), (k16, sk), (v16, sv) = _scaled_f16(q), _scaled_f16(k), _scaled_f16(v)
    ctas = n_qt * H * B
    splits = 1 if ctas >= 132 else min(n_kt, -(-132 // ctas))     # key splits: fill the 132 SMs
    rows = B * Q * H
    o_part = torch.empty(rows, D, dtype=torch.float32, device=dev)
    ml_part = torch.empty(rows, 2, dtype=torch.float32, device=dev)
    ws = torch.empty(splits * rows * (D + 2), dtype=torch.float32, device=dev) if splits > 1 else None
    _lib.call("lwm_attn_infer_partial", _lib.ptr(q16), _lib.ptr(k16), _lib.ptr(v16), _lib.ptr(sq), _lib.ptr(sk),
              _lib.ptr(sv), _lib.ptr(bits), _lib.ptr(tiles), _lib.ptr(counts), _lib.ptr(o_part), _lib.ptr(ml_part),
              _lib.ptr(ws), B, H, Q, Sk, D, splits, 1.0 / math.sqrt(D), _lib.stream_ptr())
    return o_part, ml_part


class InferOps:
    """The kernels of the q-sharded protocol (_infer_sharded); tests substitute stand-ins."""
    mask_pack = staticmethod(mask_pack)
    merge = staticmethod(decode_merge)

    @staticmethod
    def partial(q, k, v, mask, row_any, tensor_cores):
        """mask: bits [B,Q,kw] when tensor_cores, else uint8 [B,Q,Sk] (or None)"""
        if tensor_cores:
            return infer_partial(q, k, v, mask, row_any)
        return decode_partial(q, k, v, mask, 0)


class TorchComm:
    """The collectives of the q-sharded protocol over a torch.distributed group (tests substitute a fake)."""

    def __init__(self, group, world):
        self.group, self.world = group, world

    def all_gather(self, x):
        """-> [world, *x.shape], rank-major"""
        out = torch.empty((self.world * x.shape[0],) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        dist.all_gather_into_tensor(out, x.contiguous(), group=self.group)
        return out.view((self.world,) + tuple(x.shape))

    def all_to_all(self, x):
        """x [world, ...]: slab s goes to rank s; -> [world, ...], slab r came from rank r"""
        x = x.contiguous()
        out = torch.empty(x.shape, dtype=x.dtype, device=x.device)
        dist.all_to_all_single(out, x, group=self.group)
        return out


def _infer_sharded(q, k, v, mask, comm, ops=InferOps):
    """q-sharded protocol (query length > 1 on a ring of comm.world ranks): q [B,Q_loc,H,D] and mask [Bm,1,Q_loc,K]
    are this rank's query rows, k/v [B,S_loc,H,D] its KV shard (K = world*S_loc). Each rank computes the partials of
    ALL world*Q_loc rows over its own keys, so K/V never move; per rank the traffic is world*Q_loc*H*D words of q and
    of partials plus Q_loc*K/8 bytes of mask. Returns this rank's [B,Q_loc,H,D] output."""
    B, Ql, H, D = q.shape
    Sk = k.shape[1]
    W = comm.world
    qls = comm.all_gather(torch.tensor([Ql], dtype=torch.int64, device=q.device))
    if bool((qls != Ql).any()):
        raise ValueError("ringattention_inference: every rank must hold the same number of query rows, got %s"
                         % qls.flatten().tolist())
    Qg = W * Ql
    # 1. every rank gets all query rows (it stages them with one scale, from the same data)
    q_all = comm.all_gather(q).transpose(0, 1).reshape(B, Qg, H, D)
    tc = Qg >= INFER_MIN_Q
    m = row_any = None
    if mask is not None:
        if tc:
            # 2./3. bits of my rows, one slab per key owner, and the rows' global "any true" flags
            bits, any_loc = ops.mask_pack(mask, B, W, Sk)                         # [W,B,Ql,kw], [B,Ql]
            row_any = comm.all_gather(any_loc).transpose(0, 1).reshape(B, Qg)
            m = comm.all_to_all(bits).transpose(0, 1).reshape(B, Qg, -1)
        else:
            m8 = mask.view(torch.uint8) if mask.dtype == torch.bool else (mask != 0).view(torch.uint8)
            slabs = m8[:, 0, :, :W * Sk].expand(B, Ql, W * Sk).reshape(B, Ql, W, Sk).permute(2, 0, 1, 3)
            m = comm.all_to_all(slabs).transpose(0, 1).reshape(B, Qg, Sk)
    # 4. partials of all rows over my keys (key splits merged locally)
    o, ml = ops.partial(q_all, k, v, m, row_any, tc)
    # 5. each owner gets its rows' partials back
    o = comm.all_to_all(o.view(B, W, Ql, H, D).transpose(0, 1))
    ml = comm.all_to_all(ml.view(B, W, Ql, H, 2).transpose(0, 1))
    # 6. merge the world partials
    o = o.permute(1, 2, 3, 0, 4).reshape(B * Ql * H, W, D)
    ml = ml.permute(1, 2, 3, 0, 4).reshape(B * Ql * H, W, 2)
    return ops.merge(o.contiguous(), ml.contiguous(), W, (B, Ql, H, D), q.dtype)


def ringattention_inference(q, k, v, attn_mask, axis_name="sp"):
    """Drop-in for the reference's inference-time op (bound at lwm/llama.py:601-614 inside shard_map).
    q, k, v all bfloat16 or all float32; the output has their dtype (fp32: the un-rounded fp32 result).
    k/v [B,S_loc,H,D] = this rank's contiguous shard of the KV cache.
      * Q = 1 (generation): q [B,1,H,D] and attn_mask [B,1,1,K_global] are replicated along the ring. Every rank
        reduces its own shard with the GEMV kernel and the (o, lse) partials, a few KB, are all-gathered and merged.
      * Q > 1 on a ring: q [B,Q_loc,H,D] and attn_mask [B,1,Q_loc,K_global] are sharded on the query dimension
        (q_sp_dim, lwm/llama.py:598); returns this rank's rows. See _infer_sharded.
    Below INFER_MIN_Q query rows the GEMV kernel runs; from there on the tensor-core kernel over scaled fp16 copies
    of q, k, v with fp32 logits, softmax and accumulation, visiting only the KV tiles the mask leaves visible.
    attn_mask: bool/uint8 [B or 1,1,Q,K_global] (nonzero = attend) or None (every key visible). A row with no true
    entry in all of K_global averages V over all keys (the reference's finfo.min semantics)."""
    if not q.is_cuda:
        raise _lib.LwmError("ringattention_inference: tensors must live on an sm_90 GPU (no CPU fallback)")
    _check_infer_dtypes(q, k, v)
    group, rank, world = _resolve_group(axis_name)
    B, Q, H, D = q.shape
    Sk = k.shape[1]
    if attn_mask is not None:
        if attn_mask.dim() != 4 or attn_mask.shape[1] != 1 or attn_mask.shape[2] != Q or attn_mask.shape[0] not in (1, B):
            raise ValueError("attn_mask must be [B,1,Q,K_global] (lwm/llama.py:585-590)")
        if attn_mask.shape[-1] < (world if Q > 1 else rank + 1) * Sk:
            raise ValueError("attn_mask covers %d keys but the ring holds %d" % (attn_mask.shape[-1], world * Sk))
    q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
    if world > 1 and Q > 1:
        return _infer_sharded(q, k, v, attn_mask, TorchComm(group, world))
    if Q >= INFER_MIN_Q:
        bits = row_any = None
        if attn_mask is not None:
            bits, row_any = mask_pack(attn_mask, B, 1, Sk)
            bits = bits[0]
        o_part, ml_part = infer_partial(q, k, v, bits, row_any)
        return decode_merge(o_part, ml_part, 1, (B, Q, H, D), q.dtype)
    mask = None
    if attn_mask is not None:
        mask = attn_mask.to(torch.uint8).expand(B, 1, Q, attn_mask.shape[-1]).contiguous()
    o_part, ml_part = decode_partial(q, k, v, mask, rank * Sk)
    rows = B * Q * H
    if world > 1:
        o_all = torch.empty(world, rows, D, dtype=torch.float32, device=q.device)
        ml_all = torch.empty(world, rows, 2, dtype=torch.float32, device=q.device)
        dist.all_gather_into_tensor(o_all, o_part, group=group)
        dist.all_gather_into_tensor(ml_all, ml_part, group=group)
        o_part = o_all.permute(1, 0, 2).contiguous()       # [row][rank][D]
        ml_part = ml_all.permute(1, 0, 2).contiguous()
    return decode_merge(o_part, ml_part, world, (B, Q, H, D), q.dtype)
