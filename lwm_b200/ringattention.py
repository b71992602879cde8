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
import operator
import os

import numpy as np

import torch
import torch.distributed as dist

from . import _lib
from . import ring_exec as rx
from . import rope as _rope
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


def causal_attention_mask(attention_mask, segment_ids=None, query_length=None):
    """Boolean mask [B,1,Q,Q] for `ringattention_inference` without a KV cache (lwm/llama.py:580-592), the branch
    training takes for short sequences: causal (key j <= query i) AND padding (attention_mask [B,S] > 0 at the key)
    AND, with segment_ids [B,S], same segment (combine_masks). Q = query_length, default S."""
    Q = attention_mask.shape[-1] if query_length is None else int(query_length)
    dev = attention_mask.device
    causal = torch.ones(Q, Q, dtype=torch.bool, device=dev).tril_()
    m = (attention_mask[:, None, None, :Q] > 0) & causal[None, None]
    if segment_ids is not None:
        seg = segment_ids[:, :Q]
        m = m & (seg[:, :, None] == seg[:, None, :])[:, None]
    return m


def _resolve_group(axis_name):
    if not (dist.is_available() and dist.is_initialized()):
        return None, 0, 1
    group = _AXIS_GROUPS.get(axis_name, dist.group.WORLD)
    return group, dist.get_rank(group), dist.get_world_size(group)


def dropout_threshold(p):
    """attn_pdrop -> the 16-bit drop threshold of the kernels: an entry is dropped iff its Philox u16 < thr, so the
    realised rate thr / 65536 is within 2^-17 of p. 0 means no dropout."""
    p = float(p)
    if not 0.0 <= p < 1.0:
        raise ValueError("attn_pdrop must be in [0, 1), got %r" % p)
    return min(65535, int(round(p * 65536)))


def _dropout_of(kw, world):
    """blockwise_kwargs -> None (no dropout) or (seed, thr) for the dropout kernels"""
    thr = dropout_threshold(kw.get("attn_pdrop", 0.0))
    if kw.get("deterministic", True) or thr == 0:
        return None
    rng = kw.get("dropout_rng")
    if rng is None:
        if world > 1:
            raise ValueError("ringattention: attention dropout on a ring needs dropout_rng, an int seed passed alike on "
                             "every rank (a seed drawn per rank could differ between them)")
        rng = int(torch.randint(-2 ** 63, 2 ** 63 - 1, (), dtype=torch.int64))   # torch's default CPU generator
    else:
        try:
            if isinstance(rng, (bool, np.bool_)) or (isinstance(rng, torch.Tensor) and rng.dtype == torch.bool):
                raise TypeError
            rng = operator.index(rng)       # any integer: int, numpy integers, 0-d integer tensors
        except TypeError:
            raise TypeError("dropout_rng must be an integer seed or None, got %s" % type(rng).__name__) from None
    seed = int(rng) & (2 ** 64 - 1)
    return (seed - 2 ** 64 if seed >= 2 ** 63 else seed), thr


def _check_blockwise_kwargs(kw, s_q, s_k, world=1):
    """-> (causal, dropout): dropout is None, or (seed, thr) when deterministic is False and attn_pdrop > 0 (the seed,
    a signed 64-bit int, is dropout_rng, or drawn from torch's default CPU generator when that is None on one GPU)"""
    kw = dict(kw or {})
    cbs = kw.get("causal_block_size", None)
    if cbs not in (None, 1):
        raise NotImplementedError("causal_block_size must be None or 1 (lwm/llama.py:546 uses 1)")
    for name, s in (("query_chunk_size", s_q), ("key_chunk_size", s_k)):
        c = kw.get(name)
        if c is not None and s % int(c) != 0 and s > int(c):
            raise ValueError("%s=%d must divide the per-device sequence length %d" % (name, c, s))
    # policy / precision / prevent_cse / dtype are XLA-side knobs: accepted, unused.
    return cbs is not None, _dropout_of(kw, world)


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
    def forward(ctx, q, k, v, bias, seg, causal, axis_name, layout, precision, rope_pos=None, inv_freq=None,
                rope_k=True, dropout=None):
        """rope_pos / inv_freq: None, or q (and k when rope_k) are un-rotated and the rotary embedding at these positions
        (int32 [B,Sq]) is applied inside the operand staging; k and the positions are saved instead of a rotated k.
        dropout: None or (seed, thr), kept for the backward, which regenerates the same mask"""
        group, rank, world = _resolve_group(axis_name)
        rope = None if rope_pos is None else (rope_pos, inv_freq)
        out, res = ring_forward(q, k, v, bias, seg, causal, group, rank, world, layout, precision, rope, rope_k,
                                dropout=dropout)
        # residuals stay in the schedule's compute layout (zigzag chunks, operand dtype), so the backward only has
        # to permute dout on entry and dq on exit
        ctx.n_chunks = len(res["q_chunks"])
        sc = [t for t in res.get("scales", ()) if t is not None]
        ctx.n_scales = len(sc)
        ctx.save_for_backward(k, v, bias, seg, rope_pos, *res["q_chunks"], *res["out_chunks"], *res["lse_chunks"],
                              *sc)
        ctx.causal, ctx.axis_name, ctx.layout, ctx.precision = causal, axis_name, layout, precision
        ctx.inv_freq, ctx.rope_k, ctx.dropout = inv_freq, rope_k, dropout
        return out

    @staticmethod
    def backward(ctx, dout):
        saved = ctx.saved_tensors
        k, v, bias, seg, rope_pos = saved[:5]
        n = ctx.n_chunks
        res = dict(q_chunks=list(saved[5:5 + n]), out_chunks=list(saved[5 + n:5 + 2 * n]),
                   lse_chunks=list(saved[5 + 2 * n:5 + 3 * n]))
        sc = list(saved[5 + 3 * n:5 + 3 * n + ctx.n_scales])
        res["scales"] = tuple(sc) if sc else (None,) * (n + 2)
        group, rank, world = _resolve_group(ctx.axis_name)
        rope = None if rope_pos is None else (rope_pos, ctx.inv_freq)
        dq, dk, dv = ring_backward(res, k, v, dout.contiguous(), bias, seg, ctx.causal, group, rank, world,
                                   ctx.layout, ctx.precision, rope, ctx.rope_k, dropout=ctx.dropout)
        return dq, dk, dv, None, None, None, None, None, None, None, None, None, None


def _check_mask_extent(bias, seg, rank, world, Sq, Sk):
    """attn_bias / segment_ids are indexed by GLOBAL token position (they are replicated along the ring,
    lwm/llama.py:563-564): a per-shard mask would be read out of bounds by the kernels."""
    if bias is not None and bias.shape[-1] < world * Sk:
        raise ValueError("attn_bias covers %d keys but the ring holds %d: pass the un-sharded [B,1,1,S_global] bias "
                         "(lwm/llama.py:563)" % (bias.shape[-1], world * Sk))
    if seg is not None and seg.shape[-1] < max(world * Sq, world * Sk):
        raise ValueError("segment_ids covers %d positions but the ring holds %d: pass the un-sharded [B,S_global] ids "
                         "(lwm/llama.py:564)" % (seg.shape[-1], max(world * Sq, world * Sk)))


def _check_rope(freqs_cis, position_ids, q, k, rotate_k=True):
    """the rotary-embedding keywords of ringattention -> None or (position_ids int32 [B,Sq_loc] on q's device, inv_freq)"""
    if (rotate_k and freqs_cis is not None and position_ids is not None and isinstance(freqs_cis, _rope.RotaryTable)
            and q.shape[1] != k.shape[1]):
        raise ValueError("ringattention: the rotary embedding is applied to q and k at the same positions, which needs "
                         "Sq == Sk (got %d and %d); with a rotated KV cache call apply_rotary_emb on q yourself"
                         % (q.shape[1], k.shape[1]))
    return _rope.check_position_ids("ringattention", freqs_cis, position_ids, (q.shape[0], q.shape[1]), q.device)


def _quantized_kv(op, q, k, v, rotates_k):
    """whether k and v are the 8-bit cache (kv_cache.QuantizedKV); raises ValueError where it does not apply"""
    from .kv_cache import QuantizedKV
    qk, qv = isinstance(k, QuantizedKV), isinstance(v, QuantizedKV)
    if not (qk or qv):
        return False
    if qk != qv:
        raise ValueError("%s: k and v must both be QuantizedKV or neither" % op)
    if q.dtype not in (torch.bfloat16, torch.float32):
        raise ValueError("%s: with an 8-bit cache q must be bfloat16 or float32, got %s" % (op, q.dtype))
    if rotates_k:
        raise ValueError("%s: the 8-bit cache holds rotated keys; pass rotate_k=False with the rotary keywords" % op)
    if torch.is_grad_enabled() and q.requires_grad:
        raise ValueError("%s: the 8-bit cache is for generation only (no gradient); run under torch.no_grad()" % op)
    return True


def _peer_ready(q, k, causal, group, rank, world, layout, precision):
    """world > 1: whether this call runs on the peer-memory executor (sets up its heap, as ring_forward would)"""
    if _transport(group) != "peer":
        return False
    lay = rs.choose_layout(world, q.shape[1], k.shape[1], causal, layout)
    plan = rs.make_peer_plan(world, rank, q.shape[1], k.shape[1], causal, lay)
    tr = _peer_transport(group, q.device, rp._layout_for(plan, q.shape, k.shape[1], _peer_ops(precision)).total)
    return tr is not None


def ringattention(q, k, v, attn_bias=None, segment_ids=None, *, axis_name="sp", float32_logits=True,
                  cache_idx=None, blockwise_kwargs=None, layout="auto", precision=None, freqs_cis=None,
                  position_ids=None, rotate_k=True):
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
    precision: None -> module default (set_default_precision / $LWM_ATTN_PRECISION): 'fp16' | 'bf16'.

    freqs_cis, position_ids: both None (the reference call), or q and k are the UN-rotated head-split projections and
    the op applies the rotary embedding of lwm/llama.py:517-519 itself: freqs_cis is the RotaryTable of
    lwm_b200.rope.precompute_freqs_cis, position_ids [B,S_loc] the positions of this rank's rows (sharded like q; Sq ==
    Sk). Bit-identical to ringattention(*apply_rotary_emb(q, k, freqs_cis, q.dtype, position_ids=position_ids), v, ...)
    under autograd (dQ up to the order of its fp32 reductions), but on one GPU and on the peer-memory ring the rotation
    happens inside the passes that stage q and k (and the conjugate rotation inside the final casts of dQ and dK), so the
    rotated q and k are never written to memory. position_ids gets no gradient.

    rotate_k=False: k is already rotated (the KV cache of the generation path, written by ShardedKVCache.concatenate
    with the same keywords) and only q is rotated, at position_ids [B,Sq_loc]; Sq != Sk is allowed (the cached prefill:
    q against the whole cache). Bit-identical to ringattention(apply_rotary_emb(q, ...)[0], k, v, ...) in the same sense;
    dK is the gradient w.r.t. k as passed, and only dQ gets the conjugate rotation.

    k, v may be the 8-bit cache (kv_cache.QuantizedKV, both or neither) in the cached prefill: q bf16 or fp32 without
    gradient, and rotate_k=False when the rotary keywords are given. The shards are dequantized to q's dtype (exact; one
    transient copy of each) and the op runs on them as above.

    Attention dropout: blockwise_kwargs=dict(deterministic=False, attn_pdrop=p, dropout_rng=seed) with 0 < p < 1, as
    at the reference call site. A dropped (query, key) entry leaves the softmax's numerator and denominator (no 1/(1-p)
    rescale); a row left without a surviving key outputs 0 and gets zero gradients. The mask is a function of (seed, p,
    batch row, head, GLOBAL query and key position) only (lwm_b200/csrc/attn_dropout.cuh), regenerated inside the tile
    kernels, so it is the same for any layout, world size or executor. dropout_rng: an int seed (pass the same one on
    every rank of the axis group), or None on one GPU for a seed drawn from torch's default CPU generator."""
    precision = precision or _DEFAULT_PRECISION
    if precision not in ("bf16", "fp16"):
        raise ValueError("precision must be 'bf16' or 'fp16'")
    if cache_idx is not None:
        raise NotImplementedError("cache_idx is always None at the reference call site (lwm/llama.py:544)")
    if _quantized_kv("ringattention", q, k, v, bool(rotate_k) and freqs_cis is not None):
        k, v = k.dequantize(q.dtype), v.dequantize(q.dtype)
    rope = _check_rope(freqs_cis, position_ids, q, k, rotate_k)
    rotate_k = bool(rotate_k)
    if not q.is_cuda:
        raise _lib.LwmError("ringattention: tensors must live on an sm_90 GPU (no CPU fallback)")
    in_dtype = q.dtype
    if not (k.dtype == in_dtype and v.dtype == in_dtype and in_dtype in (torch.bfloat16, torch.float32)):
        raise TypeError("ringattention: q, k, v must all be bfloat16 or all float32 (fp32 logits and accumulation "
                        "are internal)")
    group, rank, world = _resolve_group(axis_name)
    native_f32 = in_dtype == torch.float32 and precision == "fp16" and (world == 1 or _transport(group) == "peer")
    B, Sq, H, D = q.shape
    causal, dropout = _check_blockwise_kwargs(blockwise_kwargs, Sq, k.shape[1], world)
    if rope is not None:
        to_bf16 = in_dtype == torch.float32 and not native_f32
        if to_bf16 or not (world == 1 or _peer_ready(q, k, causal, group, rank, world, layout, precision)):
            # bf16 operands from fp32 inputs (rotated straight into bf16: the same bits as rotating in fp32 and then
            # rounding), or the two-sided NCCL executor: the rotation is a pass of its own, then the plain op
            if rotate_k:
                q, k = _rope.apply_rotary_emb(q, k, freqs_cis, torch.bfloat16 if to_bf16 else in_dtype,
                                              position_ids=position_ids)
            else:
                q = _rope.rotate(q, freqs_cis, torch.bfloat16 if to_bf16 else in_dtype, position_ids=rope[0])
            rope = None
    if in_dtype == torch.float32 and not native_f32:
        # bf16 operand mode / NCCL transport: fp32 callers go through one rounding of q/k/v to bf16 (2^-9 relative)
        q, k, v = q.to(torch.bfloat16), k.to(torch.bfloat16), v.to(torch.bfloat16)
    bias = _prep_bias(attn_bias, B)
    seg = None
    if segment_ids is not None:
        seg = segment_ids.to(torch.int32).contiguous()
    _check_mask_extent(bias, seg, rank, world, Sq, k.shape[1])
    out = _RingAttnFn.apply(q.contiguous(), k.contiguous(), v.contiguous(), bias, seg, causal, axis_name, layout,
                            precision, *(rope or (None, None)), rotate_k, dropout)
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
             stream=None, scales=None, out_f32=None, tilemap=None, dropout=None):
    """scales: None (bf16 operands), or the device scales (sq, sk, sv) of fp16 operand copies q/k/v; out_f32 (fp16
    operands only): the un-rounded output, written on the last step. tilemap: None, or the forward map (tiles, counts)
    of step_tilemap for these arguments: the tile kernel then visits only the KV tiles in it (same results, bit for
    bit). dropout: None, or (seed, thr) of attention dropout, or (seed, thr, batch0) when q ... are rows
    batch0 .. batch0 + B - 1 of a larger batch (each batch row draws its own mask)."""
    B, Sq, H, D = q.shape
    sq, sk, sv = scales if scales is not None else (None, None, None)
    tiles, counts = tilemap if tilemap is not None else (None, None)
    _lib.call("lwm_attn_fwd_step", _lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(sq), _lib.ptr(sk), _lib.ptr(sv),
              _lib.ptr(out_f32), _lib.ptr(out), _lib.ptr(lse), _lib.ptr(acc_o), _lib.ptr(acc_m), _lib.ptr(acc_l), B, H,
              Sq, k.shape[1], D, int(q_pos0), int(k_pos0), int(bool(causal)), _lib.ptr(bias),
              0 if bias is None else bias.shape[1], _lib.ptr(seg), 0 if seg is None else seg.shape[1],
              1.0 / math.sqrt(D), int(first), int(last), _lib.ptr(tiles), _lib.ptr(counts), *_drop_args(dropout),
              _lib.stream_ptr(stream))


def bwd_prep(out, dout, delta, stream=None, scale_do=None):
    """delta = rowsum(out o dout): out fp32 or bf16; dout bf16, or its scaled fp16 copy with its device scale scale_do"""
    B, Sq, H, D = out.shape
    _lib.call("lwm_attn_bwd_prep", _lib.ptr(out), _dt(out), _lib.ptr(dout), _lib.ptr(scale_do), _lib.ptr(delta), B, H,
              Sq, D, _lib.stream_ptr(stream))


F16_P_BOOST_LOG2 = 14.0      # include/lwm_b200.h: LWM_ATTN_F16_P_BOOST_LOG2
LWM_REDUCE_MAX_SRCS = 16     # include/lwm_b200.h: sources per lwm_reduce_cast_f32 call


def lse_for_bwd(lse, stream=None, f16=False):
    """-lse*log2(e) (masked-level rows -> -inf), computed once per backward: what bwd_step takes as `lse`.
    f16=True: for the fp16-operand kernel, which keeps P^T * 2^14 (the +14 rides on this array)."""
    out = torch.empty_like(lse)
    _lib.call("lwm_attn_bwd_lse", _lib.ptr(lse), _lib.ptr(out), lse.numel(), F16_P_BOOST_LOG2 if f16 else 0.0,
              _lib.stream_ptr(stream))
    return out


def order_workspace(words, device):
    """the int32 workspace of an ordered dQ reduction (include/lwm_b200.h: lwm_attn_bwd_step's order_ws); the call
    zeroes it on its stream. Word 1 is the call's error flag."""
    return torch.empty(words, dtype=torch.int32, device=device)


def bwd_step(q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg, stream=None,
             scales=None, init=False, tilemap=None, dropout=None):
    """`lse` is the PRE-SCALED array returned by lse_for_bwd. scales: None (bf16 operands), or (sq, sk, sv, sdo) of
    fp16 operand copies q/k/v/dout. init=True: dk_acc/dv_acc rows are written, not accumulated.
    tilemap: None, or the backward map (tiles, counts) of step_tilemap for these arguments (dK, dV bit-identical; dQ
    up to the order of its reductions).
    Under torch.use_deterministic_algorithms(True) dQ is reduced in ascending key-tile order (an order_ws
    workspace): the same bits on every run. dropout: None, or the forward's (seed, thr)."""
    B, Sq, H, D = q.shape
    sq, sk, sv, sdo = scales if scales is not None else (None, None, None, None)
    tiles, counts = tilemap if tilemap is not None else (None, None)
    ws = None
    if torch.are_deterministic_algorithms_enabled():
        ws = order_workspace(2 + B * H * (Sq // 64) + (0 if tiles is None else tiles.numel()), q.device)
    _lib.call("lwm_attn_bwd_step", _lib.ptr(q), _lib.ptr(k), _lib.ptr(v), _lib.ptr(dout), _lib.ptr(sq), _lib.ptr(sk),
              _lib.ptr(sv), _lib.ptr(sdo), _lib.ptr(lse), _lib.ptr(delta), _lib.ptr(dq_acc), _lib.ptr(dk_acc),
              _lib.ptr(dv_acc), B, H, Sq, k.shape[1], D, int(q_pos0), int(k_pos0), int(bool(causal)), _lib.ptr(bias),
              0 if bias is None else bias.shape[1], _lib.ptr(seg), 0 if seg is None else seg.shape[1], 1.0 / math.sqrt(D),
              int(bool(init)), _lib.ptr(tiles), _lib.ptr(counts), _lib.ptr(ws), *_drop_args(dropout),
              _lib.stream_ptr(stream))


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


def _drop_args(dropout):
    """None, (seed, thr) or (seed, thr, batch0) -> the seed, drop_threshold and batch0 arguments of the step calls
    (drop_threshold 0: no dropout)"""
    if dropout is None:
        return 0, 0, 0
    seed, thr, batch0 = tuple(dropout) + (0,) * (3 - len(dropout))
    return int(seed), int(thr), int(batch0)


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

    def fwd_step(self, q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last, **kw):
        (q16, sq), (k16, sk), (v16, sv) = self._f16(q), self._f16(k), self._f16(v)
        o32 = None
        if last:
            o32 = torch.empty(out.shape, dtype=torch.float32, device=out.device)
            self.out_f32[out.data_ptr()] = o32
        mapped_fwd_step(q16, k16, v16, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last,
                        scales=(sq, sk, sv), out_f32=o32, **kw)

    @staticmethod
    def lse_for_bwd(lse):
        return lse_for_bwd(lse, f16=True)

    def bwd_step(self, q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg, **kw):
        (q16, sq), (k16, sk), (v16, sv), (d16, sd) = self._f16(q), self._f16(k), self._f16(v), self._f16(dout)
        mapped_bwd_step(q16, k16, v16, d16, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg,
                        scales=(sq, sk, sv, sd), **kw)


class DropoutOps:
    """The step functions of `ops` (any of the Ops classes here, or a CPU stand-in with the same `dropout` keyword)
    with attention dropout (seed, thr) applied in every fwd_step / bwd_step; everything else is ops' own. The ring
    executors pass each step its global q_pos0 / k_pos0, which is all the mask depends on."""

    def __init__(self, ops, dropout):
        self.ops, self.dropout = ops, dropout

    def __getattr__(self, name):
        return getattr(self.ops, name)

    def fwd_step(self, *args, batch0=0, **kw):
        """batch0: the global batch row of the step's batch row 0, for executors that launch a slice of the batch"""
        self.ops.fwd_step(*args, dropout=tuple(self.dropout[:2]) + (batch0,), **kw)

    def bwd_step(self, *args, batch0=0, **kw):
        self.ops.bwd_step(*args, dropout=tuple(self.dropout[:2]) + (batch0,), **kw)


def with_dropout(ops, dropout):
    """ops itself when dropout is None, else DropoutOps(ops, dropout)"""
    return ops if dropout is None else DropoutOps(ops, dropout)


def _f32_residuals(ops, res):
    """fp16 precision mode: the backward's delta = rowsum(dO o O) is taken from the un-rounded fp32 output."""
    if isinstance(ops, DropoutOps):
        ops = ops.ops
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
    def fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last, scales, out_f32,
                 **kw):
        mapped_fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last,
                        scales=scales, out_f32=out_f32, **kw)

    @staticmethod
    def bwd_prep(out, dout, sdo, delta):
        bwd_prep(out, dout, delta, scale_do=sdo)

    @staticmethod
    def lse_for_bwd(lse):
        return lse_for_bwd(lse, f16=True)

    @staticmethod
    def bwd_step(q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg, scales, init,
                 **kw):
        mapped_bwd_step(q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg,
                        scales=scales, init=init, **kw)

    @staticmethod
    def reduce_cast(srcs, dst):
        import ctypes
        arr = (ctypes.c_void_p * len(srcs))(*[t.data_ptr() for t in srcs])
        _lib.call("lwm_reduce_cast_f32", arr, len(srcs), _lib.ptr(dst), _dt(dst), dst.numel(), _lib.stream_ptr())

    cast = staticmethod(cast_f32_to_bf16)

    # -- the same passes over un-rotated q / k with the rotary embedding applied on the fly: x [..., H, 128]
    # (contiguous) with pos int32 [...] (contiguous, one position per row), inv_freq [64] of the RotaryTable
    _STAGE_DST = 2          # lwm_attn_stage_rope: scaled fp16

    @staticmethod
    def absmax_rope(x, bits, pos, inv_freq):
        _lib.call("lwm_attn_absmax_rope", _lib.ptr(x), _dt(x), _lib.ptr(pos), _lib.ptr(inv_freq), 1, pos.numel(),
                  x.shape[-2], _lib.ptr(bits), _lib.stream_ptr())

    @classmethod
    def scale_of_rope(cls, x, out, pos, inv_freq):
        """scale_of of rope(x)"""
        bits = torch.zeros(1, dtype=torch.int32, device=x.device)
        cls.absmax_rope(x, bits, pos, inv_freq)
        _lib.call("lwm_attn_scale_from_absmax", _lib.ptr(bits), 1, 1, _lib.ptr(out), _lib.stream_ptr())

    @classmethod
    def stage_rope(cls, x, dst, scale, pos, inv_freq):
        """stage of rope(x)"""
        _lib.call("lwm_attn_stage_rope", _lib.ptr(x), _dt(x), _lib.ptr(dst), cls._STAGE_DST, _lib.ptr(scale),
                  _lib.ptr(pos), _lib.ptr(inv_freq), 1, pos.numel(), x.shape[-2], _lib.stream_ptr())

    @staticmethod
    def reduce_cast_rope(srcs, dst, pos, inv_freq):
        """reduce_cast, then the conjugate rotation of the cast value, rounded again to dst's dtype"""
        import ctypes
        arr = (ctypes.c_void_p * len(srcs))(*[t.data_ptr() for t in srcs])
        _lib.call("lwm_reduce_cast_rope_f32", arr, len(srcs), _lib.ptr(dst), _dt(dst), _lib.ptr(pos),
                  _lib.ptr(inv_freq), 1, pos.numel(), dst.shape[-2], _lib.stream_ptr())

    @staticmethod
    def rope_conj(src, dst, pos, inv_freq):
        """dst = the conjugate rotation of src (a gradient w.r.t. rotated rows -> w.r.t. the un-rotated ones)"""
        _lib.call("lwm_attn_rope", _lib.ptr(src), None, _dt(src), _lib.ptr(dst), None, _dt(dst), _lib.ptr(pos),
                  _lib.ptr(inv_freq), 1, pos.numel(), src.shape[-2], 0, src.shape[-1], 1, _lib.stream_ptr())


class PeerOpsBf16(PeerOpsF16):
    """bf16 operand mode: staging is a plain copy (fp32 inputs are rounded to bf16 there), no scales."""
    op_dtype, op_itemsize, scaled = torch.bfloat16, 2, False
    _STAGE_DST = 1          # lwm_attn_stage_rope: bf16, the copy's rounding

    @staticmethod
    def stage(x, dst, scale):
        dst.copy_(x)

    @staticmethod
    def fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last, scales, out_f32,
                 **kw):
        mapped_fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last, **kw)
        if last and out_f32 is not None:
            out_f32.copy_(out)

    @staticmethod
    def lse_for_bwd(lse):
        return lse_for_bwd(lse, f16=False)

    @staticmethod
    def bwd_step(q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg, scales, init,
                 **kw):
        mapped_bwd_step(q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg, init=init,
                        **kw)


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


def _local_scales(ops, tensors, rope=None, n_rot=2):
    """single GPU: per-tensor scales from the local |max| (same kernels as the sharded exchange, world = 1).
    rope: None, or (positions, inv_freq): the first n_rot tensors (q, k) are scaled as rotated"""
    if not ops.scaled:
        return [None] * len(tensors)
    table = torch.zeros((1, 4), dtype=torch.int32, device=tensors[0].device)
    out = []
    for c, t in enumerate(tensors):
        if rope is not None and c < n_rot:
            ops.absmax_rope(t, table[0, c:c + 1], *rope)
        else:
            ops.absmax(t, table[0, c:c + 1])
        out.append(ops.make_scale(table, c))
    return out


def _stage_local(ops, x, scale, rope=None):
    """x's operand copy; rope: None, or (positions, inv_freq) to stage the rotation of x"""
    if rope is not None:
        y = torch.empty(x.shape, dtype=ops.op_dtype, device=x.device)
        ops.stage_rope(x, y, scale, *rope)
        return y
    if not ops.scaled and x.dtype == ops.op_dtype:
        return x
    y = torch.empty(x.shape, dtype=ops.op_dtype, device=x.device)
    ops.stage(x, y, scale)
    return y


def ring_forward(q, k, v, bias, seg, causal, group, rank, world, layout="auto", precision="bf16", rope=None,
                 rope_k=True, dropout=None):
    """-> (out, residuals). out is fp32 (un-rounded) for fp32 inputs, bf16 otherwise. world == 1 is the
    single-launch path (no carry buffers). rope: None, or (positions int32 [B,Sq], inv_freq): q (and k when rope_k) are
    un-rotated and are rotated while they are staged (one GPU and the peer-memory executor only). dropout: None, or
    (seed, thr) of attention dropout."""
    B, Sq, H, D = q.shape
    want_f32 = q.dtype == torch.float32
    if world == 1:
        ops = with_dropout(_peer_ops(precision), dropout)
        sq, sk, sv = _local_scales(ops, (q, k, v), rope, 2 if rope_k else 1)
        q16, k16, v16 = (_stage_local(ops, q, sq, rope), _stage_local(ops, k, sk, rope if rope_k else None),
                         _stage_local(ops, v, sv))
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
            return rp.run_forward(plan, q, k, v, bias, seg, causal, with_dropout(pops, dropout), tr, want_f32, rope,
                                  rope_k)
        if want_f32:        # the NCCL executor takes bf16 operands (documented in ringattention())
            out, res = ring_forward(q.to(torch.bfloat16), k.to(torch.bfloat16), v.to(torch.bfloat16), bias, seg, causal,
                                    group, rank, world, layout, precision, rope, dropout=dropout)
            return out.float(), res
    if rope is not None:
        raise _lib.LwmError("ring_forward: the rotary embedding is folded into the one-GPU and peer-memory paths only")
    ops = with_dropout(_ops_for(precision), dropout)
    plan = rs.make_plan(world, rank, Sq, k.shape[1], causal, lay, n_sub_first=rs.auto_sub(world, k.shape[1], lay))
    out, res = rx.run_forward(plan, q, k, v, bias, seg, causal, group, ops)
    return out, _f32_residuals(ops, res)


def ring_backward(res, k, v, dout, bias, seg, causal, group, rank, world, layout="auto", precision="bf16", rope=None,
                  rope_k=True, dropout=None):
    """rope, rope_k: as ring_forward's; dq (and dk when rope_k) are then the gradients w.r.t. the un-rotated q (and k).
    dropout: the forward's"""
    B, Sk, H, D = k.shape
    dev = k.device
    want_f32 = k.dtype == torch.float32
    if world == 1:
        ops = with_dropout(_peer_ops(precision), dropout)
        q16, out, lse = res["q_chunks"][0], res["out_chunks"][0], res["lse_chunks"][0]
        sq, sk, sv = res["scales"]
        Sq = q16.shape[1]
        sdo = _local_scales(ops, (dout,))[0]
        k16, v16 = _stage_local(ops, k, sk, rope if rope_k else None), _stage_local(ops, v, sv)
        d16 = _stage_local(ops, dout, sdo)
        delta = torch.empty((B, H, Sq), dtype=torch.float32, device=dev)
        ops.bwd_prep(out, d16, sdo, delta)
        nlse = ops.lse_for_bwd(lse)
        dq_acc = torch.zeros((B, Sq, H, D), dtype=torch.float32, device=dev)
        dk_acc = torch.empty((B, Sk, H, D), dtype=torch.float32, device=dev)     # written, not accumulated (init)
        dv_acc = torch.empty((B, Sk, H, D), dtype=torch.float32, device=dev)
        ops.bwd_step(q16, k16, v16, d16, nlse, delta, dq_acc, dk_acc, dv_acc, 0, 0, causal, bias, seg,
                     (sq, sk, sv, sdo), True)
        if rope is not None:
            # the final casts of dQ and dK carry the conjugate rotation (a single source: no sum; fp32 results are
            # rotated in place, so the rotation allocates nothing)
            if want_f32:
                dq, dk, dv = dq_acc, dk_acc, dv_acc
            else:
                dq, dk, dv = [torch.empty(t.shape, dtype=torch.bfloat16, device=dev) for t in (dq_acc, dk_acc, dv_acc)]
                cast_f32_to_bf16(dv_acc, dv)
                if not rope_k:
                    cast_f32_to_bf16(dk_acc, dk)
            ops.reduce_cast_rope([dq_acc], dq, *rope)
            if rope_k:
                ops.reduce_cast_rope([dk_acc], dk, *rope)
            return dq, dk, dv
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
        return rp.run_backward(plan, res, k, v, dout, bias, seg, causal, with_dropout(_peer_ops(precision), dropout),
                               rp.CudaPeerTransport.get(group, dev), want_f32, rope, rope_k)
    if rope is not None:
        raise _lib.LwmError("ring_backward: the rotary embedding is folded into the one-GPU and peer-memory paths only")
    if want_f32:            # forward fell back to the NCCL executor: bf16 operands in, fp32 gradients out
        dq, dk, dv = ring_backward(res, k.to(torch.bfloat16), v.to(torch.bfloat16), dout.to(torch.bfloat16), bias, seg,
                                   causal, group, rank, world, layout, precision, dropout=dropout)
        return dq.float(), dk.float(), dv.float()
    ops = with_dropout(_ops_for(precision), dropout)
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


def decode_partial(q, k, v, mask_u8, k_pos0, stream=None, rope=None):
    """This rank's partial over its KV shard with the GEMV kernel (bf16 or fp32 q/k/v, read as they are; or k / v
    the 8-bit cache, kv_cache.QuantizedKV, with bf16 or fp32 q: bit for bit the partial on the cache dequantized to q's
    dtype) -> (o_part [B*Q*H,128] fp32, ml_part [B*Q*H,2] fp32). rope: None, or (positions int32 [B,Q], inv_freq): q is
    un-rotated and the kernel rotates it as it loads it."""
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
    pos, inv_freq = rope if rope is not None else (None, None)
    q8 = k.dtype == torch.int8      # the 8-bit cache
    _lib.call("lwm_attn_decode_partial", _lib.ptr(q), _lib.ptr(k.data if q8 else k), _lib.ptr(v.data if q8 else v),
              _dt(q), _lib.ptr(k.exp if q8 else None), _lib.ptr(v.exp if q8 else None), _lib.ptr(mask_u8),
              _lib.ptr(o_part), _lib.ptr(ml_part), _lib.ptr(ws), B, H, Q, Sk, D, int(k_pos0), int(sb), int(sq), splits,
              1.0 / math.sqrt(D), _lib.ptr(pos), _lib.ptr(inv_freq), _lib.stream_ptr(stream))
    return o_part, ml_part


def decode_merge(o_parts, ml_parts, n_part, out_shape, dtype, with_lse=False):
    """merge n_part partials per row ([rows][n_part][128], [rows][n_part][2]) into the normalised output;
    with_lse: -> (out, lse [rows], natural log)"""
    out = torch.empty(out_shape, dtype=dtype, device=o_parts.device)
    rows = o_parts.shape[0]
    lse = torch.empty(rows, dtype=torch.float32, device=o_parts.device)
    _lib.call("lwm_attn_decode_merge", _lib.ptr(o_parts), _lib.ptr(ml_parts), n_part, _lib.ptr(out), _dt(out),
              _lib.ptr(lse), rows, _lib.stream_ptr())
    return (out, lse) if with_lse else out


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


def _scaled_f16_rope(x, pos, inv_freq):
    """_scaled_f16 of x rotated at pos [B,S] (rounded to x's dtype), without the rotated x in memory"""
    scale = torch.empty(1, dtype=torch.float32, device=x.device)
    PeerOpsF16.scale_of_rope(x, scale, pos, inv_freq)
    return _stage_local(PeerOpsF16, x, scale, (pos, inv_freq)), scale


def rope_rows(x, pos, inv_freq):
    """x [B,S,H,128] rotated at pos int32 [B,S], in x's dtype (lwm_attn_rope)"""
    B, S, H, D = x.shape
    y = torch.empty(x.shape, dtype=x.dtype, device=x.device)
    _lib.call("lwm_attn_rope", _lib.ptr(x), None, _dt(x), _lib.ptr(y), None, _dt(x), _lib.ptr(pos), _lib.ptr(inv_freq),
              B, S, H, 0, D, 0, _lib.stream_ptr())
    return y


def infer_partial(q, k, v, bits, row_any, staged=None):
    """This rank's partial with the tensor-core kernel: q [B,Q,H,128] against k/v [B,Sk,H,128] (bf16 or fp32, staged
    to scaled fp16 here), bits [B,Q,kw] / row_any [B,Q] (row_any over the whole ring) or None
    -> (o_part [B*Q*H,128], ml_part [B*Q*H,2]). staged: the caller's ((q16, sq), (k16, sk), (v16, sv)) of
    _scaled_f16, used instead of staging q, k, v again."""
    B, Q, H, D = q.shape
    Sk = k.shape[1]
    dev = q.device
    n_qt, n_kt = (Q + 127) // 128, (Sk + 127) // 128
    tiles = torch.empty(B, n_qt, n_kt, dtype=torch.int32, device=dev)
    counts = torch.empty(B, n_qt, dtype=torch.int32, device=dev)
    _lib.call("lwm_attn_infer_tilemap", _lib.ptr(bits), _lib.ptr(row_any), B, Q, Sk, _lib.ptr(tiles),
              _lib.ptr(counts), _lib.stream_ptr())
    if staged is None:
        staged = _scaled_f16(q), _scaled_f16(k), _scaled_f16(v)
    (q16, sq), (k16, sk), (v16, sv) = staged
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


def infer_backward(q16, k16, v16, do16, scales, lse, delta, bits, row_any):
    """One backward launch of the inference op over this rank's keys: q16 / do16 [B,Q,H,128], k16 / v16 [B,Sk,H,128]
    scaled fp16 copies, scales = (sq, sk, sv, sdo); lse [B,H,Q] (natural log, -inf for rows with no visible key),
    delta [B,H,Q] = rowsum(dO o O); bits [B,Q,kw] / row_any [B,Q] (over the whole ring) or None
    -> fp32 (dq [B,Q,H,128], dk, dv [B,Sk,H,128]). Under torch.use_deterministic_algorithms(True) dQ is reduced in
    ascending key-tile order, as in bwd_step."""
    B, Q, H, D = q16.shape
    Sk = k16.shape[1]
    dev = q16.device
    n_kt, Qp = (Sk + 127) // 128, (Q + 63) // 64 * 64
    tiles = torch.empty(B, n_kt, Qp // 64, dtype=torch.int32, device=dev)
    counts = torch.empty(B, n_kt, dtype=torch.int32, device=dev)
    _lib.call("lwm_attn_infer_bwd_tilemap", _lib.ptr(bits), _lib.ptr(row_any), B, Q, Sk, _lib.ptr(tiles),
              _lib.ptr(counts), _lib.stream_ptr())
    # lse / delta padded to whole 64-row tiles: the padding rows get P = 0
    lse_p = torch.full((B, H, Qp), -math.inf, dtype=torch.float32, device=dev)
    lse_p[..., :Q] = lse
    delta_p = torch.zeros((B, H, Qp), dtype=torch.float32, device=dev)
    delta_p[..., :Q] = delta
    nlse = lse_for_bwd(lse_p, f16=True)
    dq = torch.zeros((B, Q, H, D), dtype=torch.float32, device=dev)
    dk = torch.empty((B, Sk, H, D), dtype=torch.float32, device=dev)
    dv = torch.empty((B, Sk, H, D), dtype=torch.float32, device=dev)
    sq, sk, sv, sdo = scales
    ws = None
    if torch.are_deterministic_algorithms_enabled():
        ws = order_workspace(2 + B * H * (Qp // 64) + tiles.numel(), dev)
    _lib.call("lwm_attn_infer_bwd", _lib.ptr(q16), _lib.ptr(k16), _lib.ptr(v16), _lib.ptr(do16), _lib.ptr(sq),
              _lib.ptr(sk), _lib.ptr(sv), _lib.ptr(sdo), _lib.ptr(nlse), _lib.ptr(delta_p), _lib.ptr(bits),
              _lib.ptr(tiles), _lib.ptr(counts), _lib.ptr(dq), _lib.ptr(dk), _lib.ptr(dv), B, H, Q, Sk, D,
              1.0 / math.sqrt(D), _lib.ptr(ws), _lib.stream_ptr())
    return dq, dk, dv


class InferOps:
    """The kernels of the q-sharded protocol (_infer_sharded, _infer_sharded_bwd); tests substitute stand-ins."""
    mask_pack = staticmethod(mask_pack)
    merge = staticmethod(decode_merge)
    stage = staticmethod(_scaled_f16)
    backward = staticmethod(infer_backward)
    reduce_cast = staticmethod(PeerOpsF16.reduce_cast)
    # with the rotary embedding: (pos, inv_freq) follow the tensor they rotate
    stage_rope = staticmethod(_scaled_f16_rope)
    rope = staticmethod(rope_rows)
    reduce_cast_rope = staticmethod(PeerOpsF16.reduce_cast_rope)

    @staticmethod
    def partial_rope(q, k, v, mask, pos, inv_freq):
        """the GEMV partial of partial() with un-rotated q, rotated inside the kernel at pos [B,Q]"""
        return decode_partial(q, k, v, mask, 0, rope=(pos, inv_freq))

    @staticmethod
    def partial(q, k, v, mask, row_any, tensor_cores, staged=None):
        """mask: bits [B,Q,kw] when tensor_cores, else uint8 [B,Q,Sk] (or None); staged: see infer_partial"""
        if tensor_cores:
            return infer_partial(q, k, v, mask, row_any, staged)
        return decode_partial(q, k, v, mask, 0)

    @staticmethod
    def merge_lse(o, ml, n_part, out_shape):
        """-> (fp32 output, lse [rows], natural log)"""
        return decode_merge(o, ml, n_part, out_shape, torch.float32, with_lse=True)

    @staticmethod
    def stage_by(x, scale):
        """scaled fp16 copy of x with a given scale"""
        return _stage_local(PeerOpsF16, x, scale)

    @staticmethod
    def delta(o32, do16, sdo):
        """rowsum(dO o O) [B,H,Q] from the fp32 output and the staged dO"""
        B, Q, H, D = o32.shape
        d = torch.empty((B, H, Q), dtype=torch.float32, device=o32.device)
        PeerOpsF16.bwd_prep(o32, do16, sdo, d)
        return d

    @staticmethod
    def cast(x32, dtype):
        if dtype == torch.float32:
            return x32
        y = torch.empty(x32.shape, dtype=dtype, device=x32.device)
        cast_f32_to_bf16(x32, y)
        return y


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


class _LocalComm:
    """The collectives of a ring of one: the single-GPU backward runs the q-sharded backward with world = 1."""
    world = 1

    @staticmethod
    def all_gather(x):
        return x[None]

    @staticmethod
    def all_to_all(x):
        return x


def _return_partials(o, ml, comm, B, Ql, H, D):
    """partials of all world*Q_loc rows over my keys -> each owner's rows' partials, [B*Q_loc*H, world, D / 2]"""
    W = comm.world
    o = comm.all_to_all(o.view(B, W, Ql, H, D).transpose(0, 1))
    ml = comm.all_to_all(ml.view(B, W, Ql, H, 2).transpose(0, 1))
    o = o.permute(1, 2, 3, 0, 4).reshape(B * Ql * H, W, D)
    ml = ml.permute(1, 2, 3, 0, 4).reshape(B * Ql * H, W, 2)
    return o.contiguous(), ml.contiguous()


def _stage(ops, x, pos, inv_freq):
    """ops.stage of x, or of x rotated at pos when pos is given"""
    return ops.stage(x) if pos is None else ops.stage_rope(x, pos, inv_freq)


def _gemv_partial(ops, q, k, v, mask, pos_q, pos_k, inv_freq):
    """the GEMV partial; pos_q / pos_k: None, or the positions q / k are rotated at (k by a pass of its own first: a
    per-key rotation inside the kernel's loop would cost more than the pass)"""
    if pos_k is not None:
        k = ops.rope(k, pos_k, inv_freq)
    if pos_q is None:
        return ops.partial(q, k, v, mask, None, False)
    return ops.partial_rope(q, k, v, mask, pos_q, inv_freq)


def _infer_sharded(q, k, v, mask, comm, ops=InferOps, saved=None, rope=None):
    """q-sharded protocol (query length > 1 on a ring of comm.world ranks): q [B,Q_loc,H,D] and mask [Bm,1,Q_loc,K]
    are this rank's query rows, k/v [B,S_loc,H,D] its KV shard (K = world*S_loc). Each rank computes the partials of
    ALL world*Q_loc rows over its own keys, so K/V never move; per rank the traffic is world*Q_loc*H*D words of q and
    of partials plus Q_loc*K/8 bytes of mask. Returns this rank's [B,Q_loc,H,D] output.
    saved: None, or a dict that receives what _infer_sharded_bwd needs (the output is the same either way).
    rope: None, or (pos [B,Q_loc] of my query rows, pos_k [B,S_loc] of my keys or None, inv_freq): q (and k when pos_k
    is given) are un-rotated; the positions are all-gathered with q and every pass works on the rotated rows."""
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
    pq = pk = inv = None
    if rope is not None:
        pos, pk, inv = rope
        pq = comm.all_gather(pos).transpose(0, 1).reshape(B, Qg)
        if saved is not None:
            saved.update(pos_all=pq, pos_own=pos, **({} if pk is None else {"pos_k": pk}))
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
    if saved is None and rope is None:
        o, ml = ops.partial(q_all, k, v, m, row_any, tc)
    elif tc:
        staged = _stage(ops, q_all, pq, inv), _stage(ops, k, pk, inv), ops.stage(v)
        o, ml = ops.partial(q_all, k, v, m, row_any, tc, staged=staged)
        if saved is not None:
            saved.update(staged=staged, bits=m, row_any=row_any)
    else:
        # the backward recomputes the row statistics on tensor cores (_infer_sharded_bwd)
        o, ml = _gemv_partial(ops, q_all, k, v, m, pq, pk, inv)
        if saved is not None:
            saved.update(q_all=q_all, k=k, v=v, slabs=m)
    # 5. each owner gets its rows' partials back
    o, ml = _return_partials(o, ml, comm, B, Ql, H, D)
    # 6. merge the world partials
    out = ops.merge(o, ml, W, (B, Ql, H, D), q.dtype)
    if saved is not None and tc:
        # the fp32 output and lse of my rows, from a second merge of the same partials
        saved["o32"], saved["lse"] = ops.merge_lse(o, ml, W, (B, Ql, H, D))
    return out


def _infer_replicated(q, k, v, mask, rank, comm, ops=InferOps, rope=None):
    """Replicated protocol (one query row, the generation call, on a ring of comm.world ranks): q [B,1,H,D] and mask
    [Bm,1,1,K] are the same on every rank, k/v [B,S_loc,H,D] are this rank's KV shard (keys [rank*S_loc,
    (rank+1)*S_loc) of K). Each rank reduces its shard to an (o, max, sum) partial with the GEMV kernel, the partials
    (a few KB) are all-gathered rank-major and merged. Returns the [B,1,H,D] output, the same on every rank.
    rope: as _infer_sharded's; every rank rotates the same q at the same positions inside its GEMV."""
    B, Q, H, D = q.shape
    Sk = k.shape[1]
    m = None
    if mask is not None:
        m = mask[:, 0, :, rank * Sk:(rank + 1) * Sk].to(torch.uint8).expand(B, Q, Sk).contiguous()
    o, ml = _gemv_partial(ops, q, k, v, m, *(rope or (None, None, None)))
    o = comm.all_gather(o).transpose(0, 1).contiguous()           # [row][rank][D]
    ml = comm.all_gather(ml).transpose(0, 1).contiguous()
    return ops.merge(o, ml, comm.world, (B, Q, H, D), q.dtype)


def _row_stats_tc(q_all, k, v, slabs, comm, ops, pos_all=None, pos_k=None, inv_freq=None):
    """A forward that ran the GEMV kernel (world*Q_loc < INFER_MIN_Q): its uint8 mask slabs [B,Qg,S_loc] (or None)
    become bits, row_any is made global, and the fp32 output and lse of my rows are recomputed with one tensor-core
    partial and merge on the staged operands, so that the backward's P sums to one over each row. pos_all / pos_k: None,
    or the positions q_all / k are staged rotated at.
    -> (staged, bits, row_any, o32, lse)"""
    B, Qg, H, D = q_all.shape
    W = comm.world
    bits = row_any = None
    if slabs is not None:
        bits, any_loc = ops.mask_pack(slabs[:, None], B, 1, k.shape[1])
        bits = bits[0]
        row_any = comm.all_gather(any_loc).amax(0)
    staged = _stage(ops, q_all, pos_all, inv_freq), _stage(ops, k, pos_k, inv_freq), ops.stage(v)
    o, ml = ops.partial(q_all, k, v, bits, row_any, True, staged=staged)
    o, ml = _return_partials(o, ml, comm, B, Qg // W, H, D)
    o32, lse = ops.merge_lse(o, ml, W, (B, Qg // W, H, D))
    return staged, bits, row_any, o32, lse


def _infer_sharded_bwd(saved, dout, comm, ops=InferOps, inv_freq=None):
    """Backward of _infer_sharded (and, with world = 1, of the single-GPU op), mirroring its protocol: K and V never
    move. dout [B,Q_loc,H,D] is the gradient of this rank's rows; saved is what the forward recorded.
      1. all-gather dO; every rank stages all world*Q_loc rows with one shared scale;
      2. the owner computes delta = rowsum(dO o O) of its rows (its dO staged with that scale, its fp32 O);
      3. all-gather lse and delta;
      4. one backward launch of all rows against the local K/V: dK and dV come out complete on their owner;
      5. the fp32 dQ partials go back to the row owners (all_to_all), which sum them in rank order.
    Per rank the traffic is world*Q_loc*H*D words of dO and of fp32 dQ partials, plus world*Q_loc*H*2 floats of lse
    and delta. -> (dq, dk, dv) in dout's dtype.
    With the rotary embedding (saved "pos_own" / "pos_all", and "pos_k" when k was rotated too; inv_freq): the final
    casts of dQ (and dK) carry the conjugate rotation, so they are the gradients w.r.t. the un-rotated rows."""
    B, Ql, H, D = dout.shape
    W = comm.world
    Qg = W * Ql
    pos_own, pos_k = saved.get("pos_own"), saved.get("pos_k")
    if "o32" in saved:
        staged, bits, row_any, o32, lse = (saved[n] for n in ("staged", "bits", "row_any", "o32", "lse"))
    else:
        staged, bits, row_any, o32, lse = _row_stats_tc(saved["q_all"], saved["k"], saved["v"], saved["slabs"],
                                                        comm, ops, saved.get("pos_all"), pos_k, inv_freq)
    (q16, sq), (k16, sk), (v16, sv) = staged
    # 1.
    do_all = comm.all_gather(dout).transpose(0, 1).reshape(B, Qg, H, D)
    do16, sdo = ops.stage(do_all)
    # 2. (the owner's rows of do16, staged again from its own dout: the same values)
    delta = ops.delta(o32, ops.stage_by(dout, sdo), sdo)                         # [B,H,Ql]
    # 3.
    stats = torch.stack([lse.view(B, Ql, H).permute(0, 2, 1).to(delta.dtype), delta])
    stats = comm.all_gather(stats).permute(1, 2, 3, 0, 4).reshape(2, B, H, Qg)
    lse_all, delta_all = stats[0], stats[1]
    if row_any is not None:       # rows with no visible key over the whole ring contribute nothing
        lse_all = torch.where(row_any[:, None, :] != 0, lse_all, torch.full_like(lse_all, -math.inf))
    # 4.
    dq, dk, dv = ops.backward(q16, k16, v16, do16, (sq, sk, sv, sdo), lse_all, delta_all, bits, row_any)
    # 5.
    parts = comm.all_to_all(dq.view(B, W, Ql, H, D).transpose(0, 1))
    dq = torch.empty((B, Ql, H, D), dtype=dout.dtype, device=dout.device)
    srcs = [parts[r] for r in range(W)]
    while len(srcs) > LWM_REDUCE_MAX_SRCS:      # fold the first 16 in fp32, keep the rank order
        acc = torch.empty(srcs[0].shape, dtype=srcs[0].dtype, device=srcs[0].device)
        ops.reduce_cast(srcs[:LWM_REDUCE_MAX_SRCS], acc)
        srcs = [acc] + srcs[LWM_REDUCE_MAX_SRCS:]
    if pos_own is None:
        ops.reduce_cast([s.contiguous() for s in srcs], dq)
    else:
        ops.reduce_cast_rope([s.contiguous() for s in srcs], dq, pos_own, inv_freq)
    if pos_k is not None:       # (fp32: rotated in place)
        dk_out = dk if dout.dtype == torch.float32 else torch.empty(dk.shape, dtype=dout.dtype, device=dk.device)
        ops.reduce_cast_rope([dk], dk_out, pos_k, inv_freq)
        return dq, dk_out, ops.cast(dv, dout.dtype)
    return dq, ops.cast(dk, dout.dtype), ops.cast(dv, dout.dtype)


def ringattention_inference(q, k, v, attn_mask, axis_name="sp", *, freqs_cis=None, position_ids=None, rotate_k=True):
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
    entry in all of K_global averages V over all keys (the reference's finfo.min semantics).

    freqs_cis, position_ids, rotate_k: as on ringattention. Both None: q and k are already rotated (the reference call).
    Given: q is un-rotated and position_ids [B,Q_loc] are its rows' positions ([B,1], replicated, while generating);
      * rotate_k=False (decode and cached prefill): k is the rotated KV cache; only q is rotated, inside the GEMV kernel
        as it loads q, or inside the passes that stage q for the tensor cores (after the all-gather of q and its
        positions on a q-sharded ring);
      * rotate_k=True (no KV cache: q and k are the same rows, Q_loc == S_loc): k is rotated at the same positions, by a
        pass of its own before the GEMV kernel, or inside its staging for the tensor cores.
    Bit-identical to the call on apply_rotary_emb's rotated q (and k) under autograd (dQ up to the order of its fp32
    sums); dQ (and dK with rotate_k) are the gradients w.r.t. the un-rotated rows, and position_ids gets none.

    k, v may be the 8-bit cache (kv_cache.QuantizedKV, both or neither) with q bf16 or fp32, without gradient and with
    rotate_k=False when the rotary keywords are given. Below INFER_MIN_Q query rows (world * Q_loc on a q-sharded
    ring) the GEMV kernel reads it directly, bit for bit the call on the cache dequantized to q's dtype; from there on
    the shard is dequantized to q's dtype (exact; one transient copy) for the tensor-core path."""
    group, rank, world = _resolve_group(axis_name)
    B, Q, H, D = q.shape
    Sk = k.shape[1]
    rope = _rope.check_position_ids("ringattention_inference", freqs_cis, position_ids, (B, Q), q.device)
    quantized = _quantized_kv("ringattention_inference", q, k, v, rope is not None and bool(rotate_k))
    if rope is not None and rotate_k and Q != Sk:
        raise ValueError("ringattention_inference: rotate_k=True rotates q and k at the same positions, which needs "
                         "Q_loc == S_loc (got %d and %d); with a rotated KV cache pass rotate_k=False" % (Q, Sk))
    if not q.is_cuda:
        raise _lib.LwmError("ringattention_inference: tensors must live on an sm_90 GPU (no CPU fallback)")
    if not quantized:
        _check_infer_dtypes(q, k, v)
    elif (Q if world == 1 or Q == 1 else world * Q) >= INFER_MIN_Q:
        k, v = k.dequantize(q.dtype), v.dequantize(q.dtype)      # the tensor-core path (see the docstring)
    if attn_mask is not None:
        if attn_mask.dim() != 4 or attn_mask.shape[1] != 1 or attn_mask.shape[2] != Q or attn_mask.shape[0] not in (1, B):
            raise ValueError("attn_mask must be [B,1,Q,K_global] (lwm/llama.py:585-590)")
        if attn_mask.shape[-1] < (world if Q > 1 else rank + 1) * Sk:
            raise ValueError("attn_mask covers %d keys but the ring holds %d" % (attn_mask.shape[-1], world * Sk))
    q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
    rope_args = (None, None, True) if rope is None else (rope[0], rope[1], bool(rotate_k))
    if torch.is_grad_enabled() and (q.requires_grad or k.requires_grad or v.requires_grad):
        return _InferAttnFn.apply(q, k, v, attn_mask, axis_name, *rope_args)
    return _infer_forward(q, k, v, attn_mask, group, rank, world, rope=_infer_rope(*rope_args))


def _infer_rope(pos, inv_freq, rope_k):
    """-> None, or the (pos_q, pos_k or None, inv_freq) of _infer_sharded"""
    return None if pos is None else (pos, pos if rope_k else None, inv_freq)


def _infer_forward(q, k, v, attn_mask, group, rank, world, saved=None, rope=None):
    """the forward of ringattention_inference; saved: None, or a dict that receives what the backward needs (the
    output is bit-identical either way); rope: as _infer_sharded's"""
    B, Q, H, D = q.shape
    Sk = k.shape[1]
    if world > 1:
        if Q > 1:
            return _infer_sharded(q, k, v, attn_mask, TorchComm(group, world), saved=saved, rope=rope)
        return _infer_replicated(q, k, v, attn_mask, rank, TorchComm(group, world), rope=rope)
    pq, pk, inv = rope or (None, None, None)
    if saved is not None and rope is not None:
        saved.update(pos_all=pq, pos_own=pq, **({} if pk is None else {"pos_k": pk}))
    if Q >= INFER_MIN_Q:
        bits = row_any = None
        if attn_mask is not None:
            bits, row_any = mask_pack(attn_mask, B, 1, Sk)
            bits = bits[0]
        if saved is None and rope is None:
            o_part, ml_part = infer_partial(q, k, v, bits, row_any)
            return decode_merge(o_part, ml_part, 1, (B, Q, H, D), q.dtype)
        staged = _stage(InferOps, q, pq, inv), _stage(InferOps, k, pk, inv), _scaled_f16(v)
        o_part, ml_part = infer_partial(q, k, v, bits, row_any, staged)
        if saved is None:
            return decode_merge(o_part, ml_part, 1, (B, Q, H, D), q.dtype)
        out = decode_merge(o_part, ml_part, 1, (B, Q, H, D), q.dtype)
        o32, lse = decode_merge(o_part, ml_part, 1, (B, Q, H, D), torch.float32, with_lse=True)
        saved.update(staged=staged, bits=bits, row_any=row_any, o32=o32, lse=lse)
        return out
    mask = None
    if attn_mask is not None:
        mask = attn_mask.to(torch.uint8).expand(B, 1, Q, attn_mask.shape[-1]).contiguous()
    o_part, ml_part = _gemv_partial(InferOps, q, k, v, mask, pq, pk, inv)
    if saved is not None:
        # GEMV forward: the backward recomputes the row statistics on tensor cores (_row_stats_tc)
        saved.update(q_all=q, k=k, v=v, slabs=None if attn_mask is None else attn_mask[:, 0])
    return decode_merge(o_part, ml_part, 1, (B, Q, H, D), q.dtype)


_INFER_SAVED = ("bits", "row_any", "o32", "lse", "q_all", "k", "v", "slabs", "pos_all", "pos_own", "pos_k")


class _InferAttnFn(torch.autograd.Function):
    """ringattention_inference with a backward w.r.t. q, k, v (the mask gets none). Saves the staged fp16 operands
    with their scales, the fp32 output and lse of this rank's rows and the mask bits with row_any (tensor-core
    forward), or the operands and mask slabs (GEMV forward: the backward recomputes the row statistics); with the rotary
    embedding also the positions (the operands are the un-rotated ones)."""

    @staticmethod
    def forward(ctx, q, k, v, attn_mask, axis_name, rope_pos=None, inv_freq=None, rope_k=True):
        group, rank, world = _resolve_group(axis_name)
        saved = {}
        out = _infer_forward(q, k, v, attn_mask, group, rank, world, saved, _infer_rope(rope_pos, inv_freq, rope_k))
        ctx.axis_name, ctx.replicated = axis_name, world > 1 and q.shape[1] == 1
        ctx.inv_freq = inv_freq
        # a ring whose world*Q_loc rows run the GEMV kernel: not validated on real kernels yet (see DESIGN §3.6)
        ctx.small_ring = world > 1 and 1 < q.shape[1] and world * q.shape[1] < INFER_MIN_Q
        staged = saved.pop("staged", None)
        ctx.staged = staged is not None
        flat = [t for pair in staged for t in pair] if staged is not None else []
        ctx.keys = [n for n in _INFER_SAVED if n in saved]
        ctx.save_for_backward(*flat, *[saved[n] for n in ctx.keys])
        return out

    @staticmethod
    def backward(ctx, dout):
        if ctx.replicated:
            raise NotImplementedError("ringattention_inference: no backward for a single query row replicated along "
                                      "a ring of more than one rank (the generation call); shard the query rows instead")
        if ctx.small_ring:
            raise NotImplementedError("ringattention_inference: no backward on a ring with world * Q_loc < INFER_MIN_Q "
                                      "(%d) query rows yet" % INFER_MIN_Q)
        t = ctx.saved_tensors
        saved = {}
        if ctx.staged:
            saved["staged"] = (t[0], t[1]), (t[2], t[3]), (t[4], t[5])
            t = t[6:]
        saved.update(zip(ctx.keys, t))
        group, rank, world = _resolve_group(ctx.axis_name)
        comm = TorchComm(group, world) if world > 1 else _LocalComm()
        dq, dk, dv = _infer_sharded_bwd(saved, dout.contiguous(), comm, inv_freq=ctx.inv_freq)
        return dq, dk, dv, None, None, None, None, None
