"""Shared helpers for the parity tests (seeded inputs, error metrics)."""
import numpy as np
import torch


def rel_fro(x, ref):
    x = np.asarray(x, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.linalg.norm(x - ref) / max(np.linalg.norm(ref), 1e-30))


def make_qkv(B, Sq, Sk, H, D=128, seed=1234, device="cuda", n_extra=0):
    """N(0,1) generated in fp32 then rounded to bf16 (SURVEY.md §8d synthetic inputs)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    q = torch.randn(B, Sq, H, D, generator=g).to(torch.bfloat16)
    k = torch.randn(B, Sk, H, D, generator=g).to(torch.bfloat16)
    v = torch.randn(B, Sk, H, D, generator=g).to(torch.bfloat16)
    extra = [torch.randn(B, Sq, H, D, generator=g).to(torch.bfloat16) for _ in range(n_extra)]
    outs = [q, k, v] + extra
    return [t.to(device) for t in outs]


def to_np(t):
    return t.detach().float().cpu().numpy()


FOLDED_ENTRY_POINTS = ("lwm_attn_fwd_step", "lwm_attn_bwd_step", "lwm_attn_infer_bwd", "lwm_attn_decode_partial")


def with_options(name, args, ptr):
    """The arguments of a call row of one of FOLDED_ENTRY_POINTS with every option slot of that entry point turned on:
    dropout (seed 7, threshold 6554, batch0 0) in the training steps, an order_ws (ptr) in the backward ones, the 8-bit
    cache's k_exp / v_exp (ptr) in the decode. The argument checks of the row must give the same verdict with them."""
    a = list(args)
    if name == "lwm_attn_fwd_step":          # (..., tiles, tile_count, seed, drop_threshold, batch0, stream)
        a[29:32] = [7, 6554, 0]
    elif name == "lwm_attn_bwd_step":        # (..., tiles, tile_count, order_ws, seed, drop_threshold, batch0, stream)
        a[29:33] = [ptr, 7, 6554, 0]
    elif name == "lwm_attn_infer_bwd":       # (..., softmax_scale, order_ws, stream)
        a[-2] = ptr
    elif name == "lwm_attn_decode_partial":  # (q, k, v, dtype, k_exp, v_exp, ...)
        a[4:6] = [ptr, ptr]
    return tuple(a)


def abi_row_id(name, args):
    """Test id of a C-ABI call row: the entry point without `lwm_`, and for the attention passes whose options are
    nullable arguments, the operand mode the row selects (bf16 / f16 / f32, map: a block map, rope: the rotary
    embedding of q; for lwm_attn_bwd_prep the dtype is out's and f16 marks the scaled fp16 dout), then the options it
    turns on (ordered: an order_ws, drop: drop_threshold > 0, q8: the 8-bit cache's k_exp), so that every mode of one
    entry point has an id of its own."""
    given = [a is not None for a in args]
    dtype = {0: "f32", 1: "bf16"}
    if name in ("lwm_attn_fwd_step", "lwm_attn_bwd_step"):
        # (..., tiles, tile_count, [order_ws,] seed, drop_threshold, batch0, stream): the map is in slots 27 and 28
        scales = given[3:6] if name == "lwm_attn_fwd_step" else given[4:8]
        return (name[4:] + ("-f16" if any(scales) else "-bf16") + ("-map" if any(given[27:29]) else "")
                + ("-ordered" if name == "lwm_attn_bwd_step" and given[29] else "")
                + ("-drop" if args[-3] is not None and args[-3] > 0 else ""))
    if name == "lwm_attn_infer_bwd":         # (..., softmax_scale, order_ws, stream)
        return name[4:] + ("-ordered" if given[-2] else "")
    if name == "lwm_attn_bwd_prep":          # (out, out_dtype, dout, scale_do, ...)
        return name[4:] + "-" + dtype.get(args[1], "bad_dtype") + ("-f16" if given[3] else "")
    if name == "lwm_attn_decode_partial":    # (q, k, v, dtype, k_exp, v_exp, ..., position_ids, inv_freq, stream)
        return (name[4:] + "-" + dtype.get(args[3], "bad_dtype") + ("-rope" if any(given[-3:-1]) else "")
                + ("-q8" if given[4] else ""))
    if name == "lwm_attn_decode_merge":      # (o_parts, ml_parts, n_part, out, out_dtype, ...)
        return name[4:] + "-" + dtype.get(args[4], "bad_dtype")
    return name[4:]
