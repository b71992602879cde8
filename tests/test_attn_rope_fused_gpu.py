"""The rotary embedding folded into `ringattention`'s operand passes (freqs_cis=, position_ids=), on an H100.

Contract: the fused op is bit-identical to the composition
    ringattention(*apply_rotary_emb(q, k, freqs_cis, q.dtype, position_ids=pos), v, ...)
under autograd: out, dK and dV are torch.equal; dQ may differ by the order of the backward kernel's fp32 dQ reductions,
which already differs between two runs of one build, so it is held to the larger of a small bound and twice the
composition's own run-to-run spread.

  * kernels: lwm_attn_absmax_rope / lwm_attn_stage_rope / lwm_reduce_cast_rope_f32 against lwm_attn_rope followed by
    the plain pass, bit for bit;
  * the op on one GPU over dtypes, precision modes, batch, length, theta, position offsets near 2^20 and four masks,
    plus one case per dtype against the float64 oracles;
  * the peer-memory executor with the real kernels on an emulated ring (tests/peer_emulation.py), world 2, 4 and 8."""
import ctypes
import threading

import numpy as np
import pytest
import torch

from helpers import rel_fro, to_np

pytestmark = pytest.mark.gpu
KW = dict(axis_name="sp", blockwise_kwargs=dict(causal_block_size=1))
TOL_DQ = {torch.float32: 1e-5, torch.bfloat16: 4e-3}     # relative Frobenius, dQ fused vs composition
D = 128


def _table(theta, max_position):
    from lwm_b200.rope import precompute_freqs_cis
    return precompute_freqs_cis(D, max_position, theta)


def _rope(x, pos, table, out_dtype, conj=False):
    """lwm_attn_rope on one tensor (xk absent)"""
    from lwm_b200 import _lib
    B, S, H, _ = x.shape
    y = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    p = pos.to(torch.int32).contiguous()
    dt = {torch.float32: 0, torch.bfloat16: 1}
    _lib.call("lwm_attn_rope", _lib.ptr(x.contiguous()), None, dt[x.dtype], _lib.ptr(y), None, dt[out_dtype],
              _lib.ptr(p), _lib.ptr(table.inv_freq), B, S, H, 0, D, int(conj), _lib.stream_ptr())
    return y


# ------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------
KERNEL_CASES = [(1, 1, 1, 1e4, 0), (2, 37, 3, 1e4, 0), (1, 129, 32, 1e7, 1000), (3, 61, 4, 5e7, (1 << 20) - 61),
                (2, 1023, 2, 5e7, 1 << 19)]


def _kernel_inputs(B, S, H, theta, off, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, S, H, D, generator=g) * 3.0).to(dtype).cuda()
    pos = (off + torch.randperm(S, generator=g)[None].repeat(B, 1)
           + torch.arange(B)[:, None] % 2).to(torch.int32).cuda()
    table = _table(theta, off + S + 2)
    return x, pos, table


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("B,S,H,theta,off", KERNEL_CASES)
def test_rotating_absmax_and_stage_equal_rope_then_the_plain_pass(B, S, H, theta, off, dtype):
    from lwm_b200.ringattention import PeerOpsBf16, PeerOpsF16
    x, pos, table = _kernel_inputs(B, S, H, theta, off, dtype, 11 + S)
    y = _rope(x, pos, table, dtype)
    bits_ref = torch.zeros(1, dtype=torch.int32, device="cuda")
    bits = torch.zeros(1, dtype=torch.int32, device="cuda")
    PeerOpsF16.absmax(y, bits_ref)
    PeerOpsF16.absmax_rope(x, bits, pos, table.inv_freq)
    assert int(bits) == int(bits_ref) != 0
    for scale_exp in (-3, 0, 5):
        scale = torch.full((1,), 2.0 ** scale_exp, device="cuda")
        a, b = torch.empty(x.shape, dtype=torch.float16, device="cuda"), torch.empty(x.shape, dtype=torch.float16, device="cuda")
        PeerOpsF16.stage(y, a, scale)
        PeerOpsF16.stage_rope(x, b, scale, pos, table.inv_freq)
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    a, b = torch.empty(x.shape, dtype=torch.bfloat16, device="cuda"), torch.empty(x.shape, dtype=torch.bfloat16, device="cuda")
    PeerOpsBf16.stage(y, a, None)
    PeerOpsBf16.stage_rope(x, b, None, pos, table.inv_freq)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    s_ref, s = torch.empty(1, device="cuda"), torch.empty(1, device="cuda")
    PeerOpsF16.scale_of(y, s_ref)
    PeerOpsF16.scale_of_rope(x, s, pos, table.inv_freq)
    assert torch.equal(s, s_ref)


@pytest.mark.parametrize("n_src", [1, 2, 3, 7, 16])
@pytest.mark.parametrize("dst_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("B,S,H,theta,off", KERNEL_CASES)
def test_conjugate_reduce_cast_equals_reduce_cast_then_conjugate_rope(B, S, H, theta, off, dst_dtype, n_src):
    from lwm_b200 import _lib
    from lwm_b200.ringattention import PeerOpsF16
    g = torch.Generator().manual_seed(n_src * 100 + S)
    srcs = [(torch.randn(B, S, H, D, generator=g) * 2.0 ** (3 * i - 10)).cuda() for i in range(n_src)]
    _, pos, table = _kernel_inputs(B, S, H, theta, off, torch.float32, 7 + S)
    cast = torch.empty(srcs[0].shape, dtype=dst_dtype, device="cuda")
    PeerOpsF16.reduce_cast(srcs, cast)
    want = _rope(cast, pos, table, dst_dtype, conj=True)
    got = torch.empty(srcs[0].shape, dtype=dst_dtype, device="cuda")
    arr = (ctypes.c_void_p * n_src)(*[t.data_ptr() for t in srcs])
    p = pos.contiguous()
    _lib.call("lwm_reduce_cast_rope_f32", arr, n_src, _lib.ptr(got), int(dst_dtype == torch.bfloat16), _lib.ptr(p),
              _lib.ptr(table.inv_freq), B, S, H, _lib.stream_ptr())
    assert torch.equal(got.view(torch.int16 if dst_dtype == torch.bfloat16 else torch.int32),
                       want.view(torch.int16 if dst_dtype == torch.bfloat16 else torch.int32))


# ------------------------------------------------------------------------------------------------
# the op on one GPU
# ------------------------------------------------------------------------------------------------
MASKS = ("none", "zero_bias", "left_pad", "packed")


def _problem(B, S, H, dtype, mask, offset, seed):
    """q, k, v, dO, bias, seg, position_ids for one of the four call patterns"""
    from lwm_b200.ringattention import attention_bias_from_mask
    g = torch.Generator().manual_seed(seed)
    q, k, v, do = [torch.randn(B, S, H, D, generator=g).to(dtype).cuda() for _ in range(4)]
    pos = torch.arange(S)[None].repeat(B, 1) + offset
    bias = seg = None
    if mask == "zero_bias":
        bias = attention_bias_from_mask(torch.ones(B, S, device="cuda"), torch.float32 if dtype == torch.float32 else torch.bfloat16)
    elif mask == "left_pad":
        am = torch.ones(B, S, dtype=torch.int64)
        for b in range(B):
            am[b, :(S // 3 + 7 * b) % S] = 0
        bias = attention_bias_from_mask(am.cuda(), torch.float32 if dtype == torch.float32 else torch.bfloat16)
        p = am.cumsum(-1) - 1            # lwm/llama.py:1123; the padding rows (-1 there) get position 0
        pos = torch.where(am > 0, p + offset, torch.zeros_like(p))
    elif mask == "packed":
        seg = torch.zeros(B, S, dtype=torch.int32)
        pos = torch.zeros(B, S, dtype=torch.int64)
        for b in range(B):
            cuts = sorted({0, S} | set(torch.randint(1, S, (3 + b,), generator=g).tolist()))
            for i, (a, e) in enumerate(zip(cuts[:-1], cuts[1:])):
                seg[b, a:e] = i
                pos[b, a:e] = torch.arange(e - a) + offset
        seg = seg.cuda()
    return q, k, v, do, bias, seg, pos.cuda()


def _run(q, k, v, do, bias, seg, pos, table, precision, fused):
    from lwm_b200.rope import apply_rotary_emb
    from lwm_b200.ringattention import ringattention
    q, k, v = [t.detach().clone().requires_grad_(True) for t in (q, k, v)]
    if fused:
        out = ringattention(q, k, v, bias, seg, precision=precision, freqs_cis=table, position_ids=pos, **KW)
    else:
        out = ringattention(*apply_rotary_emb(q, k, table, q.dtype, position_ids=pos), v, bias, seg,
                            precision=precision, **KW)
    out.backward(do)
    return out.detach(), q.grad, k.grad, v.grad


def _assert_fused_matches(args, table, precision, dtype):
    ref = _run(*args, table, precision, False)
    ref2 = _run(*args, table, precision, False)
    got = _run(*args, table, precision, True)
    names = ("out", "dq", "dk", "dv")
    for n, a, b in zip(names, got, ref):
        assert a.dtype == dtype and a.shape == b.shape, n
        if n != "dq":
            assert torch.equal(a, b), "%s differs: max |diff| %.3e" % (n, float((a.float() - b.float()).abs().max()))
    spread = rel_fro(to_np(ref2[1]), to_np(ref[1]))
    err = rel_fro(to_np(got[1]), to_np(ref[1]))
    assert err <= max(TOL_DQ[dtype], 2 * spread), (err, spread)
    return got


OP_CASES = [(1, 128, 1e4, 0), (2, 128, 5e7, (1 << 20) - 128 - 5), (2, 1024, 1e7, (1 << 20) - 1024 - 3),
            (1, 1024, 1e4, 17), (1, 4096, 5e7, (1 << 20) - 4096 - 1), (2, 4096, 1e4, 0)]


@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("B,S,theta,offset", OP_CASES)
@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_fused_op_is_the_composition_on_one_gpu(dtype, precision, B, S, theta, offset, mask):
    H = 2
    args = _problem(B, S, H, dtype, mask, offset, seed=S + B + len(mask))
    table = _table(theta, (1 << 20) + 16)
    _assert_fused_matches(args, table, precision, dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_fused_op_is_the_composition_at_32k(dtype):
    args = _problem(1, 32768, 2, dtype, "zero_bias", (1 << 20) - 32768 - 9, seed=3)
    _assert_fused_matches(args, _table(5e7, (1 << 20) + 16), "fp16", dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_fused_op_against_the_float64_oracles(dtype):
    """oracle/rope.py (the reference's rotation, rounded to the input dtype as llama.py:519 does) then
    oracle/attn_dense.py in float64; the gradients w.r.t. the un-rotated q / k are the conjugate rotations of the dense
    gradients. Bounds: 1e-3 for fp32 results; 3e-3 for bf16 results (their own rounding), as for the op without the
    rotation, except 4e-3 for bf16 dQ and dK, which are rounded twice, before and after the conjugate rotation, exactly
    as the composition with apply_rotary_emb rounds them."""
    from oracle.attn_dense import attention_dense, attention_dense_grads
    from oracle.rope import precompute_freqs_cis, rope_reference
    B, S, H, theta = 2, 512, 2, 1e4
    q, k, v, do, bias, seg, pos = _problem(B, S, H, dtype, "packed", 100, seed=9)
    table = _table(theta, 4096)
    out, dq, dk, dv = _run(q, k, v, do, bias, seg, pos, table, "fp16", True)
    pn = to_np(pos).astype(np.int64)
    qr, kr = rope_reference(to_np(q).astype(np.float32), to_np(k).astype(np.float32), pn, theta, 4096)
    if dtype == torch.bfloat16:
        qr, kr = [torch.from_numpy(x).to(dtype).double().numpy() for x in (qr, kr)]
    n = [x.astype(np.float64) for x in (qr, kr, to_np(v), to_np(do))]
    kw = dict(causal=True, segment_ids=to_np(seg))
    ref = attention_dense(*n[:3], **kw)
    gq, gk, gv = attention_dense_grads(*n, **kw)
    f = precompute_freqs_cis(D, 4096, theta)[pn].astype(np.complex128)[:, :, None, :]     # [B,S,1,64]

    def unrotate(g):
        gc = g[..., 0::2] + 1j * g[..., 1::2]
        y = gc * np.conj(f)
        return np.stack((y.real, y.imag), axis=-1).reshape(g.shape)

    f32 = dtype == torch.float32
    for name, got, want, tol in (("out", out, ref, 1e-3 if f32 else 3e-3), ("dq", dq, unrotate(gq), 1e-3 if f32 else 4e-3),
                                 ("dk", dk, unrotate(gk), 1e-3 if f32 else 4e-3), ("dv", dv, gv, 1e-3 if f32 else 3e-3)):
        err = rel_fro(to_np(got), want)
        print("%s %s rel err %.2e (bound %.0e)" % (dtype, name, err, tol))
        assert err < tol, name


# ------------------------------------------------------------------------------------------------
# the peer-memory executor on an emulated ring
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world,layout", [(2, "contiguous"), (2, "zigzag"), (4, "contiguous"), (4, "zigzag"),
                                          (8, "contiguous"), (8, "zigzag")])
def test_fused_peer_ring_is_the_composition(world, layout):
    from lwm_b200 import ring_peer as rp, ring_schedule as rs
    from lwm_b200.ringattention import PeerOpsBf16, PeerOpsF16
    from peer_emulation import EmuTransport, EmuWorld
    B, H, Sl = 2, 2, 256
    S = world * Sl
    dev = torch.device("cuda", 0)
    table = _table(5e7, (1 << 20) + 16)
    passes = []
    for prec in ("fp16", "bf16"):
        for dt in (torch.float32, torch.bfloat16):
            for mask in ("zero_bias", "packed"):
                q, k, v, do, bias, seg, pos = _problem(B, S, H, dt, mask, (1 << 20) - S - 3, seed=world + len(mask))
                if bias is not None:
                    bias = bias.reshape(B, S).float().contiguous()
                passes.append((prec, dt, (q, k, v, do, bias, seg, pos)))
    emu = EmuWorld(world, device=dev)
    results, fails = {}, []

    def worker(rank):
        try:
            torch.cuda.set_device(dev)
            assert torch.cuda.current_stream(dev) == torch.cuda.default_stream(dev)
            tr = EmuTransport(emu, rank)
            plan = rs.make_peer_plan(world, rank, Sl, Sl, True, layout)
            sl = slice(rank * Sl, (rank + 1) * Sl)
            mine = []
            for prec, dt, (q, k, v, do, bias, seg, pos) in passes:
                ops = PeerOpsF16 if prec == "fp16" else PeerOpsBf16
                want_f32 = dt == torch.float32
                ql, kl, vl, dl = [t[:, sl].contiguous() for t in (q, k, v, do)]
                pl = pos[:, sl].to(torch.int32).contiguous()
                # fused
                out, res = rp.run_forward(plan, ql, kl, vl, bias, seg, True, ops, tr, want_f32, (pl, table.inv_freq))
                dq, dk, dv = rp.run_backward(plan, res, kl, vl, dl, bias, seg, True, ops, tr, want_f32,
                                             (pl, table.inv_freq))
                fused = (out, dq, dk, dv)
                # composition: rotate, plain executor, conjugate rotation of dQ and dK in the input dtype
                qr, kr = _rope(ql, pl, table, dt), _rope(kl, pl, table, dt)
                out, res = rp.run_forward(plan, qr, kr, vl, bias, seg, True, ops, tr, want_f32)
                dqr, dkr, dv = rp.run_backward(plan, res, kr, vl, dl, bias, seg, True, ops, tr, want_f32)
                comp = (out, _rope(dqr, pl, table, dt, conj=True), _rope(dkr, pl, table, dt, conj=True), dv)
                mine.append((fused, comp))
            torch.cuda.synchronize()
            results[rank] = mine
        except BaseException:   # noqa: BLE001  (reported by the main thread)
            import traceback
            fails.append((rank, traceback.format_exc()))
            emu.barrier.abort()

    ts = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    torch.cuda.synchronize()
    assert not any(t.is_alive() for t in ts), "rank threads did not finish"
    assert not fails, fails[0][1]
    for r in range(world):
        for i, (fused, comp) in enumerate(results[r]):
            prec, dt = passes[i][0], passes[i][1]
            for n, a, b in zip(("out", "dq", "dk", "dv"), fused, comp):
                assert a.dtype == dt, (r, i, n)
                if n == "dq":
                    err = rel_fro(to_np(a), to_np(b))
                    assert err <= TOL_DQ[dt], (r, i, prec, dt, err)
                else:
                    assert torch.equal(a, b), (r, i, prec, dt, n, float((a.float() - b.float()).abs().max()))
