"""GPU tests of the `ringattention_inference` backward (attn_bwd_kernel's mask-bits mode): gradients against the float64
VJP over masks and shapes off the 64/128 grid, fully masked rows, exact power-of-two scaling of dO, bit-identical
forwards with and without requires_grad, agreement with `ringattention` on the same causal + padding problem, a 32K
causal problem, the q-sharded ring emulated with threads, and a model-level check through a `wq` projection."""
import math

import numpy as np
import pytest
import torch

from helpers import rel_fro, to_np
from infer_grad_model import attention_inference_vjp, bwd_tilemap_model, pack_bits
from thread_comm import run_ranks

pytestmark = pytest.mark.gpu

TOL = {torch.float32: 1e-3, torch.bfloat16: 3e-3}


def _qkv(B, Q, K, H, dtype, seed, mags=(1.0, 1.0, 1.0)):
    g = torch.Generator().manual_seed(seed)
    t = [torch.randn(B, n, H, 128, generator=g) * m for n, m in zip((Q, K, K), mags)]
    return [x.to(dtype).cuda() for x in t]


def _mask(kind, B, Q, K, seed):
    from lwm_b200.ringattention import causal_attention_mask, decode_attention_mask
    g = torch.Generator().manual_seed(seed)
    if kind == "none":
        return None
    if kind == "train":       # llama.py:580-592 without a cache: causal, left padding, packed segments
        assert Q == K
        pad = torch.ones(B, Q, dtype=torch.int32)
        pad[0, :min(Q - 1, 23)] = 0
        seg = (torch.arange(Q)[None, :] * 3 // max(Q, 1)).repeat(B, 1)
        return causal_attention_mask(pad, seg)
    if kind == "decode":
        pad = torch.ones(B, K, dtype=torch.int32)
        pad[0, :min(K - 1, 19)] = 0
        return decode_attention_mask(pad, Q, max(0, K - Q - 5), K)
    if kind == "blocks":
        nq, nk = (Q + 63) // 64, (K + 127) // 128
        kind_t = torch.randint(0, 3, (B, nq, nk), generator=g)
        rnd = torch.rand(B, Q, K, generator=g) < 0.5
        t = kind_t.repeat_interleave(64, 1).repeat_interleave(128, 2)[:, :Q, :K]
        m = torch.where(t == 0, torch.zeros_like(rnd), torch.where(t == 1, torch.ones_like(rnd), rnd))
        m[:, min(2, Q - 1)] = False
        return m[:, None]
    if kind == "broadcast":
        m = (torch.arange(K)[None, :] <= (torch.arange(Q) + K - Q)[:, None])[None, None].clone()
        m[..., Q // 2, :] = False
        return m
    raise ValueError(kind)


def _grads(q, k, v, mask, g):
    from lwm_b200.ringattention import ringattention_inference
    q, k, v = (x.detach().clone().requires_grad_() for x in (q, k, v))
    out = ringattention_inference(q, k, v, None if mask is None else mask.cuda())
    out.backward(g)
    torch.cuda.synchronize()
    return out.detach(), q.grad, k.grad, v.grad


def _ref(q, k, v, mask, g):
    B = q.shape[0]
    m = None if mask is None else np.broadcast_to(mask.numpy(), (B,) + tuple(mask.shape[1:]))
    return attention_inference_vjp(to_np(q), to_np(k), to_np(v), m, to_np(g))


def _check(grads, ref, dtype):
    for name, x, r in zip("qkv", grads, ref):
        assert x.dtype == dtype, name
        xn = to_np(x)
        assert np.isfinite(xn).all(), name
        if not r.any():
            # one visible key per row (K = 1): dq and dk vanish in exact arithmetic; here they are rounding residue
            # of dP - delta, far below the scale of dv
            assert np.abs(xn).max() <= 1e-5 * np.abs(ref[2]).max(), name
            continue
        assert rel_fro(xn, r) < TOL[dtype], (name, rel_fro(xn, r))


CASES = [(Q, K, kind) for Q in (1, 7, 8, 200, 1000) for K in (Q, Q + 77, 4096)
         for kind in ("decode", "blocks", "broadcast", "none")] + [(Q, Q, "train") for Q in (1, 7, 8, 200, 1000)]


@pytest.mark.parametrize("Q,K,kind", CASES)
def test_gradients_match_float64_vjp_fp32(Q, K, kind):
    B, H = 2, 2
    q, k, v = _qkv(B, Q, K, H, torch.float32, Q * 7 + K)
    g = torch.randn(B, Q, H, 128, generator=torch.Generator().manual_seed(K)).cuda()
    mask = _mask(kind, B, Q, K, Q + K)
    _, dq, dk, dv = _grads(q, k, v, mask, g)
    _check((dq, dk, dv), _ref(q, k, v, mask, g), torch.float32)


@pytest.mark.parametrize("Q,K,kind", [(7, 300, "decode"), (200, 4096, "blocks"), (1000, 1000, "train"),
                                      (8, 85, "broadcast"), (200, 277, "none")])
def test_gradients_match_float64_vjp_bf16(Q, K, kind):
    B, H = 2, 3
    q, k, v = _qkv(B, Q, K, H, torch.bfloat16, Q + K)
    g = torch.randn(B, Q, H, 128, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16).cuda()
    mask = _mask(kind, B, Q, K, K)
    _, dq, dk, dv = _grads(q, k, v, mask, g)
    _check((dq, dk, dv), _ref(q, k, v, mask, g), torch.bfloat16)


@pytest.mark.parametrize("Q", [5, 200])
def test_fully_masked_rows_contribute_exactly_nothing(Q):
    K = 333
    q, k, v = _qkv(1, Q, K, 2, torch.float32, 1)
    g = torch.randn(1, Q, 2, 128, generator=torch.Generator().manual_seed(2)).cuda() * 5
    mask = torch.rand(1, 1, Q, K, generator=torch.Generator().manual_seed(3)) < 0.7
    dead = [1, Q - 1] + ([150, 151] if Q > 151 else [])
    mask[..., dead, :] = False
    _, dq, dk, dv = _grads(q, k, v, mask, g)
    assert not dq[:, dead].any()
    keep = [r for r in range(Q) if r not in dead]
    rq, rk, rv = attention_inference_vjp(to_np(q)[:, keep], to_np(k), to_np(v), mask.numpy()[:, :, keep],
                                         to_np(g)[:, keep])
    assert rel_fro(to_np(dk), rk) < 1e-3 and rel_fro(to_np(dv), rv) < 1e-3
    assert rel_fro(to_np(dq)[:, keep], rq) < 1e-3


@pytest.mark.parametrize("Q,K", [(3, 500), (300, 1000)])
@pytest.mark.parametrize("e", [-20, 7, 30])
def test_scaling_dout_scales_the_gradients_exactly(Q, K, e):
    """dO -> 2^k dO gives exactly 2^k dk and 2^k dv, and 2^k dq up to the order of its fp32 atomic sums"""
    q, k, v = _qkv(1, Q, K, 2, torch.float32, 3)
    g = torch.randn(1, Q, 2, 128, generator=torch.Generator().manual_seed(4)).cuda()
    mask = _mask("blocks", 1, Q, K, 4)
    a = _grads(q, k, v, mask, g)[1:]
    b = _grads(q, k, v, mask, g * 2.0 ** e)[1:]
    for name, x, y in zip("qkv", a, b):
        assert torch.isfinite(y).all(), name
        if name == "q":     # dq is summed with atomics in no fixed order: equal up to that order
            assert rel_fro(to_np(y), to_np(x * 2.0 ** e)) < 1e-6
        else:
            assert torch.equal(y, x * 2.0 ** e), name


@pytest.mark.parametrize("Q,K", [(3, 300), (200, 1077)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_forward_is_bit_identical_with_and_without_grad(Q, K, dtype):
    from lwm_b200.ringattention import ringattention_inference
    q, k, v = _qkv(2, Q, K, 3, dtype, 5)
    mask = _mask("decode", 2, Q, K, 0).cuda()
    plain = ringattention_inference(q, k, v, mask)
    out = ringattention_inference(q.requires_grad_(), k, v, mask)
    torch.cuda.synchronize()
    assert out.requires_grad
    assert torch.equal(out.detach(), plain)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_agrees_with_ringattention_on_causal_padding(dtype):
    """the same problem through the training op (call-site bias, causal) and through this op (dense mask)"""
    from lwm_b200.ringattention import attention_bias_from_mask, causal_attention_mask, ringattention
    B, S, H = 2, 512, 2
    q, k, v = _qkv(B, S, S, H, dtype, 21)
    g = torch.randn(B, S, H, 128, generator=torch.Generator().manual_seed(22)).to(dtype).cuda()
    pad = torch.ones(B, S, dtype=torch.int32)
    pad[0, :37] = 0
    pad[1, :200] = 0
    mask = causal_attention_mask(pad)
    out_i, *gi = _grads(q, k, v, mask, g)
    qt, kt, vt = (x.detach().clone().requires_grad_() for x in (q, k, v))
    out_t = ringattention(qt, kt, vt, attention_bias_from_mask(pad.cuda(), dtype), None,
                          blockwise_kwargs=dict(causal_block_size=1))
    out_t.backward(g)
    torch.cuda.synchronize()
    live = mask[:, 0].any(-1)                     # [B,S]: the left-padded rows see no key
    for b in range(B):
        assert rel_fro(to_np(out_i[b][live[b]]), to_np(out_t[b][live[b]])) < 2 * TOL[dtype]
    ref = _ref(q, k, v, mask, g)
    for name, x, y, r in zip("qkv", gi, (qt.grad, kt.grad, vt.grad), ref):
        assert rel_fro(to_np(x), r) < TOL[dtype], name
        assert rel_fro(to_np(y), r) < TOL[dtype], name
        assert rel_fro(to_np(x), to_np(y)) < 2 * TOL[dtype], name


def test_large_causal_problem():
    """causal S = 32768: every dk and dv row and dq on sampled rows against float64 (row-blockwise, as
    oracle/attn_rows.py, on the GPU so that all 32K rows fit in the time budget)"""
    from oracle.attn_rows import attention_rows, sample_rows
    S, H = 32768, 1
    q, k, v = _qkv(1, S, S, H, torch.bfloat16, 11)
    g = torch.randn(1, S, H, 128, generator=torch.Generator().manual_seed(12)).to(torch.bfloat16).cuda()
    mask = torch.ones(S, S, dtype=torch.bool, device="cuda").tril_()[None, None]
    _, dq, dk, dv = _grads(q, k, v, mask, g)
    q64, k64, v64, g64 = (x[0, :, 0].double() for x in (q, k, v, g))
    rdk = torch.zeros_like(k64)
    rdv = torch.zeros_like(v64)
    kpos = torch.arange(S, device="cuda")
    for a in range(0, S, 2048):
        b = a + 2048
        s = (q64[a:b] @ k64.T) / math.sqrt(128)
        s = s.masked_fill(torch.arange(a, b, device="cuda")[:, None] < kpos[None, :], -math.inf)
        p = torch.softmax(s, dim=1)
        o = p @ v64
        ds = p * ((g64[a:b] @ v64.T) - (g64[a:b] * o).sum(1, keepdim=True))
        rdk += (ds.T @ q64[a:b]) / math.sqrt(128)
        rdv += p.T @ g64[a:b]
    assert rel_fro(to_np(dk[0, :, 0]), rdk.cpu().numpy()) < 3e-3
    assert rel_fro(to_np(dv[0, :, 0]), rdv.cpu().numpy()) < 3e-3
    rows = torch.as_tensor(sample_rows(S, per_tile=1, tile=1024, tail=16))
    ref = attention_rows(q[0, rows.cuda(), 0].cpu(), rows, k[0, :, 0].cpu(), v[0, :, 0].cpu(),
                         do_rows=g[0, rows.cuda(), 0].cpu())
    assert rel_fro(to_np(dq[0, rows.cuda(), 0]), ref["dq"].numpy()) < 3e-3


def test_backward_map_kernel_matches_model():
    from lwm_b200 import _lib
    from lwm_b200.ringattention import mask_pack
    for Q, Sk, kind in [(200, 333, "blocks"), (65, 129, "decode"), (1000, 4096, "broadcast"), (7, 77, "none")]:
        B = 2
        mask = _mask(kind, B, Q, Sk, 1)
        bits = row_any = None
        if mask is not None:
            bits, row_any = mask_pack(mask.cuda(), B, 1, Sk)
            bits = bits[0]
        n_kt, n_qt = (Sk + 127) // 128, (Q + 63) // 64
        tiles = torch.empty(B, n_kt, n_qt, dtype=torch.int32, device="cuda")
        counts = torch.empty(B, n_kt, dtype=torch.int32, device="cuda")
        _lib.call("lwm_attn_infer_bwd_tilemap", _lib.ptr(bits), _lib.ptr(row_any), B, Q, Sk, _lib.ptr(tiles),
                  _lib.ptr(counts), _lib.stream_ptr())
        torch.cuda.synchronize()
        vis = None if mask is None else np.broadcast_to(mask.numpy()[:, 0], (B, Q, Sk))
        model = bwd_tilemap_model(None if vis is None else pack_bits(vis, Sk),
                                  None if vis is None else vis.any(-1), B, Q, Sk)
        got = [[tiles[b, kt, :counts[b, kt]].tolist() for kt in range(n_kt)] for b in range(B)]
        assert got == model, (Q, Sk, kind)
        if bits is not None:
            assert np.array_equal(bits.cpu().numpy(), pack_bits(vis, Sk))


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("Ql,dtype", [(37, torch.float32), (130, torch.float32), (37, torch.bfloat16)])
def test_q_sharded_backward_emulated_with_threads(world, Ql, dtype):
    """the protocol through a thread fake comm and the real kernels, against the single-rank gradients of the
    concatenated problem"""
    from lwm_b200 import ringattention as ra
    B, H, Sl = 2, 3, 300
    Q, K = world * Ql, world * Sl
    parts = [_qkv(B, Ql, Sl, H, torch.float32, 100 + r, mags=(2.0 ** -r, 2.0 ** -r, 2.0 ** (3 * r)))
             for r in range(world)]
    q = torch.cat([p[0] for p in parts], 1).to(dtype)
    k = torch.cat([p[1] for p in parts], 1).to(dtype)
    v = torch.cat([p[2] for p in parts], 1).to(dtype)
    g = torch.randn(B, Q, H, 128, generator=torch.Generator().manual_seed(7)).to(dtype).cuda()
    mask = _mask("decode", B, Q, K, 0)
    mask[..., min(1, Q - 1), :] = False
    mask_d = mask.cuda()

    def rank_fn(r, comm):
        rows, keys = slice(r * Ql, (r + 1) * Ql), slice(r * Sl, (r + 1) * Sl)
        args = (q[:, rows].contiguous(), k[:, keys].contiguous(), v[:, keys].contiguous(),
                mask_d[:, :, rows].contiguous(), comm)
        saved = {}
        out = ra._infer_sharded(*args, saved=saved)
        plain = ra._infer_sharded(*args)
        return torch.equal(out, plain), ra._infer_sharded_bwd(saved, g[:, rows].contiguous(), comm)
    res = run_ranks(world, rank_fn)
    torch.cuda.synchronize()
    assert all(r[0] for r in res)            # the recording forward returns the same output, bit for bit
    dq = torch.cat([r[1][0] for r in res], 1)
    dk = torch.cat([r[1][1] for r in res], 1)
    dv = torch.cat([r[1][2] for r in res], 1)
    _, sq, sk, sv = _grads(q, k, v, mask, g)
    ref = _ref(q, k, v, mask, g)
    for name, x, y, r in zip("qkv", (dq, dk, dv), (sq, sk, sv), ref):
        assert x.dtype == dtype
        assert rel_fro(to_np(x), r) < TOL[dtype], (name, rel_fro(to_np(x), r))
        assert rel_fro(to_np(x), to_np(y)) < TOL[dtype], name


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_projection_weights_get_gradients_through_the_op(dtype):
    """wq -> ringattention_inference -> wo inside a model: wq.weight.grad exists and matches float64 autograd"""
    from lwm_b200.ringattention import causal_attention_mask, ringattention_inference
    torch.manual_seed(0)
    B, S, H, E = 2, 100, 2, 64
    x = torch.randn(B, S, E)
    k = torch.randn(B, S, H, 128)
    v = torch.randn(B, S, H, 128)
    seg = (torch.arange(S)[None] // 40).repeat(B, 1)
    mask = causal_attention_mask(torch.ones(B, S, dtype=torch.int32), seg)   # every row sees itself
    wq = torch.nn.Linear(E, H * 128, bias=False)
    wo = torch.nn.Linear(H * 128, E, bias=False)
    wq_d, wo_d = (torch.nn.Linear(E, H * 128, bias=False).cuda().to(dtype), torch.nn.Linear(H * 128, E, bias=False).cuda().to(dtype))
    with torch.no_grad():
        wq_d.weight.copy_(wq.weight)
        wo_d.weight.copy_(wo.weight)
    q = wq_d(x.cuda().to(dtype)).view(B, S, H, 128)
    out = ringattention_inference(q, k.cuda().to(dtype), v.cuda().to(dtype), mask.cuda())
    wo_d(out.reshape(B, S, H * 128)).square().mean().backward()
    torch.cuda.synchronize()
    assert wq_d.weight.grad is not None
    # float64 autograd of the same composition, on the same (rounded) values
    r64 = lambda t: t.detach().to(dtype).double()      # noqa: E731
    wq64 = r64(wq.weight).requires_grad_()
    q64 = (r64(x) @ wq64.T).view(B, S, H, 128)
    s = torch.einsum("bqhd,bkhd->bhqk", q64, r64(k)) / math.sqrt(128)
    s = torch.where(mask, s, torch.tensor(torch.finfo(torch.bfloat16).min, dtype=torch.float64))
    o64 = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), r64(v))
    (o64.reshape(B, S, H * 128) @ r64(wo.weight).T).square().mean().backward()
    assert rel_fro(to_np(wq_d.weight.grad), wq64.grad.numpy()) < 2 * TOL[dtype]
