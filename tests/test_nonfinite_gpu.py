"""NaN and infinite inputs to the attention op (one GPU, the peer ring, ringattention_inference) and to the VQGAN fp16
planes. Every power-of-two operand scale comes from the largest FINITE |x| of its tensor, so a bad element can only
reach the results that read it.

Method: every case runs a clean input X and a dirty input X', X with one element replaced by NaN, +inf or -inf. In X
that element is 0 and not the tensor's |max|, so both runs have the same scales. Outside the results that can depend on
the element the two runs agree bit for bit (dQ, summed with fp32 atomics, within 1e-5 of its slice's max|dQ|); inside,
the dirty run is compared with the float64 oracle on X' (oracle.attn_dense.attention_visible): wherever the oracle is
non-finite the kernel is too, and wherever both are finite they agree within TOL. The tile kernels, like the
reference's blockwise einsum, multiply a masked P = 0 with the whole tile, so 0 * inf = NaN may reach other rows of a
tile that reads the element; the sets below are therefore written at tile granularity (128 keys per K tile, 128 query
rows per forward Q tile, 64 per backward Q tile), per (b, h):

  bad element in       bit-identical to the clean run                                   must be non-finite
  q row i              out / lse of rows != i; dK / dV of K tiles that i's Q tile       out row i
                       never visits; dQ rows != i (tolerance)
  k row j              out / lse of rows that cannot see j; dQ rows whose Q tile never   rows with a +inf / NaN logit
                       visits j's K tile (tolerance)
  v row j, column d    out columns != d, and column d of rows whose Q tile never visits  column d of rows that see j
                       j's K tile; lse; dV; dQ as for k
  dO row i, column d   dQ rows != i (tolerance); dK / dV of K tiles that i's Q tile      dQ row i, dV column d of the
                       never visits; dV columns != d                                    keys i sees

and every other (b, h) slice is bit-identical in every case. A row that meets a NaN or a +inf logit returns lse = -inf
(its l is NaN) and a non-finite output; a row that meets a -inf logit drops that key. The backward treats an lse = -inf
row like a row that sees no key: P = 0 at its finite logits, so it adds nothing to dV there, where the oracle's P is
NaN (its dQ and, through delta, the dK of the tiles it visits are still NaN). The "non-finite where the oracle is"
check therefore covers out in every case and the gradients for a bad dO. The bf16 operand mode and the GEMV
decode kernel apply no scale and pass these tests without the finite-maximum rule; the other cases lost whole
tensors to it before (one NaN in q set every logit of every row, head and batch entry to 0)."""
import threading

import numpy as np
import pytest
import torch

from helpers import rel_fro, to_np
from nonfinite_checks import (BAD_B, BAD_COL, BAD_H, BADS, D, DTYPES, SL_RING, TOL, _bits, _check, _check_other_slices,
                              _dq_close, _ring_inputs, _same_sets)

pytestmark = pytest.mark.gpu

LSE_TOL = 2e-3


# ------------------------------------------------------------------------------------------------ 1. staging kernels
def _dt(x):
    return 0 if x.dtype == torch.float32 else 1


def _absmax_bits(x):
    from lwm_b200 import _lib
    bits = torch.zeros(1, dtype=torch.int32, device=x.device)
    _lib.call("lwm_attn_absmax", _lib.ptr(x), _dt(x), x.numel(), _lib.ptr(bits), _lib.stream_ptr())
    return bits


def _absmax_scale(x):
    from lwm_b200 import _lib
    ws = torch.empty(1, dtype=torch.int32, device=x.device)
    s = torch.empty(1, dtype=torch.float32, device=x.device)
    _lib.call("lwm_attn_absmax_scale", _lib.ptr(x), _dt(x), x.numel(), _lib.ptr(ws), _lib.ptr(s), _lib.stream_ptr())
    return s


def _scale_from(bits):
    from lwm_b200 import _lib
    s = torch.empty(1, dtype=torch.float32, device=bits.device)
    _lib.call("lwm_attn_scale_from_absmax", _lib.ptr(bits), bits.numel(), 1, _lib.ptr(s), _lib.stream_ptr())
    return s


def _to_f16_scaled(x, s):
    from lwm_b200 import _lib
    y = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    _lib.call("lwm_attn_to_f16_scaled", _lib.ptr(x), _dt(x), _lib.ptr(y), _lib.ptr(s), x.numel(), _lib.stream_ptr())
    return y


def _rope_args(x):
    from lwm_b200.rope import precompute_freqs_cis
    B, S = x.shape[:2]
    pos = (torch.arange(S, dtype=torch.int32)[None, :] * 3 + 17 * torch.arange(B, dtype=torch.int32)[:, None])
    return pos.contiguous().to(x.device), precompute_freqs_cis(D, 4096).inv_freq


def _scale_rope(x):
    from lwm_b200.ringattention import PeerOpsF16
    s = torch.empty(1, dtype=torch.float32, device=x.device)
    PeerOpsF16.scale_of_rope(x, s, *_rope_args(x))
    return s


def _stage_rope(x, s):
    from lwm_b200.ringattention import PeerOpsF16
    y = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    PeerOpsF16.stage_rope(x, y, s, *_rope_args(x))
    return y


def _bits_rope(x):
    from lwm_b200.ringattention import PeerOpsF16
    bits = torch.zeros(1, dtype=torch.int32, device=x.device)
    PeerOpsF16.absmax_rope(x, bits, *_rope_args(x))
    return bits


def _model_scale(x):
    """the documented rule: 2^(e-12), e the exponent of the largest finite |x| (clamped at -114); 1 without one"""
    a = np.abs(to_np(x).astype(np.float64)).ravel()
    a = a[np.isfinite(a) & (a > 0)]
    if a.size == 0:
        return 1.0
    e = max(int(np.frexp(a.max())[1]) - 1, -114)
    return 2.0 ** (e - 12)


def _f16_bits(y):
    return y.view(torch.int16).cpu().numpy()


def _assert_staged(clean16, dirty16, flat_idx, bad):
    c, d = _f16_bits(clean16).ravel(), _f16_bits(dirty16).ravel()
    diff = np.nonzero(c != d)[0]
    assert set(diff.tolist()) <= {flat_idx}, diff[:8]
    v = np.float16(d[flat_idx:flat_idx + 1].view(np.float16)[0])
    if np.isnan(bad):
        assert np.isnan(v)
    else:
        assert v == bad                                   # +-inf, with its sign


SHAPE = (2, 64, 2, D)
N_EL = int(np.prod(SHAPE))
WHERE = {"first": 1, "middle": N_EL // 2 + 2, "last": N_EL - 1}   # in the first, a middle and the last 16-byte vector


@pytest.mark.parametrize("bad", list(BADS))
@pytest.mark.parametrize("where", list(WHERE))
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_staging_kernels_skip_the_bad_element(dtype, where, bad):
    from lwm_b200 import ringattention as ra
    g = torch.Generator().manual_seed(3)
    idx, val = WHERE[where], BADS[bad]
    x = (torch.randn(SHAPE, generator=g) * 3.0).to(DTYPES[dtype])
    x.view(-1)[idx] = 0
    x = x.cuda()
    xd = x.clone()
    xd.view(-1)[idx] = val
    want = _model_scale(x)
    assert _absmax_bits(xd).item() == _absmax_bits(x).item()
    s, sd = _absmax_scale(x), _absmax_scale(xd)
    assert s.item() == sd.item() == want
    # the ring's form: every shard's bit pattern in one table, one scale for all of them
    table = torch.cat([_absmax_bits(xd), _absmax_bits(x * 0.25)])
    assert _scale_from(table).item() == want
    _assert_staged(_to_f16_scaled(x, s), _to_f16_scaled(xd, sd), idx, val)
    if dtype == "bf16":
        (c16, cs), (d16, ds) = ra.to_f16(x), ra.to_f16(xd)
        assert cs[0].item() == ds[0].item() == want
        _assert_staged(c16, d16, idx, val)
    # the rotating passes: the element's rotation pair is all the bad value can reach
    assert _bits_rope(xd).item() == _bits_rope(x).item()
    sr, srd = _scale_rope(x), _scale_rope(xd)
    assert sr.item() == srd.item()
    c, d = _f16_bits(_stage_rope(x, sr)).ravel(), _f16_bits(_stage_rope(xd, srd)).ravel()
    diff = np.nonzero(c != d)[0]
    assert idx in diff.tolist() and len(diff) <= 2 and np.all(diff // D == idx // D)
    assert not np.isfinite(d[diff].view(np.float16)).any()


@pytest.mark.parametrize("bad", list(BADS) + ["zero"])
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_no_finite_nonzero_element_gives_scale_one(dtype, bad):
    from lwm_b200 import ringattention as ra
    x = torch.zeros(SHAPE, dtype=DTYPES[dtype], device="cuda")
    if bad != "zero":
        x.view(-1)[WHERE["middle"]] = BADS[bad]
        x.view(-1)[WHERE["last"]] = BADS[bad]
    assert _absmax_scale(x).item() == 1.0
    assert _scale_rope(x).item() == 1.0
    if dtype == "bf16":
        x16, s = ra.to_f16(x)
        assert s[0].item() == 1.0
        assert np.array_equal(np.isnan(x16.float().cpu().numpy()), np.isnan(x.float().cpu().numpy()))


def _edge(case):
    """a finite tensor at an edge of the scale rule"""
    g = torch.Generator().manual_seed(5)
    base = torch.randn(SHAPE, generator=g)
    if case == "bf16-max":
        x = base.to(torch.bfloat16)
        x.view(-1)[77] = torch.finfo(torch.bfloat16).max
    elif case == "fp32-max":
        x = base.clone()
        x.view(-1)[77] = torch.finfo(torch.float32).max
    elif case == "bf16-subnormal":            # every element a bf16 subnormal: |max| < 2^-126, below the -114 clamp
        mant = torch.randint(0, 0x80, SHAPE, generator=g, dtype=torch.int16)
        sign = torch.randint(0, 2, SHAPE, generator=g, dtype=torch.int16) << 15
        x = (mant | sign).view(torch.bfloat16)
    elif case == "bf16-tiny-normal":          # normal bf16 around 2^-120: still below the clamp
        x = (base * 2.0 ** -122).to(torch.bfloat16)
    elif case == "fp32-subnormal":
        x = (torch.randint(0, 1 << 23, SHAPE, generator=g, dtype=torch.int32)).view(torch.float32) * torch.sign(base)
    elif case.startswith("pow2"):             # |max| exactly a power of two, or the largest value below it
        x = (base * 0.5).clamp(-1.0, 1.0)
        x.view(-1)[77] = 32.0 if case == "pow2" else 32.0 * (1 - 2.0 ** -24)
        x = x.to(torch.bfloat16) if case == "pow2-bf16" else x
    else:
        raise ValueError(case)
    return x.cuda()


@pytest.mark.parametrize("case", ["bf16-max", "fp32-max", "bf16-subnormal", "bf16-tiny-normal", "fp32-subnormal",
                                  "pow2", "pow2-below", "pow2-bf16"])
def test_scale_rule_at_its_finite_edges(case):
    """scale and staged copy against a numpy model of the rule: 2^(e-12), e clamped at -114, x16 = fp16(x / scale)"""
    from lwm_b200 import ringattention as ra
    x = _edge(case)
    want = _model_scale(x)
    s = _absmax_scale(x)
    assert s.item() == want, (s.item(), want)
    ref16 = (to_np(x).astype(np.float64) / want).astype(np.float16)
    assert np.isfinite(ref16).all()
    assert np.array_equal(_f16_bits(_to_f16_scaled(x, s)), ref16.view(np.int16))
    if x.dtype == torch.bfloat16:
        x16, s2 = ra.to_f16(x)
        assert s2[0].item() == want
        assert np.array_equal(_f16_bits(x16), ref16.view(np.int16))


# ------------------------------------------------------------------------------------------------ 2. ringattention, one GPU
B_PUB, S_PUB, H_PUB = 2, 512, 3
BAD_ROW = 300
PAD = (29, 17)
_CLEAN = {}


def _pub_inputs(dtype):
    from oracle.attn_dense import finfo_min
    g = torch.Generator().manual_seed(11)
    q, k, v, do = [torch.randn(B_PUB, S_PUB, H_PUB, D, generator=g) for _ in range(4)]
    for t in (q, k, v, do):
        t[BAD_B, BAD_ROW, BAD_H, BAD_COL] = 0
    bias = torch.zeros(B_PUB, 1, 1, S_PUB)
    seg = torch.zeros(B_PUB, S_PUB, dtype=torch.int32)
    for b, n in enumerate(PAD):
        bias[b, ..., :n] = finfo_min("bf16")
        do[b, :n] = 0                                  # padded rows: zero upstream gradient, as in every LWM use
        seg[b, 180 + 40 * b:] = 1                      # two segments (row 300 of batch 1 sees keys 220..300)
    return [t.to(DTYPES[dtype]).cuda() for t in (q, k, v, do)], bias.cuda(), seg.cuda()


def _pub_run(q, k, v, do, bias, seg, precision, rope=None):
    from lwm_b200 import ringattention as ra
    from lwm_b200.rope import apply_rotary_emb, precompute_freqs_cis
    kw = dict(axis_name="sp", blockwise_kwargs=dict(causal_block_size=1), precision=precision)
    q, k, v = [t.detach().clone().requires_grad_(True) for t in (q, k, v)]
    lse = None
    if rope is None:
        out = ra.ringattention(q, k, v, bias, seg, **kw)
        with torch.no_grad():
            lse = ra.ring_forward(q, k, v, ra._prep_bias(bias, B_PUB), seg, True, None, 0, 1,
                                  precision=precision)[1]["lse_chunks"][0]
    else:
        table = precompute_freqs_cis(D, 4096)
        pos = (torch.arange(S_PUB)[None, :] + 7 * torch.arange(B_PUB)[:, None]).cuda()
        if rope == "fused":
            out = ra.ringattention(q, k, v, bias, seg, freqs_cis=table, position_ids=pos, **kw)
        else:
            out = ra.ringattention(*apply_rotary_emb(q, k, table, q.dtype, position_ids=pos), v, bias, seg, **kw)
    out.backward(do)
    torch.cuda.synchronize()
    res = dict(out=to_np(out), dq=to_np(q.grad), dk=to_np(k.grad), dv=to_np(v.grad))
    if lse is not None:
        res["lse"] = to_np(lse)
    return res


def _dirty(tensors, which, bad):
    names = ("q", "k", "v", "do")
    out = list(tensors)
    t = out[names.index(which)].clone()
    t[BAD_B, BAD_ROW, BAD_H, BAD_COL] = BADS[bad]
    out[names.index(which)] = t
    return out


@pytest.mark.parametrize("bad", list(BADS))
@pytest.mark.parametrize("which", ["q", "k", "v", "do"])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("precision", ["fp16", "bf16"])
def test_ringattention_one_gpu(precision, dtype, which, bad):
    from oracle.attn_dense import attention_visible, visible_pairs
    (q, k, v, do), bias, seg = _pub_inputs(dtype)
    key = (precision, dtype, None)
    if key not in _CLEAN:
        _CLEAN[key] = _pub_run(q, k, v, do, bias, seg, precision)
    clean = _CLEAN[key]
    qd, kd, vd, dod = _dirty((q, k, v, do), which, bad)
    dirty = _pub_run(qd, kd, vd, dod, bias, seg, precision)
    vis = visible_pairs(B_PUB, S_PUB, S_PUB, attn_bias=bias.reshape(B_PUB, S_PUB).cpu().numpy(),
                        segment_ids=seg.cpu().numpy())
    sl = lambda t: to_np(t)[BAD_B:BAD_B + 1, :, BAD_H:BAD_H + 1]   # noqa: E731
    out, lse, dq, dk, dv = attention_visible(sl(qd), sl(kd), sl(vd), vis[BAD_B:BAD_B + 1], sl(dod))
    ref = dict(out=out[0, :, 0], lse=lse[0, 0], dq=dq[0, :, 0], dk=dk[0, :, 0], dv=dv[0, :, 0])
    if which != "do":
        assert not np.isfinite(ref["out"]).all()         # the bad element does reach the oracle's output
    same = _same_sets(which, BAD_ROW, BAD_COL, vis[BAD_B, 0], S_PUB, S_PUB)
    bf16 = dtype == "bf16"
    for name in ("out", "dq", "dk", "dv"):
        if same[name] is None:
            continue
        _check_other_slices(name, clean[name], dirty[name], BAD_B, BAD_H, tol_dq=name == "dq", bf16=bf16)
        _check(name, clean[name][BAD_B, :, BAD_H], dirty[name][BAD_B, :, BAD_H], ref[name], same[name],
               TOL[precision], same_tol=name == "dq", bf16=bf16, strict=name == "out" or which == "do")
    if same["lse"] is not None:
        c, d, r, s = clean["lse"], dirty["lse"], ref["lse"], same["lse"]
        other = np.ones(c.shape, bool)
        other[BAD_B, BAD_H] = False
        assert np.array_equal(_bits(c[other]), _bits(d[other]))
        c, d = c[BAD_B, BAD_H], d[BAD_B, BAD_H]
        assert np.array_equal(_bits(c[s]), _bits(d[s]))
        reach = ~s
        assert np.all(d[reach & ~np.isfinite(r)] == -np.inf)          # a NaN / +inf-logit row: lse = -inf
        fin = reach & np.isfinite(r) & (np.arange(S_PUB) >= PAD[BAD_B])
        assert np.abs(d[fin] - r[fin]).max(initial=0.0) < LSE_TOL


def _nan_equal(a, b):
    return np.array_equal(np.isfinite(a), np.isfinite(b)) and np.array_equal(a[np.isfinite(a)], b[np.isfinite(b)]) \
        and np.array_equal(np.isnan(a), np.isnan(b))


@pytest.mark.parametrize("bad", list(BADS))
@pytest.mark.parametrize("which", ["q", "k"])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("precision", ["fp16", "bf16"])
def test_ringattention_one_gpu_rope(precision, dtype, which, bad):
    """the freqs_cis= / position_ids= path: the same reach as the plain op, and the same results as the composition
    ringattention(*apply_rotary_emb(q, k, ...), v, ...) on the dirty input, non-finite entries included"""
    from oracle.attn_dense import visible_pairs
    (q, k, v, do), bias, seg = _pub_inputs(dtype)
    key = (precision, dtype, "fused")
    if key not in _CLEAN:
        _CLEAN[key] = _pub_run(q, k, v, do, bias, seg, precision, "fused")
    clean = _CLEAN[key]
    args = _dirty((q, k, v, do), which, bad)
    dirty = _pub_run(*args, bias, seg, precision, "fused")
    comp = _pub_run(*args, bias, seg, precision, "composed")
    vis = visible_pairs(B_PUB, S_PUB, S_PUB, attn_bias=bias.reshape(B_PUB, S_PUB).cpu().numpy(),
                        segment_ids=seg.cpu().numpy())
    same = _same_sets(which, BAD_ROW, BAD_COL, vis[BAD_B, 0], S_PUB, S_PUB)
    for name in ("out", "dq", "dk", "dv"):
        _check_other_slices(name, clean[name], dirty[name], BAD_B, BAD_H, tol_dq=name == "dq", bf16=dtype == "bf16")
        c, d, r = clean[name][BAD_B, :, BAD_H], dirty[name][BAD_B, :, BAD_H], comp[name][BAD_B, :, BAD_H]
        s = np.broadcast_to(same[name], d.shape)
        if name == "dq":
            assert _dq_close(c[s], d[s], dtype == "bf16")
            assert np.array_equal(np.isfinite(d), np.isfinite(r))
            fin = np.isfinite(d)
            assert rel_fro(d[fin], r[fin]) < (1e-5 if dtype == "fp32" else 4e-3)
        else:
            assert np.array_equal(_bits(c[s]), _bits(d[s])), name
            assert _nan_equal(dirty[name], comp[name]), name
    if which == "q":
        assert not np.isfinite(dirty["out"][BAD_B, BAD_ROW, BAD_H]).all()


# ------------------------------------------------------------------------------------------------ 3. the peer ring
_RING_CLEAN = {}


def _ring_run(world, tensors, precision, dtype):
    """the peer executor with the real kernels, `world` rank threads on one GPU (tests/peer_emulation.py)"""
    from lwm_b200 import ring_peer as rp, ring_schedule as rs
    from lwm_b200.ringattention import PeerOpsBf16, PeerOpsF16
    from peer_emulation import EmuTransport, EmuWorld
    dev = torch.device("cuda", 0)
    emu = EmuWorld(world, device=dev)
    results, fails = {}, []
    ops = PeerOpsF16 if precision == "fp16" else PeerOpsBf16
    want_f32 = dtype == "fp32"

    def worker(rank):
        try:
            torch.cuda.set_device(dev)
            tr = EmuTransport(emu, rank)
            plan = rs.make_peer_plan(world, rank, SL_RING, SL_RING, True, "zigzag")
            sl = slice(rank * SL_RING, (rank + 1) * SL_RING)
            ql, kl, vl, dl = [t[:, sl].to(dev).contiguous() for t in tensors]
            out, res = rp.run_forward(plan, ql, kl, vl, None, None, True, ops, tr, want_f32)
            dq, dk, dv = rp.run_backward(plan, res, kl, vl, dl, None, None, True, ops, tr, want_f32)
            results[rank] = [to_np(t) for t in (out, dq, dk, dv)]
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
    return {name: np.concatenate([results[r][n] for r in range(world)], axis=1)
            for n, name in enumerate(("out", "dq", "dk", "dv"))}


@pytest.mark.parametrize("bad", list(BADS))
@pytest.mark.parametrize("which", ["k", "do"])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("world", [2, 4])
def test_peer_ring(world, precision, dtype, which, bad):
    """zigzag, causal: one owner's scale is used by every rank that reads its shard"""
    from oracle.attn_dense import attention_visible
    tensors, row = _ring_inputs(world, dtype)
    key = (world, precision, dtype)
    if key not in _RING_CLEAN:
        _RING_CLEAN[key] = _ring_run(world, tensors, precision, dtype)
    clean = _RING_CLEAN[key]
    names = ("q", "k", "v", "do")
    dirty_t = list(tensors)
    t = dirty_t[names.index(which)].clone()
    t[BAD_B, row, BAD_H, BAD_COL] = BADS[bad]
    dirty_t[names.index(which)] = t
    dirty = _ring_run(world, dirty_t, precision, dtype)
    S = world * SL_RING
    vis = np.tril(np.ones((S, S), bool))
    sl = [to_np(x)[BAD_B:BAD_B + 1, :, BAD_H:BAD_H + 1] for x in dirty_t]
    out, _, dq, dk, dv = attention_visible(*sl[:3], vis[None, None], sl[3])
    ref = dict(out=out[0, :, 0], dq=dq[0, :, 0], dk=dk[0, :, 0], dv=dv[0, :, 0])
    same = _same_sets(which, row, BAD_COL, vis, S, S)
    bf16 = dtype == "bf16"
    for name in ("out", "dq", "dk", "dv"):
        if same[name] is None:
            continue
        _check_other_slices(name, clean[name], dirty[name], BAD_B, BAD_H, tol_dq=name == "dq", bf16=bf16)
        _check(name, clean[name][BAD_B, :, BAD_H], dirty[name][BAD_B, :, BAD_H], ref[name], same[name],
               TOL[precision], same_tol=name == "dq", bf16=bf16, strict=name == "out" or which == "do")


# ------------------------------------------------------------------------------------------------ 4. ringattention_inference
def _infer_case(dtype, Q, K, which):
    from lwm_b200.ringattention import decode_attention_mask
    g = torch.Generator().manual_seed(200 + Q)
    B, H = 2, 2
    q = torch.randn(B, Q, H, D, generator=g)
    k, v = torch.randn(B, K, H, D, generator=g), torch.randn(B, K, H, D, generator=g)
    do = torch.randn(B, Q, H, D, generator=g)
    j = 960 if Q >= 8 else 996
    for t in (k, v):
        t[BAD_B, j, BAD_H, BAD_COL] = 0
    pad = torch.ones(B, K, dtype=torch.int32)
    pad[0, :19] = 0
    mask = decode_attention_mask(pad, Q, K - Q - 2, K)
    return [t.to(DTYPES[dtype]).cuda() for t in (q, k, v, do)], mask.cuda(), j


def _infer_run(q, k, v, do, mask, grad):
    from lwm_b200.ringattention import ringattention_inference
    if not grad:
        out = ringattention_inference(q, k, v, mask)
        torch.cuda.synchronize()
        return dict(out=to_np(out))
    q, k, v = [t.detach().clone().requires_grad_(True) for t in (q, k, v)]
    out = ringattention_inference(q, k, v, mask)
    out.backward(do)
    torch.cuda.synchronize()
    return dict(out=to_np(out), dq=to_np(q.grad), dk=to_np(k.grad), dv=to_np(v.grad))


@pytest.mark.parametrize("bad", list(BADS))
@pytest.mark.parametrize("which", ["k", "v"])
@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("Q,K", [(64, 1000), (1, 1000), (3, 1000)])
def test_ringattention_inference(Q, K, dtype, which, bad):
    """Q = 64: the tensor-core path (scaled fp16 operands), forward and backward; Q = 1, 3: the GEMV kernel (no scale)"""
    from oracle.attn_dense import attention_visible
    (q, k, v, do), mask, j = _infer_case(dtype, Q, K, which)
    grad = Q >= 8
    clean = _infer_run(q, k, v, do, mask, grad)
    kd, vd = k.clone(), v.clone()
    (kd if which == "k" else vd)[BAD_B, j, BAD_H, BAD_COL] = BADS[bad]
    dirty = _infer_run(q, kd, vd, do, mask, grad)
    vis = mask.cpu().numpy()[BAD_B, 0]                      # [Q, K]
    sees = vis[:, j]
    assert sees.any() and (Q == 1 or not sees.all())
    sl = lambda t: to_np(t)[BAD_B:BAD_B + 1, :, BAD_H:BAD_H + 1]   # noqa: E731
    res = attention_visible(sl(q), sl(kd), sl(vd), vis[None, None], sl(do) if grad else None)
    ref = dict(zip(("out", "lse", "dq", "dk", "dv"), [r[0, :, 0] if r.ndim == 4 else r for r in res]))
    cols = np.ones(D, bool)
    cols[BAD_COL] = False
    # one Q tile holds every row: the reach of a bad v column is column d of every row
    same = dict(out=(~sees)[:, None] & np.ones(D, bool) if which == "k" else cols[None, :],
                dq=np.zeros((Q, D), bool), dk=np.zeros((K, D), bool),
                dv=np.zeros((K, D), bool) if which == "k" else np.ones((K, D), bool))
    tol = 1e-3 if dtype == "fp32" else 3e-3
    bf16 = dtype == "bf16"
    for name in clean:
        _check_other_slices(name, clean[name], dirty[name], BAD_B, BAD_H, tol_dq=name == "dq", bf16=bf16)
        _check(name, clean[name][BAD_B, :, BAD_H], dirty[name][BAD_B, :, BAD_H], ref[name], same[name], tol,
               same_tol=name == "dq", bf16=bf16, strict=name == "out")
    if which == "v":
        assert not np.isfinite(dirty["out"][BAD_B, sees, BAD_H, BAD_COL]).any()


# ------------------------------------------------------------------------------------------------ 5. VQGAN fp16 planes
def _vq_prep(x, st, gamma, beta):
    """lwm_vq_prep_f16 -> (plane [N,H,W,C] fp16 as int16 bits, scale); st None: the raw plane (its own absmax pass)"""
    from lwm_b200 import _lib
    from lwm_b200.vqgan import GN_EPS, GN_GROUPS
    N, H, W, C = x.shape
    hi = torch.empty(N, H, W, C, dtype=torch.float16, device=x.device)
    sc = torch.empty(2, dtype=torch.float32, device=x.device)
    _lib.call("lwm_vq_prep_f16", _lib.ptr(x), _lib.ptr(st), _lib.ptr(gamma), _lib.ptr(beta), _lib.ptr(hi),
              _lib.ptr(sc), _lib.ptr(sc[1:]), 0, N, H, W, C, C, GN_GROUPS, 0, GN_EPS, _lib.stream_ptr())
    torch.cuda.synchronize()
    return hi.view(torch.int16).cpu().numpy(), sc[0].item()


@pytest.mark.parametrize("bad", list(BADS))
@pytest.mark.parametrize("gn", ["groupnorm", "raw"])
def test_vq_prep_f16_plane_scale(gn, bad):
    """a 2-image batch whose image 1 has non-finite GroupNorm statistics (or, raw, one non-finite pixel): image 0's
    plane and the scale are those of the clean call"""
    from lwm_b200.vqgan import Ops
    from oracle import vqgan_ref as vr
    g = torch.Generator().manual_seed(9)
    x = torch.randn(2, 32, 32, 128, generator=g).cuda()
    x[1, 5, 7, 9] = 0
    val = BADS[bad]
    if gn == "groupnorm":
        p = vr._gn_p(g, 128)
        gamma, beta = p["scale"].cuda(), p["bias"].cuda()
        st = Ops("fp16x2").gn_stats(x)
        std = st.clone()
        std[1, 3, 0] = val                                  # image 1, group 3: sum and sum of squares
        std[1, 3, 1] = abs(val)
        plane, s = _vq_prep(x, st, gamma, beta)
        plane_d, s_d = _vq_prep(x, std, gamma, beta)
        assert s_d == s
        assert np.array_equal(plane_d[0], plane[0])
    else:
        xd = x.clone()
        xd[1, 5, 7, 9] = val
        plane, s = _vq_prep(x, None, None, None)
        plane_d, s_d = _vq_prep(xd, None, None, None)
        assert s_d == s == _model_scale(x)
        assert np.array_equal(plane_d[0], plane[0])
        diff = np.argwhere(plane_d != plane)
        assert diff.tolist() == [[1, 5, 7, 9]]


@pytest.mark.parametrize("bad", list(BADS))
def test_vq_conv2d_f16_absmax_of_finite_outputs(bad):
    """absmax_out of a conv whose input has one non-finite pixel is the |max| over the finite entries it wrote, and
    every output the pixel cannot reach equals the clean conv's"""
    from lwm_b200.vqgan import Ops, PackedConv
    from oracle import vqgan_ref as vr
    g = torch.Generator().manual_seed(13)
    x = torch.randn(2, 64, 64, 128, generator=g).cuda()
    x[1, 20, 30, 4] = 0
    pc = PackedConv(vr._conv_p(g, 3, 128, 128), torch.device("cuda"))
    ops = Ops("fp16x2")
    xd = x.clone()
    xd[1, 20, 30, 4] = BADS[bad]
    y = ops.conv_gn(x, pc, want_stats=True)
    yd = ops.conv_gn(xd, pc, want_stats=True)
    torch.cuda.synchronize()
    yn, ydn = to_np(y), to_np(yd)
    fin = np.isfinite(ydn)
    assert not fin.all()
    amax = np.abs(ydn[fin]).max().astype(np.float32)
    assert int(yd._absmax_bits.item()) == int(amax.view(np.int32))
    reach = np.zeros(yn.shape, bool)
    reach[1, 19:22, 29:32] = True                          # the 3x3 window around the pixel
    assert np.array_equal(_bits(yn[~reach]), _bits(ydn[~reach]))
