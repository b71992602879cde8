"""The attention backward under torch.use_deterministic_algorithms(True): dQ reduced in ascending key-tile order
(lwm_attn_bwd_step / lwm_attn_infer_bwd given an order_ws, DESIGN §3.3).

  * the turns pass against a numpy count over the backward lists: packed segments, left padding, the call-site zero bias
    with packed segments, and random inference masks (Q = 72, not a multiple of 64); the semaphores end at the number
    of key tiles that reduce into their Q tile, every CTA took one ticket, and the error word stays 0;
  * repeatability: three backward calls on one graph give the same bits of dQ, dK and dV, in both precision modes, for
    bf16 and fp32 inputs (whether the unordered path differed at the same shapes is printed, not asserted);
  * against the unordered path: out, dK and dV bit-identical, dQ within _dq_close, and the float64 oracle's tolerances;
  * fp16 mode: 2^k dO gives exactly 2^k dQ;
  * the peer-memory and two-sided NCCL ring executors (ranks as threads): two runs bit-identical on every rank;
  * plumbing: with the flag off only the existing entry points are called, with it on only the ordered ones.
The flag is set by the `deterministic` fixture, which restores it afterwards and checks the error word of every ordered
call (the workspaces are recorded through ringattention.order_workspace)."""
import threading

import numpy as np
import pytest
import torch

from helpers import rel_fro, to_np
from nonfinite_checks import _dq_close

pytestmark = pytest.mark.gpu

FMIN = float(np.finfo(np.float32).min)
CAUSAL = dict(blockwise_kwargs=dict(causal_block_size=1))
TOL = {torch.float32: 1e-3, torch.bfloat16: 3e-3}


@pytest.fixture
def deterministic(monkeypatch):
    """torch.use_deterministic_algorithms(True) for the test (restored afterwards) -> the list of the order_ws
    workspaces of the ordered calls made; at the end every error word must still be 0"""
    from lwm_b200 import ringattention as ra
    wss, make = [], ra.order_workspace
    lock = threading.Lock()

    def recording(words, device):
        ws = make(words, device)
        with lock:
            wss.append(ws)
        return ws

    monkeypatch.setattr(ra, "order_workspace", recording)
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield wss
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)
    torch.cuda.synchronize()
    assert all(int(ws[1]) == 0 for ws in wss), "an ordered dQ reduction timed out waiting for its turn"


def _qkv(B, Sq, Sk, H, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, n, H, 128, generator=g) for n in (Sq, Sk, Sk))
    do = torch.randn(B, Sq, H, 128, generator=g)
    return [t.to(dtype).cuda() for t in (q, k, v, do)]


def _packed_seg(B, S, lo, hi, seed):
    rng = np.random.default_rng(seed)
    seg = np.zeros((B, S), np.int32)
    for b in range(B):
        p, i = 0, 0
        while p < S:
            n = int(rng.integers(lo, hi + 1))
            seg[b, p:p + n] = i
            p, i = p + n, i + 1
    return seg


def _masks(kind, B, S):
    """(attn_bias [B,1,1,S] or None, segment_ids [B,S] or None) on the device"""
    bias = seg = None
    if kind == "docs":
        seg = _packed_seg(B, S, 1, S // 3, S)
    elif kind == "pad":
        bias = np.zeros((B, S), np.float32)
        for b in range(B):
            bias[b, :(S // 4 + 37) * (b + 1) // 2] = FMIN
    elif kind == "callsite":       # lwm/llama.py's zero bias, with packed documents
        bias, seg = np.zeros((B, S), np.float32), _packed_seg(B, S, 100, 900, 7)
    return (None if bias is None else torch.from_numpy(bias)[:, None, None].cuda(),
            None if seg is None else torch.from_numpy(seg).cuda())


def _op_grads(q, k, v, do, bias, seg, causal, precision, calls=1):
    """out and `calls` backward passes of one forward graph of ringattention -> (out, [(dq, dk, dv)] * calls)"""
    from lwm_b200.ringattention import ringattention
    leaves = [x.detach().clone().requires_grad_() for x in (q, k, v)]
    out = ringattention(*leaves, bias, seg, precision=precision, **(CAUSAL if causal else {}))
    grads = [tuple(t.detach().clone() for t in torch.autograd.grad(out, leaves, do, retain_graph=i + 1 < calls))
             for i in range(calls)]
    torch.cuda.synchronize()
    return out.detach(), grads


def _infer_grads(q, k, v, do, mask, calls=1):
    from lwm_b200.ringattention import ringattention_inference
    leaves = [x.detach().clone().requires_grad_() for x in (q, k, v)]
    out = ringattention_inference(*leaves, None if mask is None else mask.cuda())
    grads = [tuple(t.detach().clone() for t in torch.autograd.grad(out, leaves, do, retain_graph=i + 1 < calls))
             for i in range(calls)]
    torch.cuda.synchronize()
    return out.detach(), grads


def _bits(t):
    return t.detach().contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16).cpu().numpy()


def _same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(_bits(a), _bits(b))


def _random_infer_mask(B, Q, K, seed):
    """blocks that are all masked, all visible or random, and one fully masked row"""
    g = torch.Generator().manual_seed(seed)
    nq, nk = (Q + 63) // 64, (K + 127) // 128
    kind = torch.randint(0, 3, (B, nq, nk), generator=g).repeat_interleave(64, 1).repeat_interleave(128, 2)[:, :Q, :K]
    rnd = torch.rand(B, Q, K, generator=g) < 0.5
    m = torch.where(kind == 0, torch.zeros_like(rnd), torch.where(kind == 1, torch.ones_like(rnd), rnd))
    m[:, min(2, Q - 1)] = False
    return m[:, None]


# ------------------------------------------------------------------------------------------------ the turns pass
def _turns_model(tiles, counts):
    """numpy count over the backward lists -> (turn of every entry {(b, n, pos): turn}, per (b, Q tile) the number of
    key tiles whose list holds it)"""
    B, n_kt, n_q = tiles.shape
    turns, seen = {}, np.zeros((B, n_q), np.int64)
    for b in range(B):
        for n in range(n_kt):
            for pos in range(counts[b, n]):
                qt = tiles[b, n, pos] >> 1
                turns[(b, n, pos)] = seen[b, qt]
            for pos in range(counts[b, n]):
                seen[b, tiles[b, n, pos] >> 1] += 1
    return turns, seen


def _check_workspace(ws, tiles, counts, B, H, n_kt):
    ws = ws.cpu().numpy()
    n_q = tiles.shape[2]
    assert ws[0] == B * H * n_kt, "tickets taken: %d of %d CTAs" % (ws[0], B * H * n_kt)
    assert ws[1] == 0
    turns, seen = _turns_model(tiles, counts)
    sem = ws[2:2 + B * H * n_q].reshape(B, H, n_q)
    assert (sem == seen[:, None, :]).all(), "a semaphore does not count the key tiles of its Q tile"
    got = ws[2 + B * H * n_q:].reshape(B, n_kt, n_q)
    bad = [key for key, t in turns.items() if got[key] != t]
    assert not bad, "%d of %d turns differ from the model, first %s" % (len(bad), len(turns), bad[:3])
    return len(turns)


@pytest.mark.parametrize("kind", ["docs", "pad", "callsite"])
@pytest.mark.parametrize("causal", [True, False])
def test_turns_of_training_maps_equal_numpy_count(deterministic, kind, causal):
    from lwm_b200 import ringattention as ra
    B, S, H = 2, 2048, 2
    q, k, v, do = _qkv(B, S, S, H, torch.bfloat16, 11)
    bias, seg = _masks(kind, B, S)
    _op_grads(q, k, v, do, bias, seg, causal, "fp16")
    assert len(deterministic) == 1
    b2 = None if bias is None else bias.reshape(B, S).float().contiguous()
    _, _, bt, bc = ra.step_tilemap(B, S, S, 0, 0, causal, b2, seg, fwd=False)
    n = _check_workspace(deterministic[0], bt.cpu().numpy(), bc.cpu().numpy(), B, H, S // 128)
    print("%s causal=%d: %d list entries" % (kind, causal, n))


def test_semaphores_without_a_map_count_the_causal_prefix(deterministic):
    B, S, H = 1, 4096, 3
    _op_grads(*_qkv(B, S, S, H, torch.bfloat16, 12), None, None, True, "bf16")
    ws = deterministic[0].cpu().numpy()
    n_q = S // 64
    assert ws[0] == B * H * (S // 128) and ws[1] == 0 and ws.size == 2 + B * H * n_q
    # key tile n reaches Q tile i when 64 i + 63 >= 128 n
    assert (ws[2:].reshape(B, H, n_q) == (np.arange(n_q) // 2 + 1)[None, None]).all()


@pytest.mark.parametrize("Q,K", [(72, 300), (1024, 1024), (200, 4096)])
def test_turns_of_inference_maps_equal_numpy_count(deterministic, monkeypatch, Q, K):
    from lwm_b200 import _lib, ringattention as ra
    B, H = 2, 2
    seen = []
    backward = ra.InferOps.backward

    def spy(q16, k16, v16, do16, scales, lse, delta, bits, row_any):
        seen.append((bits, row_any))
        return backward(q16, k16, v16, do16, scales, lse, delta, bits, row_any)

    monkeypatch.setattr(ra.InferOps, "backward", staticmethod(spy))
    q, k, v, do = _qkv(B, Q, K, H, torch.float32, 13)
    _infer_grads(q, k, v, do, _random_infer_mask(B, Q, K, Q + K))
    bits, row_any = seen[0]
    n_kt, n_q = (K + 127) // 128, (Q + 63) // 64
    tiles = torch.empty(B, n_kt, n_q, dtype=torch.int32, device="cuda")
    counts = torch.empty(B, n_kt, dtype=torch.int32, device="cuda")
    _lib.call("lwm_attn_infer_bwd_tilemap", _lib.ptr(bits), _lib.ptr(row_any), B, Q, K, _lib.ptr(tiles),
              _lib.ptr(counts), _lib.stream_ptr())
    assert len(deterministic) == 1
    _check_workspace(deterministic[0], tiles.cpu().numpy(), counts.cpu().numpy(), B, H, n_kt)


# ------------------------------------------------------------------------------------------------ repeatability
TRAIN_SHAPES = {"noncausal_256x32k": (1, 256, 32768, 4, False, None), "causal_8k": (1, 8192, 8192, 4, True, None),
                "callsite_map_4k": (2, 4096, 4096, 2, True, "callsite")}


def _repeat_check(ordered, unordered, label):
    """ordered: three (dq, dk, dv) that must be the same bits; unordered: the same calls without the flag (printed)"""
    for name, i in (("dq", 0), ("dk", 1), ("dv", 2)):
        for j in (1, 2):
            assert _same_bits(ordered[0][i], ordered[j][i]), "%s: %s of call %d differs from call 0" % (label, name, j)
    diff = [not _same_bits(unordered[0][0], g[0]) for g in unordered[1:]]
    print("%s: ordered dQ repeatable; unordered dQ differed between runs: %s" % (label, diff))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("shape", sorted(TRAIN_SHAPES))
def test_three_backward_calls_are_bit_identical(deterministic, shape, precision, dtype):
    B, Sq, Sk, H, causal, masks = TRAIN_SHAPES[shape]
    q, k, v, do = _qkv(B, Sq, Sk, H, dtype, 21)
    bias, seg = _masks(masks, B, Sq)
    out_o, ordered = _op_grads(q, k, v, do, bias, seg, causal, precision, calls=3)
    n_ordered = len(deterministic)
    torch.use_deterministic_algorithms(False)
    out_u, unordered = _op_grads(q, k, v, do, bias, seg, causal, precision, calls=3)
    torch.use_deterministic_algorithms(True)
    assert n_ordered == 3 and len(deterministic) == 3
    _repeat_check(ordered, unordered, "%s %s %s" % (shape, precision, dtype))
    # against the unordered path: the same out, dK and dV; dQ up to the order of its fp32 additions
    assert _same_bits(out_o, out_u)
    assert _same_bits(ordered[0][1], unordered[0][1]) and _same_bits(ordered[0][2], unordered[0][2])
    # the bf16 mode rounds fp32 inputs, and so their gradients, to bf16
    bf16_result = dtype == torch.bfloat16 or precision == "bf16"
    assert _dq_close(to_np(unordered[0][0]), to_np(ordered[0][0]), bf16_result)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("Q", [1024, 72])
def test_inference_backward_three_calls_are_bit_identical(deterministic, Q, dtype):
    B, H, K = 2, 2, 2048 if Q == 1024 else 300
    q, k, v, do = _qkv(B, Q, K, H, dtype, 22)
    mask = _random_infer_mask(B, Q, K, 5)
    out_o, ordered = _infer_grads(q, k, v, do, mask, calls=3)
    torch.use_deterministic_algorithms(False)
    out_u, unordered = _infer_grads(q, k, v, do, mask, calls=3)
    torch.use_deterministic_algorithms(True)
    assert len(deterministic) == 3
    _repeat_check(ordered, unordered, "inference Q=%d %s" % (Q, dtype))
    assert _same_bits(out_o, out_u)
    assert _same_bits(ordered[0][1], unordered[0][1]) and _same_bits(ordered[0][2], unordered[0][2])
    assert _dq_close(to_np(unordered[0][0]), to_np(ordered[0][0]), dtype == torch.bfloat16)


def test_causal_131072_fp16_three_calls(deterministic):
    B, S, H = 1, 131072, 2
    q, k, v, do = _qkv(B, S, S, H, torch.bfloat16, 23)
    _, ordered = _op_grads(q, k, v, do, None, None, True, "fp16", calls=3)
    for name, i in (("dq", 0), ("dk", 1), ("dv", 2)):
        for j in (1, 2):
            assert _same_bits(ordered[0][i], ordered[j][i]), (name, j)
    assert len(deterministic) == 3


# ------------------------------------------------------------------------------------------------ oracles, scaling
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("kind", ["docs", "callsite", None])
def test_ordered_gradients_match_float64_oracle(deterministic, kind, dtype):
    from oracle.attn_dense import attention_dense_grads
    B, S, H = 2, 1024, 2
    q, k, v, do = _qkv(B, S, S, H, dtype, 31)
    bias, seg = _masks(kind, B, S)
    _, ((dq, dk, dv),) = _op_grads(q, k, v, do, bias, seg, True, "fp16")
    kw = dict(causal=True)
    if bias is not None:
        kw["attn_bias"] = bias.reshape(B, S).cpu().numpy()
    if seg is not None:
        kw["segment_ids"] = seg.cpu().numpy()
    ref = attention_dense_grads(*[to_np(t).astype(np.float64) for t in (q, k, v, do)], **kw)
    for name, got, r in zip(("dq", "dk", "dv"), (dq, dk, dv), ref):
        err = rel_fro(to_np(got), r)
        print("%s %s %s: %.2e" % (kind, dtype, name, err))
        assert err < TOL[dtype], (name, err)


@pytest.mark.parametrize("e", [5, -7])
def test_fp16_mode_power_of_two_dout_scales_dq_exactly(deterministic, e):
    B, S, H = 1, 4096, 2
    q, k, v, do = _qkv(B, S, S, H, torch.float32, 41)
    _, ((dq, dk, dv),) = _op_grads(q, k, v, do, None, None, True, "fp16")
    _, ((dq2, dk2, dv2),) = _op_grads(q, k, v, do * 2.0 ** e, None, None, True, "fp16")
    for a, b in ((dq, dq2), (dk, dk2), (dv, dv2)):
        assert _same_bits(a * 2.0 ** e, b)


# ------------------------------------------------------------------------------------------------ rings
def _ring_inputs(world, Sl, seed):
    B, H = 2, 2
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, world * Sl, H, 128, generator=g).to(torch.bfloat16) for _ in range(4)]


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("world,layout", [(2, "zigzag"), (4, "zigzag"), (2, "contiguous"), (4, "contiguous")])
def test_peer_ring_two_runs_bit_identical(deterministic, world, layout, precision):
    from lwm_b200 import ring_peer as rp, ring_schedule as rs
    from lwm_b200.ringattention import PeerOpsBf16, PeerOpsF16
    from peer_emulation import EmuTransport, EmuWorld
    dev = torch.device("cuda", 0)
    Sl = 512
    emu = EmuWorld(world, device=dev)
    q, k, v, do = _ring_inputs(world, Sl, 51)
    ops = PeerOpsF16 if precision == "fp16" else PeerOpsBf16
    results, fails = {}, []

    def worker(rank):
        try:
            torch.cuda.set_device(dev)
            tr = EmuTransport(emu, rank)
            plan = rs.make_peer_plan(world, rank, Sl, Sl, True, layout)
            sl = slice(rank * Sl, (rank + 1) * Sl)
            ql, kl, vl, dl = [t[:, sl].to(dev).contiguous() for t in (q, k, v, do)]
            runs = []
            for _ in range(2):
                out, res = rp.run_forward(plan, ql, kl, vl, None, None, True, ops, tr, False)
                runs.append([t.clone() for t in (out,) + tuple(rp.run_backward(plan, res, kl, vl, dl, None, None,
                                                                                 True, ops, tr, False))])
            results[rank] = runs
        except BaseException:   # noqa: BLE001  (reported by the main thread)
            import traceback
            fails.append(traceback.format_exc())
            emu.barrier.abort()

    ts = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    torch.cuda.synchronize()
    assert not any(t.is_alive() for t in ts) and not fails, fails[:1]
    assert deterministic, "no ordered backward step ran"
    for r in range(world):
        for name, a, b in zip(("out", "dq", "dk", "dv"), *results[r]):
            assert _same_bits(a, b), "rank %d: %s differs between two runs" % (r, name)


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
@pytest.mark.parametrize("world,layout", [(2, "zigzag"), (4, "zigzag"), (2, "contiguous"), (4, "contiguous")])
def test_nccl_ring_two_runs_bit_identical(deterministic, monkeypatch, world, layout, precision):
    from lwm_b200 import ring_exec as rx, ringattention as ra
    from nccl_emulation import EmuComm, EmuGroup, EmuP2P, run_threads
    monkeypatch.setattr(rx, "_Comm", EmuComm)
    monkeypatch.setenv("LWM_RING_TRANSPORT", "nccl")
    Sl = 512
    emu = EmuP2P(world)
    q, k, v, do = _ring_inputs(world, Sl, 52)

    def rank_fn(rank):
        torch.cuda.set_device("cuda:0")
        grp = EmuGroup(emu, rank)
        sl = slice(rank * Sl, (rank + 1) * Sl)
        ql, kl, vl, dl = [t[:, sl].to("cuda:0").contiguous() for t in (q, k, v, do)]
        runs = []
        for i in range(2):
            grp.tag = (i, "fwd")
            out, res = ra.ring_forward(ql, kl, vl, None, None, True, grp, rank, world, layout, precision)
            grp.tag = (i, "bwd")
            grads = ra.ring_backward(res, kl, vl, dl, None, None, True, grp, rank, world, layout, precision)
            runs.append([t.clone() for t in (out,) + tuple(grads)])
            emu.end_pass(rank)
        return runs

    results = run_threads(world, emu, rank_fn)
    assert deterministic, "no ordered backward step ran"
    for r in range(world):
        for name, a, b in zip(("out", "dq", "dk", "dv"), *results[r]):
            assert _same_bits(a, b), "rank %d: %s differs between two runs" % (r, name)


# ------------------------------------------------------------------------------------------------ plumbing
def test_order_workspace_follows_the_flag(monkeypatch):
    from lwm_b200 import _lib
    calls = []     # (name, whether its order_ws slot holds a workspace; None for calls without one)
    call = _lib.call
    ws_slot = {"lwm_attn_bwd_step": 29, "lwm_attn_infer_bwd": 22}

    def spy(name, *args):
        calls.append((name, args[ws_slot[name]] is not None if name in ws_slot else None))
        return call(name, *args)

    monkeypatch.setattr(_lib, "call", spy)
    B, S, H = 1, 1024, 2
    q, k, v, do = _qkv(B, S, S, H, torch.bfloat16, 61)
    bias, seg = _masks("callsite", B, S)
    mask = _random_infer_mask(B, 200, 300, 3)
    qi, ki, vi, doi = _qkv(B, 200, 300, H, torch.bfloat16, 62)

    def run():
        del calls[:]
        _op_grads(q, k, v, do, None, None, True, "fp16")
        _op_grads(q, k, v, do, bias, seg, True, "bf16")
        _infer_grads(qi, ki, vi, doi, mask)
        return list(calls)

    prev = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(False)
        off = run()
        torch.use_deterministic_algorithms(True)
        on = run()
    finally:
        torch.use_deterministic_algorithms(prev)
    assert off.count(("lwm_attn_bwd_step", False)) == 2 and off.count(("lwm_attn_infer_bwd", False)) == 1
    assert not [c for c in off if c[1]]
    assert on.count(("lwm_attn_bwd_step", True)) == 2 and on.count(("lwm_attn_infer_bwd", True)) == 1
    assert not [c for c in on if c[1] is False]
    # apart from the backward launches' workspace, the flag changes no call
    assert [n for n, _ in on] == [n for n, _ in off]
