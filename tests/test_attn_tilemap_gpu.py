"""The training block map on the GPU: lwm_attn_step_tilemap against its numpy restatement (tests/tilemap_model.py), the
map entry points against the entry points without a map (bit for bit: out, out_f32, lse, the carries, dK, dV; dQ, whose
fp32 reductions land in no fixed order, within a tight tolerance), and the public op with packed and left-padded
sequences. Tolerances against the float64 oracle are those of tests/test_attn_public_op_gpu.py: 1e-3 for fp32 results,
3e-3 for bf16 results."""
import threading

import numpy as np
import pytest
import torch

import tilemap_model as tm

pytestmark = pytest.mark.gpu
KW = dict(axis_name="sp", float32_logits=True, cache_idx=None,
          blockwise_kwargs=dict(causal_block_size=1, deterministic=True, attn_pdrop=0.0, query_chunk_size=256,
                                key_chunk_size=256))
FMIN = float(np.finfo(np.float32).min)


def _dev(x, dtype=None):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).cuda()


CASES = tm.sweep_cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_map_kernel_equals_numpy_model(case):
    from lwm_b200 import ringattention as ra
    _, bias, seg, Sq, Sk, q0, k0, causal = case
    ft, fc, bt, bc = ra.step_tilemap(2, Sq, Sk, q0, k0, causal, _dev(bias), _dev(seg))
    fwd, bwd = tm.step_tilemap(bias, seg, Sq, Sk, q0, k0, causal)
    ft, fc, bt, bc = [t.cpu().numpy() for t in (ft, fc, bt, bc)]
    for b in range(2):
        for t, lst in enumerate(fwd[b]):
            assert fc[b, t] == len(lst) and list(ft[b, t, :len(lst)]) == lst, (b, t)
        for kt, lst in enumerate(bwd[b]):
            assert bc[b, kt] == len(lst) and list(bt[b, kt, :len(lst)]) == lst, (b, kt)


def _packed_seg(B, S, doc_lens, seed=0):
    seg = np.zeros((B, S), np.int32)
    rng = np.random.default_rng(seed)
    for b in range(B):
        p, i = 0, 0
        while p < S:
            n = int(doc_lens if np.isscalar(doc_lens) else rng.integers(doc_lens[0], doc_lens[1] + 1))
            seg[b, p:p + n] = i
            p, i = p + n, i + 1
    return seg


def _masks(kind, B, S):
    """(bias [B,S] f32 or None, seg [B,S] i32 or None) on the device"""
    bias = seg = None
    if kind == "callsite":
        bias, seg = np.zeros((B, S), np.float32), np.zeros((B, S), np.int32)
    elif kind == "docs":
        seg = _packed_seg(B, S, (1, S // 3), seed=S)
    elif kind == "pad":
        bias = np.zeros((B, S), np.float32)
        for b in range(B):
            bias[b, :(S // 4 + 37) * (b + 1) // 2] = FMIN
    elif kind == "docs+pad":
        seg = _packed_seg(B, S, 300)
        bias = np.zeros((B, S), np.float32)
        bias[:, :S // 4 + 5] = FMIN
    return _dev(bias), _dev(seg)


def _step_pair(ra, mode, q, k, v, do, bias, seg, q0, k0, causal):
    """(old, map) results of every forward first/last combination and of the backward for one step"""
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    dev = q.device
    if mode == "fp16":
        (q, sq), (k, sk), (v, sv), (do, sd) = ra.to_f16(q), ra.to_f16(k), ra.to_f16(v), ra.to_f16(do)
        fs, bs = (sq, sk, sv), (sq, sk, sv, sd)
    else:
        fs = bs = None
    ft, fc, bt, bc = ra.step_tilemap(B, Sq, Sk, q0, k0, causal, bias, seg)
    g = torch.Generator(device=dev).manual_seed(1)
    carry0 = (torch.randn(B, Sq, H, D, device=dev, generator=g), torch.randn(B, H, Sq, device=dev, generator=g) * 4,
              torch.rand(B, H, Sq, device=dev, generator=g) * 100 + 1)
    res = []
    for tmap in (None, (ft, fc)):
        r = {}
        for first, last in ((1, 1), (1, 0), (0, 1), (0, 0)):
            out = torch.full((B, Sq, H, D), 7.0, dtype=torch.bfloat16, device=dev)
            lse = torch.full((B, H, Sq), 7.0, device=dev)
            o32 = torch.full((B, Sq, H, D), 7.0, device=dev) if fs else None
            acc = [c.clone() for c in carry0]
            ra.fwd_step(q, k, v, out, lse, *acc, q0, k0, causal, bias, seg, first, last, scales=fs, out_f32=o32,
                        tilemap=tmap)
            r[(first, last)] = (out, lse, o32) if last else tuple(acc)
        out, lse = r[(1, 1)][:2]
        o_ref = r[(1, 1)][2] if fs else out
        delta = torch.empty(B, H, Sq, device=dev)
        if fs:
            from lwm_b200.ringattention import PeerOpsF16
            PeerOpsF16.bwd_prep(o_ref, do, bs[3], delta)
        else:
            ra.bwd_prep(out, do, delta)
        nl = ra.lse_for_bwd(lse, f16=bool(fs))
        grads = []
        for init in (True, False):
            dq = torch.zeros(B, Sq, H, D, device=dev)
            dk = torch.full((B, Sk, H, D), 0.5, device=dev)
            dv = torch.full((B, Sk, H, D), -0.25, device=dev)
            ra.bwd_step(q, k, v, do, nl, delta, dq, dk, dv, q0, k0, causal, bias, seg, scales=bs, init=init,
                        tilemap=None if tmap is None else (bt, bc))
            grads.append((dq, dk, dv))
        r["grads"] = grads
        res.append(r)
    return res


def _assert_steps_identical(old, new):
    for key in ((1, 1), (1, 0), (0, 1), (0, 0)):
        for a, b in zip(old[key], new[key]):
            if a is not None:
                assert torch.equal(a, b), key
    for (dq0, dk0, dv0), (dq1, dk1, dv1) in zip(old["grads"], new["grads"]):
        assert torch.equal(dk0, dk1) and torch.equal(dv0, dv1)
        scale = float(dq0.abs().max())
        assert float((dq0 - dq1).abs().max()) <= 1e-5 * max(scale, 1e-30), "dQ beyond reduction-order noise"


STEP_CASES = [("callsite", 1024, 1024, 0, 0, True), ("docs", 1024, 1024, 0, 0, True), ("pad", 1024, 1024, 0, 0, True),
              ("docs+pad", 1024, 1024, 0, 0, False), ("docs", 512, 1024, 512, 0, True),
              ("pad", 512, 512, 0, 512, True), ("docs+pad", 512, 512, 512, 0, True)]


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
@pytest.mark.parametrize("kind,Sq,Sk,q0,k0,causal", STEP_CASES)
def test_map_step_bit_identical_to_step_without_map(mode, kind, Sq, Sk, q0, k0, causal):
    from lwm_b200 import ringattention as ra
    B, H = 2, 2
    S = max(q0 + Sq, k0 + Sk)
    bias, seg = _masks(kind, B, S)
    g = torch.Generator(device="cuda").manual_seed(3)
    q = torch.randn(B, Sq, H, 128, device="cuda", generator=g).to(torch.bfloat16)
    do = torch.randn(B, Sq, H, 128, device="cuda", generator=g).to(torch.bfloat16)
    k, v = [torch.randn(B, Sk, H, 128, device="cuda", generator=g).to(torch.bfloat16) for _ in range(2)]
    old, new = _step_pair(ra, mode, q, k, v, do, bias, seg, q0, k0, causal)
    _assert_steps_identical(old, new)


def test_call_site_mask_at_128k_bit_identical():
    from lwm_b200 import ringattention as ra
    B, H, S = 1, 2, 131072
    bias, seg = _masks("callsite", B, S)
    g = torch.Generator(device="cuda").manual_seed(9)
    q, k, v, do = [torch.randn(B, S, H, 128, device="cuda", generator=g).to(torch.bfloat16) for _ in range(4)]
    (q16, sq), (k16, sk), (v16, sv), (d16, sd) = ra.to_f16(q), ra.to_f16(k), ra.to_f16(v), ra.to_f16(do)
    ft, fc, bt, bc = ra.step_tilemap(B, S, S, 0, 0, True, bias, seg)
    outs = []
    for tmap in (None, (ft, fc)):
        out = torch.empty(B, S, H, 128, dtype=torch.bfloat16, device="cuda")
        o32 = torch.empty(B, S, H, 128, device="cuda")
        lse = torch.empty(B, H, S, device="cuda")
        ra.fwd_step(q16, k16, v16, out, lse, None, None, None, 0, 0, True, bias, seg, True, True, scales=(sq, sk, sv),
                    out_f32=o32, tilemap=tmap)
        outs.append((out, o32, lse))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    out, o32, lse = outs[0]
    del outs
    delta = torch.empty(B, H, S, device="cuda")
    from lwm_b200.ringattention import PeerOpsF16
    PeerOpsF16.bwd_prep(o32, d16, sd, delta)
    nl = ra.lse_for_bwd(lse, f16=True)
    grads = []
    for tmap in (None, (bt, bc)):
        dq = torch.zeros(B, S, H, 128, device="cuda")
        dk, dv = torch.empty_like(dq), torch.empty_like(dq)
        ra.bwd_step(q16, k16, v16, d16, nl, delta, dq, dk, dv, 0, 0, True, bias, seg, scales=(sq, sk, sv, sd),
                    init=True, tilemap=tmap)
        grads.append((dq, dk, dv))
    (dq0, dk0, dv0), (dq1, dk1, dv1) = grads
    assert torch.equal(dk0, dk1) and torch.equal(dv0, dv1)
    assert float((dq0 - dq1).abs().max()) <= 1e-5 * float(dq0.abs().max())


def _public(q, k, v, do, bias, seg, dtype):
    from lwm_b200 import ringattention as ra
    q, k, v = [t.detach().to(dtype).requires_grad_(True) for t in (q, k, v)]
    out = ra.ringattention(q, k, v, None if bias is None else bias[:, None, None, :], seg, **KW)
    out.backward(do.to(dtype))
    return out.detach(), q.grad, k.grad, v.grad


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind", ["docs", "docs+pad"])
def test_public_op_packed_documents_against_dense_oracle(dtype, kind):
    from oracle.attn_dense import attention_dense, attention_dense_grads
    B, S, H = 2, 2048, 2
    bias, seg = _masks(kind, B, S)
    g = torch.Generator().manual_seed(11)
    q, k, v, do = [torch.randn(B, S, H, 128, generator=g).to(torch.bfloat16).float().cuda() for _ in range(4)]
    if bias is not None:
        do[(bias == FMIN)] = 0   # padded rows: no upstream gradient, as the loss mask gives them
    got = _public(q, k, v, do, bias, seg, dtype)
    kw = dict(causal=True, segment_ids=seg.cpu().numpy())
    if bias is not None:
        kw["attn_bias"] = bias.cpu().numpy()
    n = [t.double().cpu().numpy() for t in (q, k, v, do)]
    refs = (attention_dense(*n[:3], **kw),) + tuple(attention_dense_grads(*n, **kw))
    tol = 1e-3 if dtype == torch.float32 else 3e-3
    real = np.ones((B, S), bool) if bias is None else (bias != FMIN).cpu().numpy()
    for j, (a, r) in enumerate(zip(got, refs)):
        a = a.double().cpu().numpy()
        if j < 2:   # padded query rows of out / dq are checked in their own test
            a, r = a * real[:, :, None, None], r * real[:, :, None, None]
        err = np.linalg.norm(a - r) / np.linalg.norm(r)
        assert err <= tol, (j, err)


def test_public_op_packed_32k_equals_documents_run_alone():
    B, S, H, L = 1, 32768, 2, 4096
    seg = torch.from_numpy(_packed_seg(B, S, L)).cuda()
    g = torch.Generator().manual_seed(13)
    q, k, v, do = [torch.randn(B, S, H, 128, generator=g).to(torch.bfloat16).cuda() for _ in range(4)]
    got = _public(q, k, v, do, None, seg, torch.bfloat16)
    for d in range(S // L):
        sl = slice(d * L, (d + 1) * L)
        ref = _public(*[t[:, sl].contiguous() for t in (q, k, v, do)], None, None, torch.bfloat16)
        for a, r in zip(got, ref):
            a, r = a[:, sl].double(), r.double()
            err = float(torch.linalg.norm(a - r) / torch.linalg.norm(r))
            assert err <= 3e-3, (d, err)


@pytest.mark.parametrize("precision", ["fp16", "bf16"])
def test_left_padded_rows_average_uniformly_and_get_no_gradient(precision):
    from lwm_b200 import ringattention as ra
    B, S, H, npad = 2, 1024, 2, 300
    bias = torch.zeros(B, S, device="cuda")
    bias[:, :npad] = FMIN
    g = torch.Generator().manual_seed(17)
    q, k, v, do = [torch.randn(B, S, H, 128, generator=g).cuda() for _ in range(4)]
    q, k, v = [t.requires_grad_(True) for t in (q, k, v)]
    out = ra.ringattention(q, k, v, bias[:, None, None, :], None, precision=precision, **KW)
    out.backward(do)
    # a row that sees no key averages every key it visits with the masked logit: the keys of the 128-key tiles up to
    # and including its diagonal one (those above the diagonal carry the same masked logit)
    vv = v.detach().double() if precision == "fp16" else v.detach().to(torch.bfloat16).double()
    ends = (torch.arange(npad, device="cuda") // 128 + 1) * 128
    avg = (torch.cumsum(vv, dim=1)[:, ends - 1] / ends.double()[None, :, None, None])
    err = float((out.detach()[:, :npad].double() - avg).abs().max() / avg.abs().max())
    assert err <= (1e-3 if precision == "fp16" else 1e-2), err
    assert torch.count_nonzero(q.grad[:, :npad]) == 0


def test_peer_executor_map_path_bit_identical_to_old_entry_points():
    """zigzag ring of 2 ranks emulated with threads on one GPU, B = 2, packed and padded masks"""
    from lwm_b200 import ring_peer as rp, ring_schedule as rs
    from lwm_b200 import ringattention as ra
    from lwm_b200.ringattention import PeerOpsBf16, PeerOpsF16
    from peer_emulation import EmuTransport, EmuWorld

    class OldF16(PeerOpsF16):
        @staticmethod
        def fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q0, k0, causal, bias, seg, first, last, scales, out_f32):
            ra.fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q0, k0, causal, bias, seg, first, last, scales=scales,
                        out_f32=out_f32)

        @staticmethod
        def bwd_step(q, k, v, dout, lse, delta, dq, dk, dv, q0, k0, causal, bias, seg, scales, init):
            ra.bwd_step(q, k, v, dout, lse, delta, dq, dk, dv, q0, k0, causal, bias, seg, scales=scales, init=init)

    class OldBf16(PeerOpsBf16):
        @staticmethod
        def fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q0, k0, causal, bias, seg, first, last, scales, out_f32):
            ra.fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q0, k0, causal, bias, seg, first, last)
            if last and out_f32 is not None:
                out_f32.copy_(out)

        @staticmethod
        def bwd_step(q, k, v, dout, lse, delta, dq, dk, dv, q0, k0, causal, bias, seg, scales, init):
            ra.bwd_step(q, k, v, dout, lse, delta, dq, dk, dv, q0, k0, causal, bias, seg, init=init)

    world, Sl, B, H = 2, 512, 2, 2
    S = world * Sl
    dev = torch.device("cuda", 0)
    g = torch.Generator().manual_seed(19)
    q, k, v, do = [torch.randn(B, S, H, 128, generator=g).to(torch.bfloat16) for _ in range(4)]
    passes = []
    for kind in ("docs", "pad"):
        bias, seg = _masks(kind, B, S)
        for ops in (PeerOpsF16, OldF16, PeerOpsBf16, OldBf16):
            passes.append((kind, ops, bias, seg))
    emu = EmuWorld(world, device=dev)
    results, fails = {}, []

    def worker(rank):
        try:
            torch.cuda.set_device(dev)
            tr = EmuTransport(emu, rank)
            plan = rs.make_peer_plan(world, rank, Sl, Sl, True, "zigzag")
            sl = slice(rank * Sl, (rank + 1) * Sl)
            mine = []
            for kind, ops, bias, seg in passes:
                ql, kl, vl, dl = [t[:, sl].to(dev).contiguous() for t in (q, k, v, do)]
                out, res = rp.run_forward(plan, ql, kl, vl, bias, seg, True, ops, tr, False)
                dq, dk, dv = rp.run_backward(plan, res, kl, vl, dl, bias, seg, True, ops, tr, False)
                mine.append((out, dq, dk, dv))
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
        for i in range(0, len(passes), 2):
            new, old = results[r][i], results[r][i + 1]
            assert torch.equal(new[0], old[0]) and torch.equal(new[2], old[2]) and torch.equal(new[3], old[3]), (r, i)
            dq_err = float((new[1].float() - old[1].float()).abs().max())
            assert dq_err <= 1e-2 * float(old[1].float().abs().max()), (r, i, dq_err)
