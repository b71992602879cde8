"""Attention dropout without a GPU: the numpy Philox4x32-10 against Random123's known-answer vectors, the threshold and
the statistics of the mask, blockwise_kwargs handling, argument checks of the three C symbols, both ring executors'
host logic with the CPU stand-ins against the float64 oracle under the same mask, and the dropout instances' SASS."""
import ctypes
import os
import re
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from attn_dropout_model import (CpuDropoutOps, attention_dropout_ref, drop_mask, drop_u16,  # noqa: E402
                                philox4x32_10, threshold)
from test_attn_fwd_schedule_cpu import _cuobjdump  # noqa: E402

LIB = os.path.join(ROOT, "lwm_b200", "lib", "liblwm_b200.so")


# ------------------------------------------------------------------------------------------------ the generator
@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    got = tuple(int(w) for w in philox4x32_10([np.uint32(c) for c in ctr], key))
    assert got == want, [hex(x) for x in got]


def test_threshold_rounding():
    from lwm_b200.ringattention import dropout_threshold
    for p, thr in ((0.0, 0), (0.1, 6554), (0.5, 32768), (0.25, 16384), (1 - 2 ** -20, 65535), (2 ** -18, 0),
                   (2 ** -16, 1), (0.999, 65470)):
        assert dropout_threshold(p) == threshold(p) == thr, p
        assert abs(thr / 65536 - p) <= 2 ** -17 or thr == 65535


def _u16_sample():
    """> 10^7 draws: 3200 queries x 3200 keys of one (b, h), at positions past 2^20"""
    qp = (1 << 20) - 1600 + np.arange(3200)
    return drop_u16(0x0123456789ABCDEF, 1, 3, qp, 77 * 128 + np.arange(3200))


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_drop_rate_within_five_sigma(p):
    u = _u16_sample()
    thr = threshold(p)
    rate = thr / 65536
    n = u.size
    assert n >= 10 ** 7
    got = float((u < thr).mean())
    assert abs(got - rate) < 5 * np.sqrt(rate * (1 - rate) / n), (got, rate)


def _chi2(a, b):
    """Pearson chi-square (1 degree of freedom) of the 2x2 table of two bool arrays"""
    t = np.array([[np.sum(a & b), np.sum(a & ~b)], [np.sum(~a & b), np.sum(~a & ~b)]], dtype=np.float64)
    e = t.sum(1, keepdims=True) * t.sum(0, keepdims=True) / t.sum()
    return float(((t - e) ** 2 / e).sum())


def test_neighbours_are_independent():
    """2x2 contingency of the decisions of neighbouring keys, rows, heads and batch rows (p = 0.1 and 0.5): chi-square
    below 30 (p-value ~4e-8 under independence; the mask is a fixed function of the seed, so this never flakes)"""
    seed, qp, kp = 987654321, 5000 + np.arange(1024), 4096 + np.arange(1024)
    for p in (0.1, 0.5):
        thr = threshold(p)
        base = drop_u16(seed, 2, 5, qp, kp) < thr
        pairs = {
            "key": (base[:, 0::2], base[:, 1::2]),
            "row": (base[0::2], base[1::2]),
            "head": (base, drop_u16(seed, 2, 6, qp, kp) < thr),
            "batch": (base, drop_u16(seed, 3, 5, qp, kp) < thr),
        }
        for name, (a, b) in pairs.items():
            assert _chi2(a, b) < 30, (p, name, _chi2(a, b))


# ------------------------------------------------------------------------------------------------ arguments
def test_blockwise_kwargs():
    from lwm_b200.ringattention import _check_blockwise_kwargs as chk
    assert chk(None, 256, 256) == (False, None)
    assert chk(dict(causal_block_size=1, deterministic=True, attn_pdrop=0.3, dropout_rng=5), 256, 256) == (True, None)
    assert chk(dict(deterministic=False, attn_pdrop=0.0, dropout_rng=5), 256, 256) == (False, None)
    assert chk(dict(deterministic=False, attn_pdrop=2 ** -18, dropout_rng=5), 256, 256) == (False, None)
    assert chk(dict(deterministic=False, attn_pdrop=0.1, dropout_rng=5), 256, 256) == (False, (5, 6554))
    assert chk(dict(deterministic=False, attn_pdrop=0.1, dropout_rng=2 ** 64 - 1), 256, 256)[1] == (-1, 6554)
    assert chk(dict(deterministic=False, attn_pdrop=0.1, dropout_rng=-3), 256, 256, world=4)[1] == (-3, 6554)
    for p in (1.0, 1.5, -0.1, float("nan")):
        with pytest.raises(ValueError):
            chk(dict(deterministic=False, attn_pdrop=p, dropout_rng=1), 256, 256)
        with pytest.raises(ValueError):
            chk(dict(deterministic=True, attn_pdrop=p), 256, 256)
    for rng in (1.5, "7", True, np.bool_(True), torch.tensor(True), torch.tensor(3.0), [3]):
        with pytest.raises(TypeError):
            chk(dict(deterministic=False, attn_pdrop=0.1, dropout_rng=rng), 256, 256)
    for rng in (np.int64(3), np.uint64(3), torch.tensor(3)):      # integer-like seeds
        assert chk(dict(deterministic=False, attn_pdrop=0.1, dropout_rng=rng), 256, 256)[1] == (3, 6554)
    with pytest.raises(ValueError):
        chk(dict(deterministic=False, attn_pdrop=0.1, dropout_rng=None), 256, 256, world=2)
    # None on one GPU: a seed from torch's default CPU generator, reproduced by torch.manual_seed
    torch.manual_seed(11)
    a = chk(dict(deterministic=False, attn_pdrop=0.1), 256, 256)[1]
    torch.manual_seed(11)
    b = chk(dict(deterministic=False, attn_pdrop=0.1, dropout_rng=None), 256, 256)[1]
    assert a == b and -2 ** 63 <= a[0] < 2 ** 63


def _fwd_args(**kw):
    """lwm_attn_fwd_step's arguments with dropout on (fake non-null pointers), overridable by name"""
    a = dict(q=1, k=1, v=1, sq=None, sk=None, sv=None, o32=None, out=1, lse=1, ao=None, am=None, al=None, B=1, H=1,
             Sq=256, Sk=256, D=128, q_pos0=0, k_pos0=0, causal=1, bias=None, bias_stride=0, seg=None, seg_stride=0,
             scale=0.088, first=1, last=1, tiles=None, counts=None, seed=7, thr=6554, batch0=0, stream=None)
    a.update(kw)
    return list(a.values())


def _bwd_args(**kw):
    a = dict(q=1, k=1, v=1, do=1, sq=None, sk=None, sv=None, sdo=None, lse=1, delta=1, dq=1, dk=1, dv=1, B=1, H=1,
             Sq=256, Sk=256, D=128, q_pos0=0, k_pos0=0, causal=1, bias=None, bias_stride=0, seg=None, seg_stride=0,
             scale=0.088, init=1, tiles=None, counts=None, ws=None, seed=7, thr=6554, batch0=0, stream=None)
    a.update(kw)
    return list(a.values())


def _mask_args(**kw):
    a = dict(seed=7, thr=6554, b=0, h=0, q_pos0=0, k_pos0=0, n_q=4, n_k=4, out=1, stream=None)
    a.update(kw)
    return list(a.values())


def _status(lib, name, args):
    from lwm_b200 import _lib
    fn = getattr(lib, name)
    fn.argtypes = _lib._SIGNATURES[name]
    ptrs = [ctypes.c_void_p(a) if t is ctypes.c_void_p and a is not None else a
            for a, t in zip(args, _lib._SIGNATURES[name])]
    return fn(*ptrs), lib.lwm_last_error().decode()


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: only meaningful where the device check fails")
def test_step_entry_points_check_dropout_arguments_before_the_device(lib):
    cases = [
        ("lwm_attn_fwd_step", _fwd_args(q_pos0=64), 2, "multiple of 128"),       # accepted without dropout (below)
        ("lwm_attn_fwd_step", _fwd_args(thr=65536), 3, "drop_threshold"),
        ("lwm_attn_fwd_step", _fwd_args(k_pos0=64), 2, "multiple of 128"),
        ("lwm_attn_fwd_step", _fwd_args(q_pos0=128 + 8), 2, "multiple of 128"),
        ("lwm_attn_fwd_step", _fwd_args(batch0=-1), 3, "batch0"),
        ("lwm_attn_fwd_step", _fwd_args(batch0=2 ** 31 - 1), 2, "batch0 + B"),
        ("lwm_attn_fwd_step", _fwd_args(Sq=100), 2, "multiples of 128"),
        ("lwm_attn_fwd_step", _fwd_args(tiles=1), 3, "tiles and tile_count"),
        ("lwm_attn_bwd_step", _bwd_args(batch0=2 ** 31 - 1), 2, "batch0 + B"),  # accepted without dropout (below)
        ("lwm_attn_bwd_step", _bwd_args(thr=70000), 3, "drop_threshold"),
        ("lwm_attn_bwd_step", _bwd_args(k_pos0=128 + 16), 2, "multiple of 128"),
        ("lwm_attn_bwd_step", _bwd_args(q_pos0=64), 2, "multiple of 128"),
        ("lwm_attn_bwd_step", _bwd_args(batch0=-5), 3, "batch0"),
        ("lwm_attn_bwd_step", _bwd_args(dq=None), 3, "null pointer"),
        ("lwm_attn_dropout_mask", _mask_args(thr=0), 3, "drop_threshold"),
        ("lwm_attn_dropout_mask", _mask_args(out=None), 3, "null out"),
        ("lwm_attn_dropout_mask", _mask_args(n_q=0), 2, "n_q"),
        ("lwm_attn_dropout_mask", _mask_args(k_pos0=2 ** 31 - 2), 2, "positions"),
    ]
    for name, args, code, msg in cases:
        st, err = _status(lib, name, args)
        assert st == code and msg in err, (name, st, err)
    for name, args in (("lwm_attn_fwd_step", _fwd_args(k_pos0=256, q_pos0=384, batch0=3)),
                       ("lwm_attn_bwd_step", _bwd_args(ws=1, thr=65535, batch0=1)),
                       # drop_threshold 0 is the call without dropout: the dropout-only shape rules do not apply
                       ("lwm_attn_fwd_step", _fwd_args(q_pos0=64, thr=0)),
                       ("lwm_attn_bwd_step", _bwd_args(batch0=2 ** 31 - 1, thr=0)),
                       ("lwm_attn_dropout_mask", _mask_args(b=3, h=31, q_pos0=2 ** 20))):
        st, err = _status(lib, name, args)
        assert st == 1, (name, st, err)     # LWM_ERR_DEVICE: the arguments were accepted


# ------------------------------------------------------------------------------------------------ executors
def _inputs(world, B=1, H=2, D=16, Sl=256):
    from oracle.attn_dense import finfo_min
    S = Sl * world
    g = torch.Generator().manual_seed(1234)
    q, k, v, do = [torch.randn(B, S, H, D, generator=g) for _ in range(4)]
    bias = torch.zeros(B, S)
    bias[0, :37] = finfo_min("fp32")
    seg = torch.zeros(B, S, dtype=torch.int32)
    seg[0, S // 2 + 5:] = 1
    seg[B - 1, S // 4 + 3:] = 2
    return q, k, v, do, bias, seg


def _refs(q, k, v, do, bias, seg, dropout):
    B, S, H, _ = q.shape
    drop = drop_mask(dropout[0], dropout[1], B, H, 0, S, 0, S)
    return attention_dropout_ref(q.numpy(), k.numpy(), v.numpy(), do.numpy(), drop, attn_bias=bias.numpy(),
                                 segment_ids=seg.numpy(), causal=True)


def _rel(x, r):
    return float(np.linalg.norm(x - r) / max(np.linalg.norm(r), 1e-30))


def _gloo_worker(rank, world, port, layout, dropout, B, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from lwm_b200 import ring_exec as rx, ring_schedule as rs
        from lwm_b200.ringattention import with_dropout
        from attn_dropout_model import CpuDropoutOps as Ops
        q, k, v, do, bias, seg = _inputs(world, B)
        Sl = q.shape[1] // world
        sl = slice(rank * Sl, (rank + 1) * Sl)
        ops = with_dropout(Ops, dropout)
        loc = [t[:, sl].contiguous() for t in (q, k, v, do)]
        plan = rs.make_plan(world, rank, Sl, Sl, True, layout)
        out, res = rx.run_forward(plan, *loc[:3], bias, seg, True, None, ops)
        plan = rs.make_plan(world, rank, Sl, Sl, True, layout, n_sub_first=2, n_sub_last=2)
        dq, dk, dv = rx.run_backward(plan, res, loc[1], loc[2], loc[3], bias, seg, True, None, ops)
        ret[rank] = [t.double().numpy() for t in (out, dq, dk, dv)]
    finally:
        dist.destroy_process_group()


def _free_port():
    import socket
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _check_world(world, got, dropout, tol, B):
    ref = _refs(*_inputs(world, B), dropout)
    live = ref[4]
    Sl = ref[0].shape[1] // world
    assert (~live).any() and live.mean() > 0.9     # dead rows (padding, and rows whose every key was dropped) occur
    for r in range(world):
        sl = slice(r * Sl, (r + 1) * Sl)
        for j, (x, rf) in enumerate(zip(got[r], ref[:4])):
            e = _rel(x, rf[:, sl])
            assert e < tol, (r, j, e)
        assert np.all(got[r][0][~live[:, :, sl].transpose(0, 2, 1)] == 0)   # rows without a surviving key: out = 0


@pytest.mark.parametrize("world,layout,B", [(2, "contiguous", 1), (2, "zigzag", 2), (4, "zigzag", 1),
                                            (4, "contiguous", 2)])
def test_nccl_executor_with_dropout_matches_oracle(world, layout, B):
    dropout = (0x5EED0000 + world, threshold(0.3))
    ret = mp.Manager().dict()
    mp.spawn(_gloo_worker, args=(world, _free_port(), layout, dropout, B, ret), nprocs=world, join=True)
    assert len(ret) == world
    _check_world(world, dict(ret), dropout, 1e-5, B)


@pytest.mark.parametrize("world,layout,B", [(2, "zigzag", 2), (4, "contiguous", 1), (4, "zigzag", 2)])
def test_peer_executor_with_dropout_matches_oracle(world, layout, B):
    """the peer executor launches one batch row at a time: with B = 2 each row must still draw its own mask"""
    from lwm_b200 import ring_peer as rp, ring_schedule as rs
    from lwm_b200.ringattention import with_dropout
    from peer_emulation import EmuOps, EmuTransport, EmuWorld

    class EmuDropoutOps(EmuOps):
        """EmuOps over the dropout stand-ins (scales folded in as EmuOps does)"""

        def fwd_step(self, q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last,
                     scales, out_f32, dropout=None):
            sq, sk, sv = [1.0 if s is None else s for s in scales]
            if last and out_f32 is not None:      # the un-rounded output first: `out` is the emulated kernel's bf16
                tmp = torch.empty(out.shape, dtype=torch.float64)
                CpuDropoutOps.fwd_step(q * sq, k * sk, v * sv, tmp, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal,
                                       bias, seg, first, last, dropout=dropout)
                out_f32.copy_(tmp)
            CpuDropoutOps.fwd_step(q * sq, k * sk, v * sv, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias,
                                   seg, first, last, dropout=dropout)

        def bwd_step(self, q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg,
                     scales, init, dropout=None):
            sq, sk, sv, sdo = [1.0 if s is None else s for s in scales]
            if init:
                dk_acc.zero_()
                dv_acc.zero_()
            CpuDropoutOps.bwd_step(q * sq, k * sk, v * sv, dout * sdo, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0,
                                   k_pos0, causal, bias, seg, dropout=dropout)

    dropout = (-12345, threshold(0.3))
    emu = EmuWorld(world)
    q, k, v, do, bias, seg = _inputs(world, B)
    Sl = q.shape[1] // world
    got, fails = {}, []

    def worker(rank):
        try:
            tr = EmuTransport(emu, rank)
            ops = with_dropout(EmuDropoutOps(True), dropout)
            sl = slice(rank * Sl, (rank + 1) * Sl)
            plan = rs.make_peer_plan(world, rank, Sl, Sl, True, layout, fwd_group_chunks=2)
            loc = [t[:, sl].contiguous() for t in (q, k, v, do)]
            out, res = rp.run_forward(plan, *loc[:3], bias, seg, True, ops, tr, True)
            dq, dk, dv = rp.run_backward(plan, res, loc[1], loc[2], loc[3], bias, seg, True, ops, tr, True)
            got[rank] = [t.double().numpy() for t in (out, dq, dk, dv)]
        except BaseException:   # noqa: BLE001  (propagated to the main thread)
            import traceback
            fails.append(traceback.format_exc())
            emu.barrier.abort()

    ts = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=300)
    assert not fails, fails[0]
    _check_world(world, got, dropout, 2e-5, B)


# ------------------------------------------------------------------------------------------------ SASS
# attn_fwd_dropout_kernel<kF16, kMap>, attn_bwd_dropout_kernel<kF16, kMap, kOrdered>
_FWD = "_ZN3lwm23attn_fwd_dropout_kernelILb%dELb%dEEEv14CUtensorMap_stS1_S1_NS_9FwdParamsE"
_BWD = "_ZN3lwm23attn_bwd_dropout_kernelILb%dELb%dELb%dEEEv14CUtensorMap_stS1_S1_S1_S1_NS_9BwdParamsE"
DROPOUT_INSTANCES = ([_FWD % (f, m) for f in (0, 1) for m in (0, 1)]
                     + [_BWD % (f, m, o) for f in (0, 1) for m in (0, 1) for o in (0, 1)])


def test_dropout_instances_keep_everything_in_registers():
    tool = _cuobjdump()
    if tool is None or not os.path.exists(LIB):
        pytest.skip("needs cuobjdump and the built liblwm_b200.so")
    r = subprocess.run([tool, "-sass", "-fun", ",".join(DROPOUT_INSTANCES), LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    fns, cur = {}, None
    for line in r.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = fns.setdefault(m.group(1), [])
        elif cur is not None and re.search(r"/\*[0-9a-f]{4,}\*/", line):
            cur.append(line)
    assert sorted(fns) == sorted(DROPOUT_INSTANCES)
    for name, insns in fns.items():
        assert len(insns) > 1000, name
        local = [t for t in insns if re.search(r"\b(LDL|STL)\b", t)]
        assert not local, (name, local[:4])
