"""The training block map (lwm_attn_step_tilemap), restated in numpy (tests/tilemap_model.py), against a brute-force
per-element mask: a pair left out of a list has every entry masked, a clean pair has no mask beyond the causal one, and
a forward Q tile with a row that does not see its own key visits its whole causal range as mixed. Also the argument
checks of the map and of the step entry points given one, which run before any device is looked for."""
import ctypes

import numpy as np
import pytest
import torch

import tilemap_model as tm
from helpers import FOLDED_ENTRY_POINTS, abi_row_id, with_options

CASES = tm.sweep_cases()


def _ranges(Sq, Sk, q0, k0, causal):
    n_kt, n_q64 = Sk // 128, Sq // 64

    def fwd_range(t):
        if not causal:
            return n_kt
        vis = q0 + 128 * t + 127 - k0
        return 0 if vis < 0 else min(n_kt, vis // 128 + 1)

    def bwd_start(kt):
        if not causal:
            return 0
        d = k0 + 128 * kt - q0
        return 0 if d <= 0 else min(d // 64, n_q64)
    return fwd_range, bwd_start


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_block_map_invariants(case):
    _, bias, seg, Sq, Sk, q0, k0, causal = case
    fwd, bwd = tm.step_tilemap(bias, seg, Sq, Sk, q0, k0, causal)
    fwd_range, bwd_start = _ranges(Sq, Sk, q0, k0, causal)
    for b in range(len(fwd)):
        for t, lst in enumerate(fwd[b]):
            qpos = q0 + 128 * t + np.arange(128)
            proven = all(tm.row_proven(bias, b, int(p), k0, Sk) for p in qpos)
            ents = {e >> 1: e & 1 for e in lst}
            assert [e >> 1 for e in lst] == sorted(ents), "ascending, no repeats"
            assert all(kt < fwd_range(t) for kt in ents)
            for kt in range(fwd_range(t)):
                kpos = k0 + 128 * kt + np.arange(128)
                full, cm = tm.element_masks(bias, seg, b, qpos, kpos, causal)
                if not proven:
                    assert ents.get(kt) == 1, "an unproven Q tile visits its causal range as mixed"
                elif kt not in ents:
                    assert full.all(), "skipped pair with a visible entry"
                elif ents[kt] == 0:
                    assert (full == cm).all() and (bias is None or (bias[b, kpos] == 0).all())
        for kt, lst in enumerate(bwd[b]):
            kpos = k0 + 128 * kt + np.arange(128)
            ents = {e >> 1: e & 1 for e in lst}
            assert [e >> 1 for e in lst] == sorted(ents)
            assert all(bwd_start(kt) <= qi < Sq // 64 for qi in ents)
            for qi in range(bwd_start(kt), Sq // 64):
                qpos = q0 + 64 * qi + np.arange(64)
                full, cm = tm.element_masks(bias, seg, b, qpos, kpos, causal)
                if qi not in ents:
                    assert full.all(), "skipped pair with a visible entry"
                elif ents[qi] == 0:
                    assert (full == cm).all() and (bias is None or (bias[b, kpos] == 0).all())


def test_block_map_skips_where_it_should():
    """packed documents and left padding leave pairs out; the call-site mask (zero bias, one segment) is all clean"""
    by_name = {c[0]: c for c in CASES}
    for name in ("docs-c-0-0", "leftpad-c-0-0", "bias-nc-0-0"):
        _, bias, seg, Sq, Sk, q0, k0, causal = by_name[name]
        fwd, bwd = tm.step_tilemap(bias, seg, Sq, Sk, q0, k0, causal)
        full_f = sum(min(Sk // 128, t + 1) if causal else Sk // 128 for t in range(Sq // 128)) * len(fwd)
        assert sum(len(x) for f in fwd for x in f) < full_f, name
    G = 1024
    fwd, bwd = tm.step_tilemap(np.zeros((1, G), np.float32), np.zeros((1, G), np.int32), G, G, 0, 0, True)
    assert all(e & 1 == 0 for x in fwd[0] + bwd[0] for e in x)
    assert [len(x) for x in fwd[0]] == list(range(1, 9))


P = ctypes.c_void_p(0x1000)
N = None
SHAPE, ARG, DEVICE = 2, 3, 1

BAD_CALLS = [
    ("lwm_attn_step_tilemap", (N, 0, N, 0, 1, 256, 256, 0, 0, 1, P, P, P, P, P, N), ARG, "bias or segment_ids"),
    ("lwm_attn_step_tilemap", (P, 256, N, 0, 1, 256, 256, 0, 0, 1, P, N, P, P, P, N), ARG, "null"),
    ("lwm_attn_step_tilemap", (P, 256, N, 0, 1, 256, 256, 0, 0, 1, N, N, N, N, P, N), ARG, "null"),
    ("lwm_attn_step_tilemap", (P, 256, N, 0, 1, 256, 256, 0, 0, 1, P, P, P, P, N, N), ARG, "null"),
    ("lwm_attn_step_tilemap", (P, 256, N, 0, 1, 200, 256, 0, 0, 1, P, P, P, P, P, N), SHAPE, "multiples of 128"),
    ("lwm_attn_step_tilemap", (P, 256, N, 0, 0, 256, 256, 0, 0, 1, P, P, P, P, P, N), SHAPE, "multiples of 128"),
    ("lwm_attn_step_tilemap", (P, 256, N, 0, 1, 256, 256, -128, 0, 1, P, P, P, P, P, N), SHAPE, "positions"),
    ("lwm_attn_step_tilemap", (P, 256, N, 0, 1, 256, 256, 0, 1 << 31, 1, P, P, P, P, P, N), SHAPE, "positions"),
    ("lwm_attn_step_tilemap", (P, 256, N, 0, 1, 256, 256, 0, 128, 1, P, P, P, P, P, N), SHAPE, "bias_stride"),
    ("lwm_attn_step_tilemap", (N, 0, P, 256, 1, 256, 256, 128, 0, 1, P, P, P, P, P, N), SHAPE, "seg_stride"),
    # lwm_attn_fwd_step(q, k, v, scale_q, scale_k, scale_v, out_f32, out, lse, acc_o, acc_m, acc_l, B, H, Sq, Sk, D,
    #                   q_pos0, k_pos0, causal, bias, bias_stride, segment_ids, seg_stride, softmax_scale, first, last,
    #                   tiles, tile_count, seed, drop_threshold, batch0, stream)
    ("lwm_attn_fwd_step", (P, P, P, N, N, N, N, P, P, N, N, N, 1, 2, 128, 128, 128, 0, 0, 1, N, 0, N, 0, 0.1, 1, 1,
                           P, P, 0, 0, 0, N), ARG, "bias or segment_ids"),
    ("lwm_attn_fwd_step", (P, P, P, N, N, N, N, P, P, N, N, N, 1, 2, 128, 128, 128, 0, 0, 1, P, 128, N, 0, 0.1, 1, 1,
                           N, P, 0, 0, 0, N), ARG, "tiles"),
    ("lwm_attn_fwd_step", (P, P, P, N, N, N, N, P, P, N, N, N, 1, 2, 128, 128, 128, 0, 0, 1, P, 64, N, 0, 0.1, 1, 1,
                           P, P, 0, 0, 0, N), SHAPE, "bias_stride"),
    ("lwm_attn_fwd_step", (P, P, P, N, N, N, N, P, P, N, N, N, 1, 2, 100, 128, 128, 0, 0, 1, P, 128, N, 0, 0.1, 1, 1,
                           P, P, 0, 0, 0, N), SHAPE, "multiples of 128"),
    ("lwm_attn_fwd_step", (P, P, P, N, P, P, N, P, P, N, N, N, 1, 2, 128, 128, 128, 0, 0, 1, P, 128, N, 0, 0.1, 1, 1,
                           P, P, 0, 0, 0, N), ARG, "scales"),
    ("lwm_attn_fwd_step", (P, P, P, P, P, P, N, P, P, N, N, N, 1, 2, 128, 128, 128, 0, 0, 1, N, 0, P, 128, 0.1, 1, 1,
                           P, N, 0, 0, 0, N), ARG, "tiles"),
    # lwm_attn_bwd_step(q, k, v, dout, scale_q, scale_k, scale_v, scale_do, lse, delta, dq_acc, dk_acc, dv_acc, B, H, Sq,
    #                   Sk, D, q_pos0, k_pos0, causal, bias, bias_stride, segment_ids, seg_stride, softmax_scale,
    #                   dkv_init, tiles, tile_count, order_ws, seed, drop_threshold, batch0, stream)
    ("lwm_attn_bwd_step", (P, P, P, P, N, N, N, N, P, P, P, P, P, 1, 2, 128, 128, 128, 0, 0, 1, N, 0, N, 0, 0.1, 1,
                           P, P, N, 0, 0, 0, N), ARG, "bias or segment_ids"),
    ("lwm_attn_bwd_step", (P, P, P, P, N, N, N, N, P, P, P, P, P, 1, 2, 128, 128, 128, 0, 0, 1, N, 0, P, 128, 0.1, 1,
                           P, N, N, 0, 0, 0, N), ARG, "tiles"),
    ("lwm_attn_bwd_step", (P, P, P, P, N, N, N, N, P, P, P, P, P, 1, 2, 128, 128, 128, 128, 0, 1, N, 0, P, 128, 0.1, 1,
                           P, P, N, 0, 0, 0, N), SHAPE, "seg_stride"),
    ("lwm_attn_bwd_step", (P, P, P, P, P, P, P, N, P, P, P, P, P, 1, 2, 128, 128, 128, 0, 0, 1, P, 128, N, 0, 0.1, 1,
                           P, P, N, 0, 0, 0, N), ARG, "scales"),
    ("lwm_attn_bwd_step", (P, P, P, P, P, P, P, P, P, P, P, P, P, 1, 2, 128, 128, 128, 0, 0, 1, P, 128, N, 0, 0.1, 1,
                           N, P, N, 0, 0, 0, N), ARG, "tiles"),
]

# the same rows with the options of the folded entry points turned on: no option slot bypasses these checks
BAD_CALLS += [(n, with_options(n, a, P), c, f) for n, a, c, f in BAD_CALLS if n in FOLDED_ENTRY_POINTS]


def _status(lib, name, *args):
    from lwm_b200 import _lib
    _lib.load()
    return getattr(lib, name)(*args), lib.lwm_last_error().decode()


@pytest.mark.parametrize("name,args,code,frag", BAD_CALLS,
                         ids=["%s-%d-%s" % (abi_row_id(*c[:2]), i, c[3].replace(" ", "_")) for i, c in enumerate(BAD_CALLS)])
def test_map_entry_points_reject_bad_arguments(lib, name, args, code, frag):
    status, msg = _status(lib, name, *args)
    assert status == code, (status, msg)
    assert frag in msg, msg


GOOD_CALLS = [
    ("lwm_attn_step_tilemap", (P, 256, N, 0, 1, 256, 256, 0, 0, 1, P, P, P, P, P, N)),
    ("lwm_attn_step_tilemap", (N, 0, P, 512, 2, 256, 256, 256, 0, 1, N, N, P, P, P, N)),
    ("lwm_attn_fwd_step", (P, P, P, N, N, N, N, P, P, N, N, N, 1, 2, 128, 128, 128, 0, 0, 1, P, 128, N, 0, 0.1, 1, 1,
                           P, P, 0, 0, 0, N)),
    ("lwm_attn_fwd_step", (P, P, P, P, P, P, N, P, P, N, N, N, 1, 2, 128, 128, 128, 0, 0, 1, N, 0, P, 128, 0.1, 1, 1,
                           P, P, 0, 0, 0, N)),
    ("lwm_attn_bwd_step", (P, P, P, P, N, N, N, N, P, P, P, P, P, 1, 2, 128, 128, 128, 0, 0, 1, P, 128, N, 0, 0.1, 1,
                           P, P, N, 0, 0, 0, N)),
    ("lwm_attn_bwd_step", (P, P, P, P, P, P, P, P, P, P, P, P, P, 1, 2, 128, 128, 128, 0, 0, 1, N, 0, P, 128, 0.1, 0,
                           P, P, N, 0, 0, 0, N)),
]

GOOD_CALLS += [(n, with_options(n, a, P)) for n, a in GOOD_CALLS if n in FOLDED_ENTRY_POINTS]


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: only meaningful where the device check fails")
@pytest.mark.parametrize("name,args", GOOD_CALLS, ids=["%s-%d" % (abi_row_id(*c), i) for i, c in enumerate(GOOD_CALLS)])
def test_well_formed_map_calls_fail_with_device_error_without_gpu(lib, name, args):
    status, msg = _status(lib, name, *args)
    assert status == DEVICE, (status, msg)
