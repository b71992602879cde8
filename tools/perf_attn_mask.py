"""Device-side timing of the training tile kernels under masks, with and without the block map (lwm_attn_step_tilemap).

One GPU, B = 1, H = 32, causal, single step (q_pos0 = k_pos0 = 0), S = 32768 and 131072, both precision modes. Per mask
it alternates the entry points without a map (the per-element path) and the map entry points in one process, checks that
they agree bit for bit (out, out_f32, lse, dK, dV; dQ up to the order of its fp32 reductions) and prints one line per
(S, mode, mask): the fraction of visible tiles counted from the map, ms per kernel (median of the alternating rounds;
the map build is timed on its own and included in "map" times), and TFLOP/s over the VISIBLE algorithmic FLOPs (4 D H
per visible (q, k) pair forward, 2.5x that backward). The card and its power limit are read in the same run.

usage: python tools/perf_attn_mask.py [--sizes 32768,131072] [--modes fp16,bf16] [--rounds 3] [--json OUT]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from lwm_b200 import ringattention as ra  # noqa: E402

H, D = 32, 128
FMIN = float(np.finfo(np.float32).min)
MASKS = ("none", "callsite", "docs4k", "docs1-16k", "pad25", "pad50")


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)


def make_mask(kind, S):
    """-> (bias [1,S] f32 or None, seg [1,S] i32 or None, run_start [S] (start of each row's document), npad)"""
    run_start = np.zeros(S, np.int64)
    bias = seg = None
    npad = 0
    if kind == "callsite":
        bias, seg = np.zeros((1, S), np.float32), np.zeros((1, S), np.int32)
    elif kind.startswith("docs"):
        rng = np.random.default_rng(1234)
        seg = np.zeros((1, S), np.int32)
        p, i = 0, 0
        while p < S:
            n = 4096 if kind == "docs4k" else int(rng.integers(1, 16384 + 1))
            seg[0, p:p + n] = i
            run_start[p:p + n] = p
            p, i = p + n, i + 1
    elif kind.startswith("pad"):
        npad = S * int(kind[3:]) // 100
        bias = np.zeros((1, S), np.float32)
        bias[0, :npad] = FMIN
    dev = lambda x: None if x is None else torch.from_numpy(x).cuda()  # noqa: E731
    return dev(bias), dev(seg), run_start, npad


def visible_pairs(S, run_start, npad):
    """causal (q, k) pairs with k in the row's document, k >= npad (left padding keys are masked)"""
    q = np.arange(S, dtype=np.int64)
    lo = np.maximum(run_start, npad)
    return int(np.maximum(q - lo + 1, 0)[q >= npad].sum())


def time_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def run(S, mode, kinds, rounds):
    B = 1
    g = torch.Generator(device="cuda").manual_seed(S)
    q, k, v, do = [torch.randn(B, S, H, D, device="cuda", generator=g).to(torch.bfloat16) for _ in range(4)]
    fs = bs = None
    if mode == "fp16":
        (q, sq), (k, sk), (v, sv), (do, sd) = [ra.to_f16(t) for t in (q, k, v, do)]
        fs, bs = (sq, sk, sv), (sq, sk, sv, sd)
    iters = 1 if S > 65536 else 4
    n_qt = S // 128
    full_f = n_qt * (n_qt + 1) // 2
    full_b = sum(min(S // 64, S // 64 - 2 * kt) for kt in range(S // 128))
    rows = []
    for kind in kinds:
        bias, seg, run_start, npad = make_mask(kind, S)
        pairs = visible_pairs(S, run_start, npad)
        res = {}
        if bias is None and seg is None:
            paths = [None]
            vis_f = vis_b = 1.0
            maps = None
        else:
            paths = [None, "map"]
            maps = ra.step_tilemap(B, S, S, 0, 0, True, bias, seg)
            vis_f = float(maps[1].sum()) / (B * full_f)
            vis_b = float(maps[3].sum()) / (B * full_b)
        outs = {p: (torch.empty(B, S, H, D, dtype=torch.bfloat16, device="cuda"),
                    torch.empty(B, S, H, D, device="cuda") if fs else None,
                    torch.empty(B, H, S, device="cuda")) for p in paths}
        grads = {p: [torch.zeros(B, S, H, D, device="cuda") for _ in range(3)] for p in paths}

        def fwd(p):
            out, o32, lse = outs[p]
            tm = None if p is None else ra.step_tilemap(B, S, S, 0, 0, True, bias, seg, bwd=False)[:2]
            ra.fwd_step(q, k, v, out, lse, None, None, None, 0, 0, True, bias, seg, True, True, scales=fs, out_f32=o32,
                        tilemap=tm)
        fwd(paths[0])
        out, o32, lse = outs[paths[0]]
        delta = torch.empty(B, H, S, device="cuda")
        if fs:
            ra.PeerOpsF16.bwd_prep(o32, do, bs[3], delta)
        else:
            ra.bwd_prep(out, do, delta)
        nl = ra.lse_for_bwd(lse, f16=bool(fs))

        def bwd(p):
            dq, dk, dv = grads[p]
            dq.zero_()
            tm = None if p is None else ra.step_tilemap(B, S, S, 0, 0, True, bias, seg, fwd=False)[2:]
            ra.bwd_step(q, k, v, do, nl, delta, dq, dk, dv, 0, 0, True, bias, seg, scales=bs, init=True, tilemap=tm)
        times = {(p, w): [] for p in paths for w in ("fwd", "bwd")}
        for p in paths:     # warm-up
            fwd(p)
            bwd(p)
        torch.cuda.synchronize()
        for _ in range(rounds):
            for p in paths:
                times[(p, "fwd")].append(time_ms(lambda: fwd(p), iters))
                times[(p, "bwd")].append(time_ms(lambda: bwd(p), iters))
        map_ms = time_ms(lambda: ra.step_tilemap(B, S, S, 0, 0, True, bias, seg), 4) if maps else 0.0
        ident = None
        if maps:
            fwd(None)
            fwd("map")
            bwd(None)
            dq_old = grads[None][0].clone()
            bwd(None)
            spread = float((grads[None][0] - dq_old).abs().max())
            bwd("map")
            torch.cuda.synchronize()
            a, b = outs[None], outs["map"]
            same_f = all(torch.equal(x, y) for x, y in zip(a, b) if x is not None)
            same_kv = all(torch.equal(x, y) for x, y in zip(grads[None][1:], grads["map"][1:]))
            dq_diff = float((grads[None][0] - grads["map"][0]).abs().max())
            dq_scale = float(grads[None][0].abs().max())
            ident = dict(out_lse=same_f, dk_dv=same_kv, dq_maxdiff=dq_diff, dq_spread=spread, dq_max=dq_scale,
                         dq_ok=dq_diff <= max(4 * spread, 1e-5 * dq_scale))
        med = {key: float(np.median(t)) for key, t in times.items()}
        f_vis = 4.0 * B * H * D * pairs
        row = dict(S=S, mode=mode, mask=kind, vis_tiles_fwd=vis_f, vis_tiles_bwd=vis_b, visible_pairs=pairs,
                   fwd_ms_old=med[(None, "fwd")], bwd_ms_old=med[(None, "bwd")], tilemap_ms=map_ms, identical=ident)
        if maps:
            row.update(fwd_ms_map=med[("map", "fwd")], bwd_ms_map=med[("map", "bwd")])
        rows.append(row)
        line = "S=%6d %-4s %-9s vis %.3f/%.3f  fwd %8.2f ms %6.1f TF/s" % (
            S, mode, kind, vis_f, vis_b, row["fwd_ms_old"], f_vis / row["fwd_ms_old"] / 1e9)
        line += "  bwd %8.2f ms %6.1f TF/s" % (row["bwd_ms_old"], 2.5 * f_vis / row["bwd_ms_old"] / 1e9)
        if maps:
            line += "  | map: fwd %8.2f ms %6.1f TF/s  bwd %8.2f ms %6.1f TF/s  (build %.3f ms)  identical=%s" % (
                row["fwd_ms_map"], f_vis / row["fwd_ms_map"] / 1e9, row["bwd_ms_map"],
                2.5 * f_vis / row["bwd_ms_map"] / 1e9, map_ms,
                ident["out_lse"] and ident["dk_dv"] and ident["dq_ok"])
        print(line, flush=True)
        del outs, grads
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="32768,131072")
    ap.add_argument("--modes", default="fp16,bf16")
    ap.add_argument("--masks", default=",".join(MASKS))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_attn_mask: needs a GPU")
    info = card()
    print("card: %s" % info, flush=True)
    rows = []
    for S in [int(x) for x in a.sizes.split(",")]:
        for mode in a.modes.split(","):
            rows += run(S, mode, a.masks.split(","), a.rounds)
    ok = all(r["identical"] is None or (r["identical"]["out_lse"] and r["identical"]["dk_dv"] and
                                        r["identical"]["dq_ok"]) for r in rows)
    print("all map paths bit-identical: %s" % ok)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)
    if not ok:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
