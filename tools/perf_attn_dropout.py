"""Device-side cost of attention dropout in the training tile kernels.

One GPU, B = 1, H = 32, causal, single step (q_pos0 = k_pos0 = 0), S = 32768 and 131072, both precision modes, with the
call site's zero bias (the block-map kernels) and without a mask (the plain kernels). Per configuration it alternates
p = 0 and p = 0.1 (lwm_attn_fwd_step / lwm_attn_bwd_step with drop_threshold 0 and 6554) in one process, times each
step with CUDA events and prints one JSON line: ms per kernel (median of the alternating rounds) and the ratio. The card, its
power limit and SM clock are read in the same run.

usage: python tools/perf_attn_dropout.py [--sizes 32768,131072] [--modes fp16,bf16] [--rounds 3] [--json OUT]"""
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


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    return r.stdout.strip().splitlines()[0]


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def run(S, mode, mask, rounds, drop):
    f16 = mode == "fp16"
    g = torch.Generator(device="cuda").manual_seed(S)
    q, k, v, do = [torch.randn(1, S, H, D, generator=g, device="cuda").to(torch.bfloat16) for _ in range(4)]
    bias = torch.zeros(1, S, device="cuda") if mask == "callsite" else None
    fmap = bmap = None
    if bias is not None:
        ft, fc, bt, bc = ra.step_tilemap(1, S, S, 0, 0, True, bias, None)
        fmap, bmap = (ft, fc), (bt, bc)
    fkw, bkw = {}, {}
    if f16:
        (q, sq), (k, sk), (v, sv), (do, sd) = [ra.to_f16(t) for t in (q, k, v, do)]
        o32 = torch.empty(1, S, H, D, device="cuda")
        fkw, bkw = dict(scales=(sq, sk, sv), out_f32=o32), dict(scales=(sq, sk, sv, sd))
    out = torch.empty(1, S, H, D, dtype=torch.bfloat16, device="cuda")
    lse = torch.empty(1, H, S, device="cuda")
    delta = torch.empty(1, H, S, device="cuda")
    dq, dk, dv = [torch.zeros(1, S, H, D, device="cuda") for _ in range(3)]

    def fwd(dropout):
        ra.fwd_step(q, k, v, out, lse, None, None, None, 0, 0, True, bias, None, 1, 1, tilemap=fmap, dropout=dropout,
                    **fkw)

    fwd(None)
    ra.bwd_prep(o32 if f16 else out, do, delta, scale_do=sd if f16 else None)
    nlse = ra.lse_for_bwd(lse, f16=f16)

    def bwd(dropout):
        ra.bwd_step(q, k, v, do, nlse, delta, dq, dk, dv, 0, 0, True, bias, None, init=True, tilemap=bmap,
                    dropout=dropout, **bkw)

    reps = max(1, 131072 // S) * 2
    for d in (None, drop):       # warm-up: module loads, attributes
        fwd(d)
        bwd(d)
    torch.cuda.synchronize()
    t = {key: [] for key in ("fwd0", "fwdp", "bwd0", "bwdp")}
    for _ in range(rounds):
        t["fwd0"].append(timed(lambda: fwd(None), reps))
        t["fwdp"].append(timed(lambda: fwd(drop), reps))
        t["bwd0"].append(timed(lambda: bwd(None), reps))
        t["bwdp"].append(timed(lambda: bwd(drop), reps))
    med = {key: float(np.median(val)) for key, val in t.items()}
    return dict(S=S, mode=mode, mask=mask, fwd_ms_p0=round(med["fwd0"], 3), fwd_ms_p01=round(med["fwdp"], 3),
                fwd_ratio=round(med["fwdp"] / med["fwd0"], 3), bwd_ms_p0=round(med["bwd0"], 3),
                bwd_ms_p01=round(med["bwdp"], 3), bwd_ratio=round(med["bwdp"] / med["bwd0"], 3),
                rounds=rounds, reps=reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="32768,131072")
    ap.add_argument("--modes", default="fp16,bf16")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_attn_dropout: needs a GPU")
    drop = (0x5EED, ra.dropout_threshold(0.1))
    lines = [dict(card=card(), p=0.1, thr=drop[1])]
    print(json.dumps(lines[0]), flush=True)
    for S in [int(x) for x in a.sizes.split(",")]:
        for mode in a.modes.split(","):
            for mask in ("none", "callsite"):
                r = run(S, mode, mask, a.rounds, drop)
                lines.append(r)
                print(json.dumps(r), flush=True)
                torch.cuda.empty_cache()
    lines.append(dict(card_after=card()))
    print(json.dumps(lines[-1]), flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
