"""Time `ringattention` with the rotary embedding folded into its operand passes (freqs_cis=, position_ids=) against the
composition `ringattention(*apply_rotary_emb(q, k, ...), v, ...)`, on one GPU.

B = 1, H = 32, D = 128, fp16 precision mode, the LWM call-site bias (attention_bias_from_mask of an all-ones mask, i.e.
zeros), causal, bf16 and fp32 inputs. The two variants run alternately, step by step; every step is one forward and one
backward, timed with CUDA events (forward, backward, and the two together), and torch.cuda.max_memory_allocated is
reset before each step. Medians over the rounds are reported, with the bytes of HBM traffic the fusion removes as
counted from shapes (not measured):
  forward   the rotation pass reads q and k and writes their rotated copies, which the staging passes then read: one
            read and one write of q and k go away;
  backward  bf16: the rotation pass reads the cast dQ / dK and writes them again: one read and one write of dQ and dK go
            away. fp32: the conjugate rotation replaces the pass the composition makes over the fp32 accumulators, so
            the bytes are the same.
The first step of each variant checks that both give the same out, dK and dV, bit for bit.
The card and its power limit are read in the same run.

usage: python tools/perf_rope_attn.py [--sizes 8192,32768,131072] [--dtypes bf16,fp32] [--rounds 5] [--json OUT]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lwm_b200 import ringattention as ra  # noqa: E402
from lwm_b200 import rope  # noqa: E402

H, D = 32, 128
KW = dict(axis_name="sp", blockwise_kwargs=dict(causal_block_size=1), precision="fp16")
DT = {"bf16": torch.bfloat16, "fp32": torch.float32}


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)


def removed_bytes(S, dtype):
    n = S * H * D
    isz = torch.empty((), dtype=dtype).element_size()
    fwd = 2 * 2 * n * isz                          # q and k: one read + one write each
    bwd = 2 * 2 * n * isz if dtype == torch.bfloat16 else 0
    return fwd, bwd


def step(q, k, v, do, bias, pos, table, fused):
    q, k, v = [t.detach().requires_grad_(True) for t in (q, k, v)]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    e[0].record()
    if fused:
        out = ra.ringattention(q, k, v, bias, None, freqs_cis=table, position_ids=pos, **KW)
    else:
        out = ra.ringattention(*rope.apply_rotary_emb(q, k, table, q.dtype, position_ids=pos), v, bias, None, **KW)
    e[1].record()
    out.backward(do)
    e[2].record()
    torch.cuda.synchronize()
    t = (e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2]))
    peak = torch.cuda.max_memory_allocated() - base
    return t, peak, (out.detach(), q.grad, k.grad, v.grad)


def run_case(S, dtype, rounds):
    g = torch.Generator(device="cuda").manual_seed(S)
    q, k, v, do = [torch.randn(1, S, H, D, device="cuda", generator=g).to(dtype) for _ in range(4)]
    bias = ra.attention_bias_from_mask(torch.ones(1, S, device="cuda"), dtype)
    pos = torch.arange(S, device="cuda")[None]
    table = rope.precompute_freqs_cis(D, max(S, 4096), 1e4)
    times = {False: [], True: []}
    peaks = {}
    first = {}
    for r in range(rounds + 1):                    # round 0 warms up (and compares the results)
        for fused in (False, True):
            t, peak, res = step(q, k, v, do, bias, pos, table, fused)
            if r == 0:
                first[fused] = res
            else:
                times[fused].append(t)
                peaks[fused] = peak
        if r == 0:    # out, dK, dV (dQ differs by the order of its fp32 reductions)
            same = all(torch.equal(first[False][i], first[True][i]) for i in (0, 2, 3))
            first.clear()
    row = dict(S=S, dtype=str(dtype).split(".")[-1], same_out_dk_dv=bool(same))
    for fused, name in ((False, "composition"), (True, "fused")):
        f = statistics.median(t[0] for t in times[fused])
        b = statistics.median(t[1] for t in times[fused])
        fb = statistics.median(t[0] + t[1] for t in times[fused])
        row[name] = dict(fwd_ms=round(f, 3), bwd_ms=round(b, 3), fwd_bwd_ms=round(fb, 3),
                         peak_mib=round(peaks[fused] / 2 ** 20, 1))
    rf, rb = removed_bytes(S, dtype)
    row["removed_MB"] = dict(fwd=round(rf / 1e6, 1), bwd=round(rb / 1e6, 1))
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="8192,32768,131072")
    ap.add_argument("--dtypes", default="bf16,fp32")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_rope_attn: needs a GPU (nothing is timed on the CPU)")
    info = card()
    print("card:", info)
    rows = []
    for S in [int(s) for s in a.sizes.split(",")]:
        for d in a.dtypes.split(","):
            row = run_case(S, DT[d], a.rounds)
            rows.append(row)
            c, f = row["composition"], row["fused"]
            print("S=%6d %s  fwd %8.3f -> %8.3f ms  bwd %8.3f -> %8.3f ms  fwd+bwd %8.3f -> %8.3f ms (%+.2f%%)  "
                  "peak %8.1f -> %8.1f MiB  removed fwd %.0f MB bwd %.0f MB  same=%s" % (
                      S, row["dtype"], c["fwd_ms"], f["fwd_ms"], c["bwd_ms"], f["bwd_ms"], c["fwd_bwd_ms"],
                      f["fwd_bwd_ms"], 100.0 * (f["fwd_bwd_ms"] / c["fwd_bwd_ms"] - 1.0), c["peak_mib"],
                      f["peak_mib"], row["removed_MB"]["fwd"], row["removed_MB"]["bwd"], row["same_out_dk_dv"]),
                  flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
