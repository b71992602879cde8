"""The cached prefill on the 8-bit KV cache: `ringattention(q, ck, cv, bias, ...)` with ck / cv QuantizedKV (operand
copies staged straight from the codes) against the explicit composition `ringattention(q, ck.dequantize(q.dtype),
cv.dequantize(q.dtype), bias, ...)` that the op ran before.

One GPU, B = 1, H = 32, D = 128, causal (causal_block_size=1) with the call site's zero bias [B,1,1,Sk]. Cases: Sq =
32768 queries against Sk = 131072 cached keys, and Sq = Sk = 131072; q fp32 and bf16; the fp16 and fp8 modes. The one-GPU
op places both q and the cache at positions 0 .., so with Sq < Sk the causal mask leaves query row i keys 0 .. i. Per
configuration the two routes are first checked to give identical outputs, their peak allocated memory above the inputs
is read (torch.cuda.max_memory_allocated), and then they alternate in one process for --rounds rounds of --reps calls
each, timed with CUDA events; the medians are reported. The card, its power limit and SM clock are read in the same
run. One JSON line per configuration.

usage: python tools/perf_kv_q8_prefill.py [--cases all|prefill,full] [--rounds 5] [--reps 2] [--json OUT]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from lwm_b200 import ringattention as ra  # noqa: E402
from lwm_b200.kv_cache import QuantizedKV, kv_cache_write_q8  # noqa: E402

B, H, D = 1, 32, 128
CASES = {"prefill": (32768, 131072), "full": (131072, 131072)}     # name: (Sq, Sk)
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}


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


def peak_above(fn):
    """-> (fn's result, peak allocated bytes during fn above what was allocated before it)"""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def cache(Sk, dtype, seed):
    """QuantizedKV k / v [B,Sk,H,128] quantized from N(0,1) rows of dtype"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ck, cv = QuantizedKV.zeros(B, Sk, H), QuantizedKV.zeros(B, Sk, H)
    k, v = [torch.randn(B, Sk, H, D, generator=g, device="cuda").to(dtype) for _ in range(2)]
    kv_cache_write_q8(k, v, 0, Sk, ck, cv, 0)
    return ck, cv


def run(case, dname, precision, rounds, reps):
    Sq, Sk = CASES[case]
    dtype = DTYPES[dname]
    g = torch.Generator(device="cuda").manual_seed(Sq)
    q = torch.randn(B, Sq, H, D, generator=g, device="cuda").to(dtype)
    ck, cv = cache(Sk, dtype, Sk + Sq)
    bias = torch.zeros(B, 1, 1, Sk, device="cuda", dtype=dtype)
    kw = dict(blockwise_kwargs=dict(causal_block_size=1), precision=precision)
    routes = {
        "dequantize_first": lambda: ra.ringattention(q, ck.dequantize(dtype), cv.dequantize(dtype), bias, **kw),
        "from_codes": lambda: ra.ringattention(q, ck, cv, bias, **kw),
    }
    with torch.no_grad():
        outs, peaks = {}, {}
        for n, fn in routes.items():            # also the warm-up of every launch either route makes
            outs[n], peaks[n] = peak_above(fn)
        identical = bool(torch.equal(outs["dequantize_first"], outs["from_codes"]))
        if not identical:
            sys.exit("perf_kv_q8_prefill: the two routes differ (%s %s %s)" % (case, dname, precision))
        del outs
        t = {n: [] for n in routes}
        for _ in range(rounds):
            for n, fn in routes.items():
                t[n].append(timed(fn, reps))
    med = {n: float(np.median(v)) for n, v in t.items()}
    return dict(case=case, B=B, H=H, Sq=Sq, Sk=Sk, causal=True, bias=True, q_dtype=dname, precision=precision,
                identical=identical, rounds=rounds, reps=reps, card=card(),
                ms={n: med[n] for n in routes}, ms_all={n: t[n] for n in routes},
                peak_mib={n: peaks[n] / 2 ** 20 for n in routes},
                dequantized_kv_mib=2 * B * Sk * H * D * torch.empty((), dtype=dtype).element_size() / 2 ** 20,
                peak_saved_mib=(peaks["dequantize_first"] - peaks["from_codes"]) / 2 ** 20,
                time_saved_ms=med["dequantize_first"] - med["from_codes"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="all")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("perf_kv_q8_prefill: needs an H100")
    names = list(CASES) if a.cases == "all" else a.cases.split(",")
    out = []
    for case in names:
        for dname in DTYPES:
            for precision in ("fp16", "fp8"):
                r = run(case, dname, precision, max(3, a.rounds), a.reps)
                print(json.dumps(r), flush=True)
                out.append(r)
                torch.cuda.empty_cache()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
