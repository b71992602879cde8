"""Speed and error of the fp8 mode's forward (precision='fp8': e4m3 Q K^T, fp16 P V) against the fp16 mode's.

One GPU, B = 1, H = 32, D = 128, one step (first = last). Cases: causal S = 32768 and 131072 without a mask (the plain
kernels) and with the call site's zero bias (the block-map kernels), and the cached prefill: the last Sq = 32768
positions against a 131072-key cache (q_pos0 = Sk - Sq, causal). Per case the two modes alternate in one process for
--rounds rounds; each round times --reps launches with CUDA events, and the median over rounds is reported for
  staging  the operand passes (per-tensor |max| -> power-of-two scale -> scaled copy of q, k and v),
  kernel   the tile kernel alone (lwm_attn_fwd_step with fp16 operands / lwm_attn_fwd_e4m3_step),
  total    both, back to back,
with algorithmic TFLOP/s (4 * D * visible (query, key) pairs * H) of kernel and total. The error of each mode's output
against the float64 row oracle (oracle/attn_rows.py) on sampled rows of head 0, relative to max |ref|, is measured on
the same inputs. The card, its power limit and SM clock are read in the same run. One JSON line per case.

usage: python tools/perf_attn_e4m3.py [--cases all|c32k,c32k_bias,c128k,c128k_bias,prefill] [--rounds 5] [--reps 3]
                                      [--json OUT]"""
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
CASES = {   # name: (Sq, Sk, block map from the call-site zero bias)
    "c32k": (32768, 32768, False), "c32k_bias": (32768, 32768, True),
    "c128k": (131072, 131072, False), "c128k_bias": (131072, 131072, True),
    "prefill": (32768, 131072, False),
}


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


def visible_pairs(Sq, Sk, q_pos0):
    """causal (query, key) pairs: row i (global q_pos0 + i) sees keys 0 .. q_pos0 + i"""
    return Sq * (q_pos0 + 1) + Sq * (Sq - 1) // 2


class Mode:
    """one precision mode's staging and kernel on fixed inputs"""

    def __init__(self, name, q, k, v, q_pos0, bias, tilemap):
        self.name, self.q, self.k, self.v, self.q_pos0, self.bias, self.tilemap = name, q, k, v, q_pos0, bias, tilemap
        qk_ops = ra.PeerOpsE4m3 if name == "fp8" else ra.PeerOpsF16
        self.ops = (qk_ops, qk_ops, ra.PeerOpsF16)
        self.scales = [torch.empty(1, dtype=torch.float32, device="cuda") for _ in range(3)]
        self.staged = [torch.empty(t.shape, dtype=o.op_dtype, device="cuda") for t, o in zip((q, k, v), self.ops)]
        self.out = torch.empty(q.shape, dtype=torch.bfloat16, device="cuda")
        self.o32 = torch.empty(q.shape, dtype=torch.float32, device="cuda")
        self.lse = torch.empty((1, H, q.shape[1]), dtype=torch.float32, device="cuda")

    def stage(self):
        for o, t, s, y in zip(self.ops, (self.q, self.k, self.v), self.scales, self.staged):
            o.scale_of(t, s)
            o.stage(t, y, s)

    def kernel(self):
        q, k, v = self.staged
        args = (q, k, v, self.out, self.lse, None, None, None, self.q_pos0, 0, True, self.bias, None, True, True)
        if self.name == "fp8":
            ra.fwd_e4m3_step(*args, tuple(self.scales), out_f32=self.o32, tilemap=self.tilemap)
        else:
            ra.fwd_step(*args, scales=tuple(self.scales), out_f32=self.o32, tilemap=self.tilemap)

    def total(self):
        self.stage()
        self.kernel()


def error(mode, q, k, v, q_pos0, rows):
    from oracle.attn_rows import attention_rows
    ref = attention_rows(q[0, rows, 0].cpu(), q_pos0 + rows, k[0, :, 0].cpu(), v[0, :, 0].cpu())["out"]
    got = mode.o32[0, rows, 0].double().cpu()
    return float((got - ref).abs().max() / ref.abs().max())


def run(name, rounds, reps):
    Sq, Sk, with_map = CASES[name]
    q_pos0 = Sk - Sq
    g = torch.Generator(device="cuda").manual_seed(Sk)
    q = torch.randn(1, Sq, H, D, generator=g, device="cuda").to(torch.bfloat16)
    k, v = [torch.randn(1, Sk, H, D, generator=g, device="cuda").to(torch.bfloat16) for _ in range(2)]
    bias = torch.zeros(1, Sk, device="cuda") if with_map else None
    tilemap = ra.step_tilemap(1, Sq, Sk, q_pos0, 0, True, bias, None, bwd=False)[:2] if with_map else None
    modes = [Mode(n, q, k, v, q_pos0, bias, tilemap) for n in ("fp16", "fp8")]
    for m in modes:          # warm-up: module load, shared-memory attribute, tensor maps
        m.total()
    torch.cuda.synchronize()
    t = {m.name: {"staging": [], "kernel": [], "total": []} for m in modes}
    for _ in range(rounds):
        for m in modes:
            t[m.name]["staging"].append(timed(m.stage, reps))
            t[m.name]["kernel"].append(timed(m.kernel, reps))
            t[m.name]["total"].append(timed(m.total, reps))
    flops = 4.0 * D * H * visible_pairs(Sq, Sk, q_pos0)
    from oracle.attn_rows import sample_rows
    rows = sample_rows(Sq)[::16]
    res = dict(case=name, B=1, H=H, Sq=Sq, Sk=Sk, q_pos0=q_pos0, causal=True, block_map=with_map, rounds=rounds,
               reps=reps, card=card())
    for m in modes:
        med = {n: float(np.median(v_)) for n, v_ in t[m.name].items()}
        res[m.name] = dict(staging_ms=med["staging"], kernel_ms=med["kernel"], total_ms=med["total"],
                           kernel_tflops=flops / med["kernel"] / 1e9, total_tflops=flops / med["total"] / 1e9,
                           err_vs_max=error(m, q, k, v, q_pos0, rows))
    res["kernel_speedup"] = res["fp16"]["kernel_ms"] / res["fp8"]["kernel_ms"]
    res["total_speedup"] = res["fp16"]["total_ms"] / res["fp8"]["total_ms"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="all")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("perf_attn_e4m3: needs an H100")
    names = list(CASES) if a.cases == "all" else a.cases.split(",")
    out = []
    for n in names:
        r = run(n, max(5, a.rounds), a.reps)
        print(json.dumps(r), flush=True)
        out.append(r)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
