"""Cost of the ordered dQ reduction (torch.use_deterministic_algorithms(True), DESIGN §3.3) on one GPU.

1. The backward tile step, unordered against ordered, alternating in one process: B = 1, H = 32, causal, S = 32768 and
   131072, both precision modes, without a mask and with the call-site bias (zero bias and segment ids: the block-map
   path). Each timed call is the step as the op makes it (ringattention's one-GPU backward: block map, then
   lwm_attn_bwd_step without or with an order_ws, the latter with its workspace zeroing and turns pass), timed with
   CUDA events;
   median over the rounds. The two dQ are compared within 1e-5 of max|dQ| and dK / dV bit for bit.
2. One full forward + backward of ringattention at S = 32768 (fp16 mode, no mask) with the flag off and on, and with
   torch.utils.deterministic.fill_uninitialized_memory at its default (True) and False.
The card, its power limit and SM clock are read in the same run.

usage: python tools/perf_attn_ordered.py [--sizes 32768,131072] [--rounds 3] [--json OUT]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from lwm_b200 import ringattention as ra  # noqa: E402

H, D = 32, 128


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def step_inputs(S, precision, mask, seed=0):
    """the one-GPU backward step's operands, as ring_backward (world = 1) stages them"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    q, k, v, do = (torch.randn(1, S, H, D, device="cuda", generator=g).to(torch.bfloat16) for _ in range(4))
    bias = seg = None
    if mask == "callsite":
        bias = torch.zeros(1, S, device="cuda")
        seg = torch.zeros(1, S, dtype=torch.int32, device="cuda")
    _, res = ra.ring_forward(q, k, v, bias, seg, True, None, 0, 1, "auto", precision)
    ops = ra._peer_ops(precision)
    sq, sk, sv = res["scales"]
    sdo = ra._local_scales(ops, (do,))[0]
    k16, v16, d16 = ra._stage_local(ops, k, sk), ra._stage_local(ops, v, sv), ra._stage_local(ops, do, sdo)
    delta = torch.empty(1, H, S, device="cuda")
    ops.bwd_prep(res["out_chunks"][0], d16, sdo, delta)
    nlse = ops.lse_for_bwd(res["lse_chunks"][0])
    acc = [torch.zeros(1, S, H, D, device="cuda") for _ in range(3)]
    return ops, (res["q_chunks"][0], k16, v16, d16, nlse, delta, *acc, 0, 0, True, bias, seg, (sq, sk, sv, sdo), True)


def run_step(ops, args, ordered):
    torch.use_deterministic_algorithms(ordered)
    args[6].zero_()
    torch.cuda.synchronize()
    ms, _ = timed(lambda: ops.bwd_step(*args))
    return ms, [t.clone() for t in args[6:9]]


def kernel_rows(sizes, rounds):
    rows = []
    for S in sizes:
        for precision in ("fp16", "bf16"):
            for mask in ("none", "callsite"):
                ops, args = step_inputs(S, precision, mask)
                run_step(ops, args, False)
                run_step(ops, args, True)                      # warm-up of both
                t = {False: [], True: []}
                res = {}
                for _ in range(rounds):
                    for ordered in (False, True):
                        ms, res[ordered] = run_step(ops, args, ordered)
                        t[ordered].append(ms)
                torch.use_deterministic_algorithms(False)
                (dq0, dk0, dv0), (dq1, dk1, dv1) = res[False], res[True]
                dq_ok = bool(((dq0 - dq1).abs() <= 1e-5 * dq0.abs().max()).all())
                same = bool(torch.equal(dk0, dk1) and torch.equal(dv0, dv1))
                u, o = statistics.median(t[False]), statistics.median(t[True])
                row = dict(S=S, precision=precision, mask=mask, unordered_ms=u, ordered_ms=o, overhead=o / u - 1,
                           dq_close=dq_ok, dkdv_identical=same, rounds=rounds)
                print("bwd step S=%6d %s %-8s unordered %8.2f ms  ordered %8.2f ms  (%+.1f%%)  dq_close=%s dk/dv same=%s"
                      % (S, precision, mask, u, o, 100 * (o / u - 1), dq_ok, same), flush=True)
                rows.append(row)
                del args
                torch.cuda.empty_cache()
    return rows


def step_rows(S, rounds):
    from torch.utils import deterministic as tud
    g = torch.Generator(device="cuda").manual_seed(1)
    q, k, v, do = (torch.randn(1, S, H, D, device="cuda", generator=g).to(torch.bfloat16) for _ in range(4))
    leaves = [x.requires_grad_() for x in (q, k, v)]
    kw = dict(blockwise_kwargs=dict(causal_block_size=1), precision="fp16")

    def step():
        out = ra.ringattention(*leaves, None, None, **kw)
        return torch.autograd.grad(out, leaves, do)

    configs = [("flag off", False, True), ("flag on", True, True), ("flag on, fill_uninitialized_memory=False", True,
                                                                    False), ("flag off (again)", False, True)]
    prev_fill = tud.fill_uninitialized_memory
    t = {c[0]: [] for c in configs}
    try:
        for name, flag, fill in configs:            # warm-up
            torch.use_deterministic_algorithms(flag)
            tud.fill_uninitialized_memory = fill
            timed(step)
        for _ in range(rounds):
            for name, flag, fill in configs:
                torch.use_deterministic_algorithms(flag)
                tud.fill_uninitialized_memory = fill
                t[name].append(timed(step)[0])
    finally:
        torch.use_deterministic_algorithms(False)
        tud.fill_uninitialized_memory = prev_fill
    rows = []
    for name, _, _ in configs:
        ms = statistics.median(t[name])
        print("fwd+bwd S=%d fp16 causal, %-42s %8.2f ms" % (S, name, ms), flush=True)
        rows.append(dict(S=S, config=name, ms=ms, rounds=rounds))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="32768,131072")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_attn_ordered: needs a GPU")
    c = card()
    print("card: %s (name, power limit, SM clock, max SM clock)" % c, flush=True)
    rows = kernel_rows([int(s) for s in a.sizes.split(",")], max(3, a.rounds))
    steps = step_rows(32768, max(3, a.rounds))
    print("card after: %s" % card())
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=c, kernel=rows, step=steps), f, indent=1)


if __name__ == "__main__":
    main()
