"""Cost of the reproducible VQGAN tokenizer (torch.use_deterministic_algorithms(True): ordered GroupNorm statistics and
per-image fp16 plane scales, DESIGN.md §4) on one GPU, default VQGANConfig, synthetic weights, 256x256 frames.

Three workloads, each timed with the flag off and on, alternating in one process, CUDA events, median over the rounds:
  encode16   VQGAN.encode of a 16-frame clip (dataset preparation, bench.py's workload)
  decode16   VQGAN.decode of 16 frames of codes
  encode1x16 the B = 1 per-frame loop of vision_chat.py: 16 encodes of one frame each
The number of codes that differ between two flag-off encodes of the same clip is reported as well (with the flag on it
is 0 by construction). The card, its power limit and SM clock are read in the same run.

usage: python tools/perf_vqgan_ordered.py [--precision fp16x2] [--rounds 7] [--json OUT]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from lwm_b200.vqgan import VQGAN, init_params  # noqa: E402

T = 16


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="fp16x2", choices=["fp16x2", "bf16x3", "bf16"])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_vqgan_ordered needs a GPU")
    dev_card = card()
    print("card:", dev_card)
    tok = VQGAN(init_params(seed=0), precision=a.precision)
    g = torch.Generator(device="cuda").manual_seed(0)
    clip = torch.rand(T, 256, 256, 3, device="cuda", generator=g) * 2 - 1
    codes = torch.randint(0, 8192, (T, 16, 16), device="cuda", generator=g)
    work = {
        "encode16": lambda: tok.encode(clip),
        "decode16": lambda: tok.decode(codes),
        "encode1x16": lambda: [tok.encode(clip[t:t + 1]) for t in range(T)],
    }
    prev = torch.are_deterministic_algorithms_enabled()
    times = {(w, o): [] for w in work for o in (False, True)}
    try:
        for o in (False, True):               # warm-up: every shape and both paths
            torch.use_deterministic_algorithms(o)
            for fn in work.values():
                fn()
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for w, fn in work.items():
                for o in (False, True):
                    torch.use_deterministic_algorithms(o)
                    times[(w, o)].append(timed(fn)[0])
        torch.use_deterministic_algorithms(False)
        flips = int((timed(work["encode16"])[1][1] != timed(work["encode16"])[1][1]).sum())
    finally:
        torch.use_deterministic_algorithms(prev)
    res = {"card": dev_card, "precision": a.precision, "rounds": a.rounds, "flag_off_code_changes_of_4096": flips,
           "ms": {}}
    print("%-11s %12s %12s %8s" % ("workload", "flag off ms", "flag on ms", "on/off"))
    for w in work:
        off, on = statistics.median(times[(w, False)]), statistics.median(times[(w, True)])
        res["ms"][w] = {"off": off, "on": on, "off_all": times[(w, False)], "on_all": times[(w, True)]}
        print("%-11s %12.2f %12.2f %8.3f   (off %.2f-%.2f, on %.2f-%.2f)" % (
            w, off, on, on / off, min(times[(w, False)]), max(times[(w, False)]), min(times[(w, True)]),
            max(times[(w, True)])))
    print("flag off: %d of %d codes differ between two encodes of the same clip" % (flips, T * 256))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
