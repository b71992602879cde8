"""ringattention_inference timing on one GPU: the GEMV kernel against the tensor-core kernel.

Sweeps Q in {1, 2, 4, ..., 256, 2048, 32768} with K in {Q + 512, 131072}, H = 32, fp32 and bf16, with the mask of
a generation step (row i sees keys <= K - Q + i). For Q <= 256 both paths are timed, alternating, one call each per
round; above, only the tensor-core path. Prints ms per call (staging and mask packing included) and algorithmic
TFLOP/s = 4 * D * H * (true mask entries) / time, then the training forward at S = 32768 for comparison.
Usage: python tools/perf_infer.py [--quick]"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from lwm_b200 import ringattention as ra


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def run(Q, K, dtype, min_q, reps, H=32):
    g = torch.Generator(device="cuda").manual_seed(0)
    q = torch.randn(1, Q, H, 128, device="cuda", generator=g).to(dtype)
    k = torch.randn(1, K, H, 128, device="cuda", generator=g).to(dtype)
    v = torch.randn(1, K, H, 128, device="cuda", generator=g).to(dtype)
    mask = (torch.arange(K, device="cuda")[None, :] <= (torch.arange(Q, device="cuda") + K - Q)[:, None])[None, None]
    true = Q * (K - Q) + Q * (Q + 1) // 2
    paths = {"gemv": 1 << 30, "tc": 1} if Q < min_q else {"tc": 1}
    res = {}
    for name, m in paths.items():            # warm-up
        ra.INFER_MIN_Q = m
        ra.ringattention_inference(q, k, v, mask)
    torch.cuda.synchronize()
    times = {n: [] for n in paths}
    for _ in range(reps):                    # alternate the paths
        for name, m in paths.items():
            ra.INFER_MIN_Q = m
            times[name].append(timed(lambda: ra.ringattention_inference(q, k, v, mask), 1))
    for name, ts in times.items():
        ms = sorted(ts)[len(ts) // 2]
        res[name] = (ms, 4 * 128 * H * true / ms / 1e9)
    del q, k, v, mask
    torch.cuda.empty_cache()
    return res


def main():
    quick = "--quick" in sys.argv
    print("card: %s" % card())
    default_min = ra.INFER_MIN_Q
    qs = [1 << i for i in range(9)] + [2048, 32768]
    for dtype in (torch.float32, torch.bfloat16):
        for Q in qs:
            for K in (Q + 512, 131072):
                if quick and (K > 8192 or Q > 2048):
                    continue
                reps = 3 if Q * K > 1 << 26 else 5
                r = run(Q, K, dtype, 512, reps)
                print("%s Q=%6d K=%6d  " % (str(dtype)[6:], Q, K) + "  ".join(
                    "%s %9.3f ms %7.2f TFLOP/s" % (n, ms, tf) for n, (ms, tf) in r.items()), flush=True)
    ra.INFER_MIN_Q = default_min
    # the causal training forward at S = 32768, H = 32 (bf16 inputs, default precision), forward only
    S, H = 32768, 32
    q, k, v = (torch.randn(1, S, H, 128, device="cuda").to(torch.bfloat16) for _ in range(3))
    f = lambda: ra.ringattention(q, k, v, blockwise_kwargs={"causal_block_size": 1})   # noqa: E731
    with torch.no_grad():
        f()
        torch.cuda.synchronize()
        print("training forward (ringattention, causal) S=%d H=%d: %.3f ms" % (S, H, timed(f, 5)))
    mask = torch.ones(S, S, dtype=torch.bool, device="cuda").tril_()[None, None]
    g = lambda: ra.ringattention_inference(q, k, v, mask)    # noqa: E731
    g()
    torch.cuda.synchronize()
    print("ringattention_inference causal Q=K=%d H=%d bf16: %.3f ms" % (S, H, timed(g, 5)))


if __name__ == "__main__":
    main()
