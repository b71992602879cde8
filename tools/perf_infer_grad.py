"""Forward + backward timing of `ringattention_inference` with the no-cache training mask of lwm/llama.py:580-592
(causal, no padding) against `ringattention` (causal, the call site's all-zero padding bias) on the same inputs.

S in {1024, 4096, 32768}, H = 32, B = 1, bf16 and fp32. The two ops alternate, one forward + backward each per
round; the median over rounds is printed (ms), with the mask packing and the two tile maps of the inference op
timed on their own (their time is included in its forward + backward). Prints the card and its power limit first.
Usage: python tools/perf_infer_grad.py [--quick]"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from lwm_b200 import _lib
from lwm_b200 import ringattention as ra


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def median(ts):
    return sorted(ts)[len(ts) // 2]


def run(S, dtype, rounds, H=32):
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v, do = (torch.randn(1, S, H, 128, device="cuda", generator=g).to(dtype) for _ in range(4))
    q, k, v = (x.requires_grad_() for x in (q, k, v))
    pad = torch.ones(1, S, dtype=torch.int32, device="cuda")
    mask = ra.causal_attention_mask(pad)
    bias = ra.attention_bias_from_mask(pad, torch.bfloat16)

    def infer():
        ra.ringattention_inference(q, k, v, mask).backward(do)

    def train():
        ra.ringattention(q, k, v, bias, None, blockwise_kwargs=dict(causal_block_size=1)).backward(do)

    def pack():
        return ra.mask_pack(mask, 1, 1, S)

    bits, row_any = pack()
    n_kt = (S + 127) // 128
    t_f = torch.empty(1, (S + 127) // 128, n_kt, dtype=torch.int32, device="cuda")
    c_f = torch.empty(1, (S + 127) // 128, dtype=torch.int32, device="cuda")
    t_b = torch.empty(1, n_kt, (S + 63) // 64, dtype=torch.int32, device="cuda")
    c_b = torch.empty(1, n_kt, dtype=torch.int32, device="cuda")

    def maps():
        _lib.call("lwm_attn_infer_tilemap", _lib.ptr(bits[0]), _lib.ptr(row_any), 1, S, S, _lib.ptr(t_f),
                  _lib.ptr(c_f), _lib.stream_ptr())
        _lib.call("lwm_attn_infer_bwd_tilemap", _lib.ptr(bits[0]), _lib.ptr(row_any), 1, S, S, _lib.ptr(t_b),
                  _lib.ptr(c_b), _lib.stream_ptr())

    for fn in (infer, train, pack, maps):     # warm-up
        fn()
    torch.cuda.synchronize()
    ts = {"infer": [], "train": [], "pack": [], "maps": []}
    for _ in range(rounds):
        for name, fn in (("infer", infer), ("train", train), ("pack", pack), ("maps", maps)):
            ts[name].append(timed(fn))
    return {n: median(t) for n, t in ts.items()}


def main():
    quick = "--quick" in sys.argv
    print("card:", card())
    print("%6s %5s | %22s | %22s | %9s | %9s" % ("S", "dtype", "inference fwd+bwd (ms)", "ringattention (ms)",
                                                 "pack (ms)", "maps (ms)"))
    for S in ((1024, 4096) if quick else (1024, 4096, 32768)):
        for dtype in (torch.bfloat16, torch.float32):
            r = run(S, dtype, rounds=3 if S > 8192 else 7)
            print("%6d %5s | %22.3f | %22.3f | %9.3f | %9.3f" % (S, str(dtype)[6:], r["infer"], r["train"], r["pack"],
                                                                  r["maps"]))
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
