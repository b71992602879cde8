"""Decode step and cached prefill with the 8-bit KV cache against fp32 and bf16 caches, on one GPU.

Decode step = the cache write of one row (ShardedKVCache.concatenate) + ringattention_inference with Q = 1, B = 1,
H = 32, at K = 16384, 131072 and 1048576 keys per rank. q in fp32 (fp32 vs int8 cache) and in bf16 (bf16 vs int8). The
caches of one K live side by side and their steps alternate; each number is the median of --steps steps. Reported:
step time, attention time (CUDA events around ringattention_inference alone), the GB/s that time implies for the
bytes one step has to read (K and V rows + exponents, computed from the shapes), and the cache bytes per rank, taken
from the allocations. Cached prefill: ringattention(q, cache_k, cache_v, rotate_k=False) at S = 32768, causal, bf16 q,
bf16 vs int8 cache (the int8 call dequantizes the shard first).

    python tools/perf_kv_q8.py [--steps 20] [--ks 16384,131072,1048576] [--out results.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

H, D = 32, 128


def _card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:       # noqa: BLE001 - reported, not fatal
        return "unknown (%s)" % e


def _fill(cache, K, dtype, seed):
    """random rows in every slot of the cache (bf16 / fp32 rows, or quantized from bf16 rows)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    chunk = 1 << 15
    for j in range(0, K, chunk):
        n = min(chunk, K - j)
        k = torch.randn((1, n, H, D), generator=g, device="cuda").to(dtype)
        v = torch.randn((1, n, H, D), generator=g, device="cuda").to(dtype)
        if cache.quantized:
            cache.write_q8(k, v, 0, n, cache.cached_key, cache.cached_value, j)
        else:
            cache.cached_key[:, j:j + n].copy_(k)
            cache.cached_value[:, j:j + n].copy_(v)


def _cache_bytes(cache):
    if cache.quantized:
        return cache.cached_key.nbytes + cache.cached_value.nbytes
    return sum(t.numel() * t.element_size() for t in (cache.cached_key, cache.cached_value))


def decode(K, q_dtype, steps, warmup=3):
    from lwm_b200.kv_cache import ShardedKVCache
    from lwm_b200.ringattention import ringattention_inference
    caches = {}
    for dt in (q_dtype, torch.int8):
        c = ShardedKVCache(1, K, H, D, dtype=dt)
        _fill(c, K, q_dtype, seed=K)
        caches[dt] = c
    g = torch.Generator(device="cuda").manual_seed(1)
    q, k1, v1 = (torch.randn((1, 1, H, D), generator=g, device="cuda").to(q_dtype) for _ in range(3))
    times = {dt: ([], []) for dt in caches}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    with torch.no_grad():
        for i in range(warmup + steps):
            for dt, c in caches.items():          # alternate the caches step by step
                c.cache_index = K - 1
                ev[0].record()
                ck, cv = c.concatenate(k1, v1)
                ev[1].record()
                ringattention_inference(q, ck, cv, None)
                ev[2].record()
                torch.cuda.synchronize()
                if i >= warmup:
                    times[dt][0].append(ev[0].elapsed_time(ev[2]))
                    times[dt][1].append(ev[1].elapsed_time(ev[2]))
    rows = []
    for dt, c in caches.items():
        step, attn = statistics.median(times[dt][0]), statistics.median(times[dt][1])
        row_bytes = {torch.float32: 2 * D * 4, torch.bfloat16: 2 * D * 2, torch.int8: 2 * (D + 4)}[dt]
        read = K * H * row_bytes
        rows.append(dict(K=K, q=str(q_dtype)[6:], cache=str(dt)[6:], step_ms=round(step, 4), attn_ms=round(attn, 4),
                         read_GB=round(read / 1e9, 4), GBps=round(read / 1e9 / (attn / 1e3), 1),
                         cache_bytes_per_rank=_cache_bytes(c)))
    del caches
    torch.cuda.empty_cache()
    return rows


def prefill(S, reps=10, warmup=2):
    from lwm_b200.kv_cache import ShardedKVCache
    from lwm_b200.ringattention import ringattention
    g = torch.Generator(device="cuda").manual_seed(2)
    q = torch.randn((1, S, H, D), generator=g, device="cuda").to(torch.bfloat16)
    caches = {}
    for dt in (torch.bfloat16, torch.int8):
        c = ShardedKVCache(1, S, H, D, dtype=dt)
        _fill(c, S, torch.bfloat16, seed=S)
        caches[dt] = c
    times = {dt: [] for dt in caches}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    kw = dict(blockwise_kwargs=dict(causal_block_size=1))
    with torch.no_grad():
        for i in range(warmup + reps):
            for dt, c in caches.items():
                ev[0].record()
                ringattention(q, c.cached_key, c.cached_value, None, None, **kw)
                ev[1].record()
                torch.cuda.synchronize()
                if i >= warmup:
                    times[dt].append(ev[0].elapsed_time(ev[1]))
    return [dict(S=S, q="bfloat16", cache=str(dt)[6:], prefill_ms=round(statistics.median(t), 3),
                 cache_bytes_per_rank=_cache_bytes(caches[dt])) for dt, t in times.items()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--ks", default="16384,131072,1048576")
    ap.add_argument("--prefill", type=int, default=32768)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_kv_q8 needs a GPU")
    card = _card()
    print("card:", card)
    res = dict(card=card, decode=[], prefill=[])
    for K in (int(x) for x in a.ks.split(",")):
        for q_dtype in (torch.float32, torch.bfloat16):
            for r in decode(K, q_dtype, max(20, a.steps)):
                print(json.dumps(r))
                res["decode"].append(r)
    if a.prefill:
        for r in prefill(a.prefill):
            print(json.dumps(r))
            res["prefill"].append(r)
    res["card_after"] = _card()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
