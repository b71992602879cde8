"""Time the generation path with the rotary embedding inside the KV-cache write and inside the attention ops
(`ShardedKVCache.concatenate(freqs_cis=, position_ids=)`, `ringattention_inference(..., rotate_k=False)`,
`ringattention(..., rotate_k=False)`) against the composition (apply_rotary_emb, the plain cache update, the plain op),
on one GPU.

B = 1, H = 32, D = 128, bf16 and fp32, the two variants alternating step by step in one run; medians over the rounds.
  decode step  cache write of one new row + ringattention_inference with Q = 1 against K cache rows: per-step time from
               CUDA events and from the host clock up to a synchronise, kernel launches per step (torch.profiler, one
               untimed step), and device->host synchronisations per step (torch.cuda.set_sync_debug_mode) with the
               positions on the device and on the host.
  prefill      ringattention over S new rows against the S-row cache (causal, the LWM bias of an all-ones mask, fp16
               precision mode): forward time from CUDA events and torch.cuda.max_memory_allocated above the inputs.
The first step of each case checks that both variants give the same output, bit for bit. The card and its power limit
are read in the same run.

usage: python tools/perf_rope_decode.py [--decode 16384,131072] [--prefill 32768,131072] [--dtypes bf16,fp32]
                                        [--rounds 20] [--json OUT]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lwm_b200 import ringattention as ra  # noqa: E402
from lwm_b200 import rope  # noqa: E402
from lwm_b200.kv_cache import ShardedKVCache  # noqa: E402

B, H, D = 1, 32, 128
DT = {"bf16": torch.bfloat16, "fp32": torch.float32}


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)


def decode_step(cache, K, q, k, v, mask, pos, table, fused):
    cache.cache_index = K - 1                       # the step writes the cache's last row and attends to all K
    if fused:
        ck, cv = cache.concatenate(k, v, freqs_cis=table, position_ids=pos)
        return ra.ringattention_inference(q, ck, cv, mask, freqs_cis=table, position_ids=pos, rotate_k=False)
    qr, kr = rope.apply_rotary_emb(q, k, table, q.dtype, position_ids=pos)
    ck, cv = cache.concatenate(kr, v)
    return ra.ringattention_inference(qr, ck, cv, mask)


def count_launches(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def count_syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    return sum(1 for x in w if "synchroniz" in str(x.message))


def bench_decode(K, dtype, rounds):
    table = rope.precompute_freqs_cis(D, K + 16, 1e4)
    g = torch.Generator().manual_seed(K)
    q, k, v = [torch.randn(B, 1, H, D, generator=g).to(dtype).cuda() for _ in range(3)]
    cache = ShardedKVCache(B, K, H, D, dtype=dtype)
    cache.cached_key.normal_()
    cache.cached_value.normal_()
    mask = ra.decode_attention_mask(torch.ones(B, K, dtype=torch.int64, device="cuda"), 1, K - 1, K)
    pos = torch.full((B, 1), K - 1, dtype=torch.int64, device="cuda")
    pos_host = pos.cpu()
    res = {}
    outs = {f: decode_step(cache, K, q, k, v, mask, pos, table, f).clone() for f in (False, True)}
    assert torch.equal(outs[True], outs[False]), "decode step: fused and composition differ"
    for f in (False, True):
        res[f] = dict(dev=[], host=[],
                      launches=count_launches(lambda: decode_step(cache, K, q, k, v, mask, pos, table, f)),
                      syncs_dev_pos=count_syncs(lambda: decode_step(cache, K, q, k, v, mask, pos, table, f)),
                      syncs_host_pos=count_syncs(lambda: decode_step(cache, K, q, k, v, mask, pos_host, table, f)))
    for _ in range(3):
        for f in (False, True):
            decode_step(cache, K, q, k, v, mask, pos, table, f)
    for _ in range(rounds):
        for f in (False, True):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record()
            decode_step(cache, K, q, k, v, mask, pos, table, f)
            e1.record()
            torch.cuda.synchronize()
            res[f]["host"].append((time.perf_counter() - t0) * 1e3)
            res[f]["dev"].append(e0.elapsed_time(e1))
    return {("fused" if f else "composition"): dict(step_ms_events=statistics.median(r["dev"]),
                                                    step_ms_host=statistics.median(r["host"]),
                                                    launches=r["launches"], syncs_dev_pos=r["syncs_dev_pos"],
                                                    syncs_host_pos=r["syncs_host_pos"]) for f, r in res.items()}


def prefill_step(q, ck, cv, bias, pos, table, fused):
    kw = dict(axis_name="sp", blockwise_kwargs=dict(causal_block_size=1), precision="fp16")
    if fused:
        return ra.ringattention(q, ck, cv, bias, freqs_cis=table, position_ids=pos, rotate_k=False, **kw)
    return ra.ringattention(rope.rotate(q, table, q.dtype, position_ids=pos.to(torch.int32)), ck, cv, bias, **kw)


def bench_prefill(S, dtype, rounds):
    table = rope.precompute_freqs_cis(D, S + 16, 1e4)
    g = torch.Generator(device="cuda").manual_seed(S)
    q, ck, cv = [torch.randn(B, S, H, D, generator=g, device="cuda").to(dtype) for _ in range(3)]
    bias = ra.attention_bias_from_mask(torch.ones(B, S, device="cuda"), torch.float32 if dtype == torch.float32
                                       else torch.bfloat16)
    pos = torch.arange(S, device="cuda")[None]
    with torch.no_grad():
        a, b = (prefill_step(q, ck, cv, bias, pos, table, f) for f in (False, True))
        assert torch.equal(a, b), "prefill: fused and composition differ"
        del a, b
        res = {f: dict(ms=[], mem=[]) for f in (False, True)}
        for _ in range(rounds):
            for f in (False, True):
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = prefill_step(q, ck, cv, bias, pos, table, f)
                e1.record()
                torch.cuda.synchronize()
                res[f]["ms"].append(e0.elapsed_time(e1))
                res[f]["mem"].append((torch.cuda.max_memory_allocated() - base) / 2 ** 30)
                del out
    return {("fused" if f else "composition"): dict(fwd_ms=statistics.median(r["ms"]), peak_gib=max(r["mem"]))
            for f, r in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--decode", default="16384,131072")
    ap.add_argument("--prefill", default="32768,131072")
    ap.add_argument("--dtypes", default="bf16,fp32")
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_rope_decode.py needs a GPU")
    out = dict(card=card(), decode={}, prefill={})
    print("card:", out["card"])
    for name in a.dtypes.split(","):
        for K in [int(x) for x in a.decode.split(",") if x]:
            r = bench_decode(K, DT[name], a.rounds)
            out["decode"]["%s K=%d" % (name, K)] = r
            print("decode %s K=%d %s" % (name, K, json.dumps(r)))
        for S in [int(x) for x in a.prefill.split(",") if x]:
            r = bench_prefill(S, DT[name], max(3, a.rounds // 5))
            out["prefill"]["%s S=%d" % (name, S)] = r
            print("prefill %s S=%d %s" % (name, S, json.dumps(r)))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
