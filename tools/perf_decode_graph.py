"""Time the generation decode step eagerly against the same step captured once in a CUDA graph and replayed, on one GPU.

Decode step of one layer = the cache write of one new row (ShardedKVCache.concatenate with the rotary keywords) +
ringattention_inference with Q = 1 over the K-row cache (rotate_k=False), B = 1, H = 32, D = 128; a token runs it once
per layer, so the graph holds 1 or 32 layers. Caches: bf16, fp32 and int8 (bf16 rows and q).
  eager   the calls as a generation loop makes them: cache_index, positions and mask from host ints, no synchronisation;
  graph   the positions and mask derived from ShardedKVCache.cursor on the device, the step recorded once with
          torch.cuda.graph (after a warm-up on a side stream) and replayed, new rows copied into static buffers first.
Every timed step writes slot K - 1 (the cursors are rewound outside the timed window) and attends to all K keys. The two
modes alternate step by step; medians over the rounds of the CUDA-event time and of the host clock up to a synchronise.
Before timing, one step of each mode from the same cache state must give the same outputs, bit for bit. The 32 layers
have caches of their own where all of them fit in 40 GB, else they share one K/V storage (each keeps its own cursor,
write and read), as "kv_storage" records. The card and its power limit are read in the same run.

usage: python tools/perf_decode_graph.py [--K 4096,16384,131072] [--kinds bf16,fp32,int8] [--layers 1,32]
                                         [--rounds 30] [--json OUT]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lwm_b200 import ringattention as ra  # noqa: E402
from lwm_b200 import rope  # noqa: E402
from lwm_b200.kv_cache import ShardedKVCache  # noqa: E402

B, H, D = 1, 32, 128
KINDS = {"bf16": (torch.bfloat16, torch.bfloat16), "fp32": (torch.float32, torch.float32),
         "int8": (torch.int8, torch.bfloat16)}         # cache dtype, row dtype
SHARED_ABOVE = 40 << 30


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)


def kv_bytes(cdt, K):
    return K * H * (D + 4) * 2 if cdt == torch.int8 else K * H * D * 2 * torch.tensor([], dtype=cdt).element_size()


class Layer:
    def __init__(self, kind, K, seed, table, share=None):
        cdt, dt = KINDS[kind]
        g = torch.Generator().manual_seed(seed)
        self.q, self.k, self.v = [torch.randn(B, 1, H, D, generator=g).to(dt).cuda() for _ in range(3)]
        self.q_in, self.k_in, self.v_in = (torch.empty_like(t) for t in (self.q, self.k, self.v))
        self.cache = ShardedKVCache(B, K, H, D, dtype=cdt)
        if share is not None:
            self.cache.cached_key, self.cache.cached_value = share.cache.cached_key, share.cache.cached_value
        elif cdt == torch.int8:
            for c in (self.cache.cached_key, self.cache.cached_value):
                c.data.random_(-127, 128)
                c.exp.random_(-12, 0)
        else:
            self.cache.cached_key.normal_()
            self.cache.cached_value.normal_()
        self.K, self.table = K, table
        self.am = torch.ones(B, K, dtype=torch.int64, device="cuda")

    def step(self, q, k, v, index, pos):
        mask = ra.decode_attention_mask(self.am, 1, index, self.K)
        ck, cv = self.cache.concatenate(k, v, freqs_cis=self.table, position_ids=pos)
        return ra.ringattention_inference(q, ck, cv, mask, freqs_cis=self.table, position_ids=pos, rotate_k=False)

    def eager(self):
        idx = self.K - 1                             # the host's own count (what a generation loop keeps)
        return self.step(self.q, self.k, self.v, idx, torch.full((B, 1), idx, dtype=torch.int64))

    def graph_step(self):
        cur = self.cache.cursor
        pos = cur.expand(B).view(B, 1) + 0           # a tensor of its own, made before the write advances the cursor
        return self.step(self.q_in, self.k_in, self.v_in, cur, pos)

    def load(self):
        self.q_in.copy_(self.q)
        self.k_in.copy_(self.k)
        self.v_in.copy_(self.v)


def rewind(layers):
    for ly in layers:
        ly.cache.cache_index = ly.K - 1


def capture(layers):
    rewind(layers)
    for ly in layers:
        ly.load()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for ly in layers:
            ly.graph_step()
    torch.cuda.current_stream().wait_stream(s)
    rewind(layers)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = [ly.graph_step() for ly in layers]
    return g, outs


def bench(kind, K, n_layers, rounds):
    table = rope.precompute_freqs_cis(D, K + 16, 1e4)
    cdt = KINDS[kind][0]
    shared = n_layers * kv_bytes(cdt, K) > SHARED_ABOVE
    first = Layer(kind, K, 0, table)
    layers = [first] + [Layer(kind, K, i, table, first if shared else None) for i in range(1, n_layers)]
    g, outs = capture(layers)

    def run_eager():
        return [ly.eager() for ly in layers]

    def run_graph():
        for ly in layers:
            ly.load()
        g.replay()
        return outs

    # bits first: one step of each mode from the same state
    rewind(layers)
    want = [o.clone() for o in run_eager()]
    rewind(layers)
    got = [o.clone() for o in run_graph()]
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), "%s K=%d layer %d: graph and eager differ" % (kind, K, i)
    assert first.cache.take_errors() == 0
    res = {m: dict(dev=[], host=[]) for m in ("eager", "graph")}
    fns = {"eager": run_eager, "graph": run_graph}
    for r in range(rounds + 3):
        for m in ("eager", "graph"):
            rewind(layers)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record()
            fns[m]()
            e1.record()
            torch.cuda.synchronize()
            if r >= 3:                               # the first rounds warm up
                res[m]["host"].append((time.perf_counter() - t0) * 1e3)
                res[m]["dev"].append(e0.elapsed_time(e1))
    out = {m: dict(step_ms_events=statistics.median(v["dev"]), step_ms_host=statistics.median(v["host"]),
                   per_layer_ms_events=statistics.median(v["dev"]) / n_layers) for m, v in res.items()}
    out["kv_storage"] = "shared" if shared else "per layer"
    del g, outs, layers, first
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--K", default="4096,16384,131072")
    ap.add_argument("--kinds", default="bf16,fp32,int8")
    ap.add_argument("--layers", default="1,32")
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_decode_graph.py needs a GPU")
    out = dict(card=card(), B=B, H=H, results={})
    print("card:", out["card"])
    for kind in a.kinds.split(","):
        for K in [int(x) for x in a.K.split(",") if x]:
            for n in [int(x) for x in a.layers.split(",") if x]:
                r = bench(kind, K, n, a.rounds)
                out["results"]["%s K=%d layers=%d" % (kind, K, n)] = r
                print("%s K=%d layers=%d %s" % (kind, K, n, json.dumps(r)), flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
