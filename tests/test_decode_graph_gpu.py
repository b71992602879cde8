"""The generation decode step captured in a CUDA graph, on an H100: the cache write at the device cursor
(`ShardedKVCache.concatenate`, lwm_kv_cache_write_at), the mask from `decode_attention_mask(..., cache.cursor)` and
`ringattention_inference` with Q = 1, recorded once with torch.cuda.graph and replayed token after token.

Contract: every replayed step's output, the final cache (codes and exponents for the 8-bit cache) and cache_index are
bit-identical to the same steps run eagerly, for bf16, fp32 and int8 caches, with and without the rotary keywords, at
B = 1 and 2 and at cache lengths across the GEMV kernel's split edges; also with 32 caches (one per layer) in one graph.
The capture makes no host synchronisation. A replay past max_length or at a position outside the rotary table writes
nothing and sets the device error word. The cursor write on emulated ranks changes only the owner's shard, exactly as
the write at the host index does."""
import types

import pytest
import torch

pytestmark = pytest.mark.gpu
D = 128
KINDS = {"bf16": (torch.bfloat16, torch.bfloat16), "fp32": (torch.float32, torch.float32),
         "int8": (torch.int8, torch.bfloat16)}          # cache dtype, row (and q) dtype


def _randn(shape, seed, dtype, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


def _state(cache):
    """the cache's contents as a list of tensors (codes and exponents for the 8-bit cache)"""
    if cache.quantized:
        return [t.clone() for c in (cache.cached_key, cache.cached_value) for t in (c.data, c.exp)]
    return [cache.cached_key.clone(), cache.cached_value.clone()]


def _eq(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, what
    assert torch.equal(a, b), "%s differs: max |diff| %.3e" % (what, float((a.float() - b.float()).abs().max()))


class Layer:
    """one attention layer's decode inputs: a cache of max_length K prefilled eagerly with K - n rows, and n steps of
    q / k / v rows; left padding of the second sequence (positions = slot - pad)"""

    def __init__(self, kind, rope, B, K, n, H, seed, table):
        from lwm_b200.kv_cache import ShardedKVCache
        self.cdt, self.dt = KINDS[kind]
        self.B, self.K, self.n, self.H, self.table = B, K, n, H, table if rope else None
        self.pad = torch.tensor([0, 5][:B], dtype=torch.int32)
        am = torch.ones(B, K, dtype=torch.int64)
        am[1:, :5] = 0
        self.am = am.cuda()
        self.q = [_randn((B, 1, H, D), seed + 3 * t, self.dt, 3.0) for t in range(n)]
        self.k = [_randn((B, 1, H, D), seed + 3 * t + 1, self.dt) for t in range(n)]
        self.v = [_randn((B, 1, H, D), seed + 3 * t + 2, self.dt) for t in range(n)]
        P = K - n
        kp, vp = _randn((B, P, H, D), seed - 1, self.dt), _randn((B, P, H, D), seed - 2, self.dt)
        self.cache = ShardedKVCache(B, K, H, D, dtype=self.cdt)
        pos = (torch.arange(P)[None] - self.pad[:, None].long()).clamp(min=0)
        self.cache.concatenate(kp, vp, **self.kw(pos.cuda()))

    def kw(self, pos, q=False):
        if self.table is None:
            return {}
        return dict(freqs_cis=self.table, position_ids=pos, **({"rotate_k": False} if q else {}))

    def step(self, q, k, v, index, pos):
        """one decode step; index: int or the cursor (0-d device tensor), pos [B,1] (host or device)"""
        from lwm_b200.ringattention import decode_attention_mask, ringattention_inference
        mask = decode_attention_mask(self.am, 1, index, self.K)
        ck, cv = self.cache.concatenate(k, v, **self.kw(pos))
        return ringattention_inference(q, ck, cv, mask, **self.kw(pos, q=True))

    def eager(self):
        outs = []
        for t in range(self.n):
            idx = self.cache.cache_index
            pos = (idx - self.pad[:, None]).long()
            outs.append(self.step(self.q[t], self.k[t], self.v[t], idx, pos))
        return outs

    def static_inputs(self):
        self.q_in, self.k_in, self.v_in = (torch.empty_like(x[0]) for x in (self.q, self.k, self.v))
        self.pad_dev = self.pad.cuda()
        self.load(0)

    def load(self, t):
        self.q_in.copy_(self.q[t])
        self.k_in.copy_(self.k[t])
        self.v_in.copy_(self.v[t])

    def graph_step(self):
        cur = self.cache.cursor
        pos = (cur - self.pad_dev).view(self.B, 1)           # derived before the write advances the cursor
        return self.step(self.q_in, self.k_in, self.v_in, cur, pos)


def _capture(layers):
    """warm up on a side stream (then rewind the cursors), capture one step of every layer with host synchronisations
    turned into errors -> (graph, static outputs)"""
    for ly in layers:
        ly.static_inputs()
    start = [ly.cache.cache_index for ly in layers]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for ly in layers:
            ly.graph_step()
    torch.cuda.current_stream().wait_stream(s)
    for ly, i in zip(layers, start):
        ly.cache.cache_index = i
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        torch.cuda.set_sync_debug_mode("error")
        try:
            outs = [ly.graph_step() for ly in layers]
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return g, outs


def _replay(layers, g, outs, steps):
    got = []
    for t in range(steps):
        for ly in layers:
            ly.load(t)
        g.replay()
        got.append([o.clone() for o in outs])
    torch.cuda.synchronize()
    return got


@pytest.mark.parametrize("K", [2048, 2049, 16384])
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("rope", [False, True], ids=["plain", "rope"])
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_replayed_decode_steps_are_bit_identical_to_eager(kind, rope, B, K):
    from lwm_b200.rope import precompute_freqs_cis
    table = precompute_freqs_cis(D, 1 << 16, 1e4)
    n, H = 8, 4
    seed = 1000 * B + K + 7 * rope
    eager, graphed = (Layer(kind, rope, B, K, n, H, seed, table) for _ in range(2))
    assert graphed.cache.take_errors() == 0
    want = eager.eager()
    g, outs = _capture([graphed])
    got = _replay([graphed], g, outs, n)
    for t in range(n):
        _eq(got[t][0], want[t], "step %d" % t)
    for i, (a, b) in enumerate(zip(_state(graphed.cache), _state(eager.cache))):
        _eq(a, b, "cache tensor %d" % i)
    assert graphed.cache.cache_index == eager.cache.cache_index == K
    assert graphed.cache.take_errors() == 0


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_one_graph_holds_32_layers(kind):
    from lwm_b200.rope import precompute_freqs_cis
    table = precompute_freqs_cis(D, 1 << 16, 1e4)
    n, H, K, B = 8, 2, 2049, 2
    eager = [Layer(kind, True, B, K, n, H, 50 * i, table) for i in range(32)]
    graphed = [Layer(kind, True, B, K, n, H, 50 * i, table) for i in range(32)]
    want = [ly.eager() for ly in eager]
    g, outs = _capture(graphed)
    got = _replay(graphed, g, outs, n)
    for i in range(32):
        for t in range(n):
            _eq(got[t][i], want[i][t], "layer %d step %d" % (i, t))
        for j, (a, b) in enumerate(zip(_state(graphed[i].cache), _state(eager[i].cache))):
            _eq(a, b, "layer %d cache tensor %d" % (i, j))
        assert graphed[i].cache.cache_index == eager[i].cache.cache_index
    assert graphed[0].cache.take_errors() == 0


@pytest.mark.parametrize("kind", sorted(KINDS))
def test_replay_past_the_cache_or_the_table_writes_nothing_and_sets_the_error_word(kind):
    from lwm_b200 import rope as R
    table = R.precompute_freqs_cis(D, 1 << 16, 1e4)
    n, H, K, B = 1, 2, 2048, 2
    ly = Layer(kind, True, B, K, n, H, 99, table)
    assert ly.cache.take_errors() == 0
    g, outs = _capture([ly])
    _replay([ly], g, outs, 1)                         # writes the last slot, K - 1
    assert ly.cache.take_errors() == 0
    before = _state(ly.cache)
    g.replay()                                         # slot K: past the cache
    torch.cuda.synchronize()
    assert ly.cache.take_errors() == R.ERR_SLOT
    for i, (a, b) in enumerate(zip(_state(ly.cache), before)):
        _eq(a, b, "cache tensor %d after the overflow" % i)
    assert ly.cache.cache_index == K + 1

    # a position outside the table: the pad makes slot - pad exceed max_position
    ly.cache.cache_index = K - 1
    ly.pad_dev.fill_(-(1 << 16))
    g.replay()
    torch.cuda.synchronize()
    assert ly.cache.take_errors() == R.ERR_POSITION
    for i, (a, b) in enumerate(zip(_state(ly.cache), before)):
        _eq(a, b, "cache tensor %d after the bad position" % i)
    assert ly.cache.cache_index == K


@pytest.mark.parametrize("kind", sorted(KINDS))
@pytest.mark.parametrize("rope", [False, True], ids=["plain", "rope"])
def test_cursor_write_on_emulated_ranks_matches_the_host_index_write(kind, rope):
    """4 ranks of 48 rows; slots on a rank's first and last row and in the middle: only the owner's shard changes, and
    it changes as the write at the host index (the CPU path of concatenate's decode: write_rope / write_q8 / copy_)"""
    from lwm_b200.kv_cache import ShardedKVCache, kv_cache_write_q8, kv_cache_write_rope
    from lwm_b200.rope import precompute_freqs_cis
    table = precompute_freqs_cis(D, 1 << 16, 5e5)
    cdt, dt = KINDS[kind]
    W, L, B, H = 4, 48, 3, 8
    for step, slot in enumerate((0, 47, 48, 100, 191)):
        k = _randn((B, 1, H, D), 10 + step, dt, 4.0)
        v = _randn((B, 1, H, D), 20 + step, dt)
        pos = (slot + 7 * torch.arange(B)[:, None]).to(torch.int32).cuda()
        kw = dict(freqs_cis=table, position_ids=pos) if rope else {}
        for r in range(W):
            cache = ShardedKVCache(B, W * L, H, D, dtype=cdt, comm=types.SimpleNamespace(world=W, rank=r))
            ref = ShardedKVCache(B, W * L, H, D, dtype=cdt, comm=types.SimpleNamespace(world=W, rank=r))
            cache.cache_index = slot
            before = _state(cache)
            cache.concatenate(k, v, **kw)
            cur = slot - r * L
            if 0 <= cur < L:
                p, inv = (pos, table.inv_freq) if rope else (None, None)
                if kind == "int8":
                    kv_cache_write_q8(k, v, 0, 1, ref.cached_key, ref.cached_value, cur, p, inv)
                elif rope:
                    kv_cache_write_rope(k, v, 0, 1, ref.cached_key, ref.cached_value, cur, p, inv)
                else:
                    ref.cached_key[:, cur].copy_(k[:, 0])
                    ref.cached_value[:, cur].copy_(v[:, 0])
                want = _state(ref)
            else:
                want = before
            for i, (a, b) in enumerate(zip(_state(cache), want)):
                _eq(a, b, "slot %d rank %d tensor %d" % (slot, r, i))
            assert cache.cache_index == slot + 1 and int(cache.cursor) == slot + 1
    assert cache.take_errors() == 0
