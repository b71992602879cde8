"""The fp8 mode (ringattention(..., precision='fp8')) on the GPU: the e4m3 staging bit for bit against torch's cast,
the forward against float64 at small and long-context shapes, its instances and paths against each other, and the
peer-memory ring on emulated ranks.

The acceptance bound calibrates itself on the inputs of each case: with e = max |out - ref| / max |ref|,
    e(fp8) <= e(model) + e(fp16) + SLACK,
where the model (tests/e4m3_attn_model.py) is exact attention over the staged e4m3 q, k and fp16 v, and fp16 is the
fp16 mode's forward on the same inputs: what the fp8 kernel adds to the operand rounding is the fp16 mode's own error,
plus what the model leaves out. SLACK = 2.5e-4: on fp32 inputs, whose fp16-mode error is only ~1e-4 (the output is not
rounded to bf16), the kernel sits up to 1.6e-4 further from the model than the fp16 mode sits from the oracle
(S = 512 causal, H100). The model takes the S GEMM as an exact sum of the e4m3 products; the tensor cores' own
accumulation of an FP8 GEMM is the likely rest (DESIGN.md §5)."""
import threading

import pytest
import torch

import e4m3_attn_model as em
import score_distributions as sd

pytestmark = pytest.mark.gpu

KW = dict(axis_name="sp", float32_logits=True, cache_idx=None, blockwise_kwargs=dict(causal_block_size=1))
KW_NONCAUSAL = dict(axis_name="sp", float32_logits=True, cache_idx=None, blockwise_kwargs=dict(causal_block_size=None))


def _ra():
    from lwm_b200 import ringattention as ra
    return ra


def _fp8_bytes(x, scale):
    """torch's cast of x / scale to e4m3, as bytes"""
    return (x.float() / scale).to(torch.float8_e4m3fn).view(torch.uint8)


# ---------------------------------------------------------------------------------------------------- staging
def _staging_input(dtype, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(2, 256, 4, 128, generator=g, device="cuda") * 3.0
    # every binade of e4m3 down to its subnormals and below, relative to the tensor maximum
    x[0, :64] *= torch.exp2(-torch.randint(0, 24, (64, 4, 128), generator=g, device="cuda").float())
    return x.to(dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_staging_matches_the_torch_cast(dtype):
    ra = _ra()
    x = _staging_input(dtype)
    s = torch.empty(1, dtype=torch.float32, device="cuda")
    ra.PeerOpsE4m3.scale_of(x, s)
    assert float(s) == em.pow2_scale(x.cpu(), 7)
    y = torch.empty(x.shape, dtype=torch.float8_e4m3fn, device="cuda")
    ra.PeerOpsE4m3.stage(x, y, s)
    torch.cuda.synchronize()
    assert torch.equal(y.view(torch.uint8), _fp8_bytes(x, float(s)))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_rotating_staging_matches_rotate_then_cast(dtype):
    from lwm_b200 import rope
    ra = _ra()
    x = _staging_input(dtype, seed=1)
    table = rope.precompute_freqs_cis(128, 65536)
    pos = torch.randint(0, 65536, (2, 256), dtype=torch.int32, device="cuda")
    xr = rope.rotate(x, table, dtype, position_ids=pos)
    s = torch.empty(1, dtype=torch.float32, device="cuda")
    ra.PeerOpsE4m3.scale_of_rope(x, s, pos, table.inv_freq)
    assert float(s) == em.pow2_scale(xr.cpu(), 7)
    y = torch.empty(x.shape, dtype=torch.float8_e4m3fn, device="cuda")
    ra.PeerOpsE4m3.stage_rope(x, y, s, pos, table.inv_freq)
    torch.cuda.synchronize()
    assert torch.equal(y.view(torch.uint8), _fp8_bytes(xr, float(s)))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_nonfinite_inputs_become_the_nan_byte(dtype):
    ra = _ra()
    x = _staging_input(dtype, seed=2)
    bad = [(0, 3, 1, 5, float("inf")), (1, 7, 2, 0, float("-inf")), (1, 9, 3, 127, float("nan")),
           (0, 200, 0, 64, -float("nan"))]
    for b, s_, h, d, val in bad:
        x[b, s_, h, d] = val
    s = torch.empty(1, dtype=torch.float32, device="cuda")
    ra.PeerOpsE4m3.scale_of(x, s)        # the largest FINITE |x|: unchanged by the planted values
    clean = x.clone()
    for b, s_, h, d, _ in bad:
        clean[b, s_, h, d] = 0
    assert float(s) == em.pow2_scale(clean.cpu(), 7)
    y = torch.empty(x.shape, dtype=torch.float8_e4m3fn, device="cuda")
    ra.PeerOpsE4m3.stage(x, y, s)
    torch.cuda.synchronize()
    got = y.view(torch.uint8)
    for b, s_, h, d, val in bad:
        byte = int(got[b, s_, h, d])
        assert byte & 0x7F == 0x7F, (val, byte)            # a NaN byte, never +-448 (0x7e / 0xfe)
        if val in (float("inf"), float("-inf")):
            assert byte == (0x80 if val < 0 else 0) | 0x7F, (val, byte)    # torch's cast: the sign of the inf
    finite = torch.isfinite(x)
    assert torch.equal(got[finite], _fp8_bytes(x, float(s))[finite])


# ---------------------------------------------------------------------------------------------------- small shapes
def _errors(q, k, v, causal=True, **kw):
    """(e fp8, e model, e fp16, fp8 output) against the float64 dense oracle, relative to max |ref|"""
    from oracle.attn_dense import attention_dense
    ra = _ra()
    bias = kw.get("attn_bias")
    with torch.no_grad():
        o8 = ra.ringattention(q, k, v, bias, None, precision="fp8", **(KW if causal else KW_NONCAUSAL))
        o16 = ra.ringattention(q, k, v, bias, None, precision="fp16", **(KW if causal else KW_NONCAUSAL))
    torch.cuda.synchronize()
    okw = dict(causal=causal)
    if bias is not None:
        okw["attn_bias"] = bias.float().cpu().numpy()
    qc, kc, vc = [t.cpu() for t in (q, k, v)]
    ref = attention_dense(qc.double().numpy(), kc.double().numpy(), vc.double().numpy(), **okw)
    model, _ = em.attention_e4m3_model(qc, kc, vc, **okw)
    return em.err_vs_max(o8.double().cpu(), ref), em.err_vs_max(model, ref), em.err_vs_max(o16.double().cpu(), ref), o8


SLACK = 2.5e-4


def _check(label, e8, em_, e16):
    print("%s fp8 %.2e model %.2e fp16 %.2e" % (label, e8, em_, e16))
    assert e8 <= em_ + e16 + SLACK, (label, e8, em_, e16)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("S", [128, 512, 2048])
def test_forward_against_the_dense_oracle(S, causal, dtype):
    from helpers import make_qkv
    q, k, v = [t.to(dtype) for t in make_qkv(1, S, S, 2, seed=S + causal)]
    e8, em_, e16, o8 = _errors(q, k, v, causal)
    assert o8.dtype == dtype
    _check("S=%d causal=%d %s" % (S, causal, dtype), e8, em_, e16)


def test_cached_prefill_sq_ne_sk():
    from helpers import make_qkv
    q, k, v = make_qkv(2, 256, 1024, 2, seed=7)
    e8, em_, e16, _ = _errors(q, k, v, True)
    _check("Sq=256 Sk=1024", e8, em_, e16)


def test_padding_bias_takes_the_block_map():
    from helpers import make_qkv
    ra = _ra()
    S = 1024
    q, k, v = make_qkv(2, S, S, 2, seed=11)
    mask = torch.ones(2, S, dtype=torch.int32, device="cuda")
    mask[1, 700:] = 0
    bias = ra.attention_bias_from_mask(mask)
    e8, em_, e16, _ = _errors(q, k, v, True, attn_bias=bias)
    _check("S=1024 padding bias", e8, em_, e16)


@pytest.mark.parametrize("causal", [True, False])
def test_plain_and_block_map_instances_are_bit_identical(causal):
    """the step with a zero bias, once over its block map (attn_fwd_e4m3_kernel<true>) and once without
    (attn_fwd_e4m3_kernel<false>, which reads the bias on every tile)"""
    from helpers import make_qkv
    ra = _ra()
    S, B, H = 1024, 2, 2
    q, k, v = make_qkv(B, S, S, H, seed=3)
    E, F = ra.PeerOpsE4m3, ra.PeerOpsF16
    sq, sk, sv = [torch.empty(1, dtype=torch.float32, device="cuda") for _ in range(3)]
    E.scale_of(q, sq), E.scale_of(k, sk), F.scale_of(v, sv)
    q8, k8 = [torch.empty(t.shape, dtype=torch.float8_e4m3fn, device="cuda") for t in (q, k)]
    v16 = torch.empty(v.shape, dtype=torch.float16, device="cuda")
    E.stage(q, q8, sq), E.stage(k, k8, sk), F.stage(v, v16, sv)
    bias = torch.zeros(B, S, dtype=torch.float32, device="cuda")
    outs = []
    for tm in (None, ra.step_tilemap(B, S, S, 0, 0, causal, bias, None, bwd=False)[:2]):
        out = torch.empty(q.shape, dtype=torch.bfloat16, device="cuda")
        o32 = torch.empty(q.shape, dtype=torch.float32, device="cuda")
        lse = torch.empty((B, H, S), dtype=torch.float32, device="cuda")
        ra.fwd_e4m3_step(q8, k8, v16, out, lse, None, None, None, 0, 0, causal, bias, None, True, True, (sq, sk, sv),
                         out_f32=o32, tilemap=tm)
        outs.append((out, o32, lse))
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("rotate_k", [True, False])
def test_rotary_keywords_are_bit_identical_to_rotating_first(rotate_k, dtype):
    from helpers import make_qkv
    from lwm_b200 import rope
    ra = _ra()
    Sq, Sk = (512, 512) if rotate_k else (256, 1024)
    q, k, v = [t.to(dtype) for t in make_qkv(2, Sq, Sk, 2, seed=5)]
    table = rope.precompute_freqs_cis(128, 65536)
    pos = (torch.arange(Sq, dtype=torch.int32, device="cuda") + 1000)[None].repeat(2, 1)
    with torch.no_grad():
        fused = ra.ringattention(q, k, v, precision="fp8", freqs_cis=table, position_ids=pos, rotate_k=rotate_k, **KW)
        if rotate_k:
            qr, kr = rope.apply_rotary_emb(q, k, table, dtype, position_ids=pos)
        else:
            qr, kr = rope.rotate(q, table, dtype, position_ids=pos), k
        first = ra.ringattention(qr, kr, v, precision="fp8", **KW)
    assert torch.equal(fused, first)


def test_quantized_kv_cache_prefill():
    """an 8-bit KV cache is dequantized transiently: the same bits as passing the dequantized tensors"""
    from helpers import make_qkv
    from lwm_b200 import kv_cache
    ra = _ra()
    q, k, v = make_qkv(1, 256, 1024, 2, seed=9)
    ck, cv = kv_cache.QuantizedKV.zeros(1, 1024, 2), kv_cache.QuantizedKV.zeros(1, 1024, 2)
    kv_cache.kv_cache_write_q8(k, v, 0, 1024, ck, cv, 0)
    with torch.no_grad():
        o_q = ra.ringattention(q, ck, cv, precision="fp8", **KW)
        o_d = ra.ringattention(q, ck.dequantize(q.dtype), cv.dequantize(q.dtype), precision="fp8", **KW)
    assert torch.equal(o_q, o_d)


# ---------------------------------------------------------------------------------------------------- long context
DISTRIBUTIONS = {
    "white_sigma1": None, "white_sigma3": None,
    "sink_gap18": ("sink", dict(gap=18.0, sigma=0.5)),
    "recency": ("recency", {}),
    "peaked": ("peaked", {}),
}


def _long_inputs(name, S, H):
    if DISTRIBUTIONS[name] is None:
        sigma = 1.0 if name == "white_sigma1" else 3.0
        g = torch.Generator().manual_seed(S)
        q, k, v = [torch.randn(1, S, H, 128, generator=g) for _ in range(3)]
        k = k * sigma
        return [t.to(torch.bfloat16).float() for t in (q, k, v)]
    kind, kw = DISTRIBUTIONS[name]
    return [sd.shard(kind, n, 0, S, S, H, **kw) for n in ("q", "k", "v")]


@pytest.mark.parametrize("name", sorted(DISTRIBUTIONS))
@pytest.mark.parametrize("S", [32768, 131072])
def test_long_context_against_the_row_oracle(S, name):
    from oracle.attn_rows import attention_rows, sample_rows
    ra = _ra()
    H = 1
    q, k, v = _long_inputs(name, S, H)
    rows = sample_rows(S)
    qd, kd, vd = [t.cuda().to(torch.bfloat16) for t in (q, k, v)]
    with torch.no_grad():
        o8 = ra.ringattention(qd, kd, vd, precision="fp8", **KW)[0, rows].double().cpu()
        o16 = ra.ringattention(qd, kd, vd, precision="fp16", **KW)[0, rows].double().cpu()
    qm, km, vm = em.model_operands(q, k, v)
    worst = dict(fp8=0.0, model=0.0, fp16=0.0)
    for h in range(H):
        ref = attention_rows(q[0, rows, h], rows, k[0, :, h], v[0, :, h])["out"]
        mod = attention_rows(qm[0, rows, h], rows, km[0, :, h], vm[0, :, h])["out"]
        for n, a in (("fp8", o8[:, h]), ("model", mod), ("fp16", o16[:, h])):
            worst[n] = max(worst[n], em.err_vs_max(a, ref))
    _check("S=%d %s" % (S, name), worst["fp8"], worst["model"], worst["fp16"])


# ---------------------------------------------------------------------------------------------------- peer ring
@pytest.mark.parametrize("world,causal", [(2, True), (4, True), (4, False)])
def test_peer_ring_matches_one_gpu(world, causal):
    """ranks as threads on one GPU (tests/peer_emulation.py). Every shard holds the same largest |q|, |k| and |v|, so
    every owner's scales are the one-GPU scales and the staged bytes are the same. The outputs (fp32) differ by the
    fp32 carry merges and by P, which each launch packs in fp16 against its own running row max: 1e-5 .. 1.1e-4 of
    max |out| measured (H100). K and Q travel at one byte per element."""
    from helpers import make_qkv
    from lwm_b200 import ring_peer as rp, ring_schedule as rs
    from peer_emulation import EmuTransport, EmuWorld
    ra = _ra()
    Sl, H = 512, 2
    q, k, v = [t.float() for t in make_qkv(1, world * Sl, world * Sl, H, seed=world)]   # fp32 out: no final rounding
    for t in (q, k, v):
        for r in range(world):
            t[0, r * Sl + 5, 0, 0] = 6.0       # above every N(0,1) sample: one |max| for the whole tensor
    with torch.no_grad():
        one = ra.ringattention(q, k, v, precision="fp8", **(KW if causal else KW_NONCAUSAL))
    dev = torch.device("cuda", 0)
    emu = EmuWorld(world, device=dev)
    outs, fails = {}, []

    def worker(rank):
        try:
            torch.cuda.set_device(dev)
            tr = EmuTransport(emu, rank)
            plan = rs.make_peer_plan(world, rank, Sl, Sl, causal, "zigzag" if causal else "contiguous")
            sl = slice(rank * Sl, (rank + 1) * Sl)
            with torch.no_grad():
                out, _ = rp.run_forward(plan, q[:, sl].contiguous(), k[:, sl].contiguous(), v[:, sl].contiguous(),
                                        None, None, causal, ra.PeerOpsE4m3, tr, True)
            outs[rank] = out
            pulled = sum(n for op, _, n in tr.log if op == "pull")
            outs[("log", rank)] = pulled
        except BaseException:   # noqa: BLE001  (reported by the main thread)
            import traceback
            fails.append(traceback.format_exc())
            emu.barrier.abort()

    ts = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    torch.cuda.synchronize()
    assert not any(t.is_alive() for t in ts) and not fails, fails[:1]
    ring = torch.cat([outs[r] for r in range(world)], dim=1)
    e = float((ring - one).abs().max() / one.abs().max())
    print("world=%d causal=%d ring vs one GPU %.2e, bytes pulled per rank %s"
          % (world, causal, e, [outs[("log", r)] for r in range(world)]))
    assert e < 5e-4, e
