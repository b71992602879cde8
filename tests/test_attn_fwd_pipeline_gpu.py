"""GPU parity of the forward tile kernel for the shapes its software pipeline depends on: two and three KV tiles
per CTA (the shortest runs through prologue, loop and epilogue), a long loop over many KV tiles for one Q tile (the
K/V ring wraps many times), causal offsets where only one warpgroup's rows are masked on some iteration, bias and
segment ids (every iteration takes the masked path), a two-step carry, and B > 1 with an odd head count. Each case
runs in both precision modes against the float64 oracle of oracle/attn_dense.py; tolerances as in
test_attn_fwd_gpu.py (bf16: the bf16 `out`) and test_attn_fp16_mode_gpu.py (fp16: the fp32 `out_f32`)."""
import numpy as np
import pytest
import torch

from helpers import make_qkv, rel_fro, to_np

pytestmark = pytest.mark.gpu
TOL_OUT = {"bf16": 3e-3, "fp16": 1e-3}
TOL_LSE = {"bf16": 2e-3, "fp16": 1e-3}


def _run(mode, q, k, v, causal, q_pos0=0, k_pos0=0, bias=None, seg=None):
    """one launch with first = last = 1 -> (out as float32, lse); fp16 mode returns the un-rounded out_f32"""
    from lwm_b200 import ringattention as ra
    B, Sq, H, D = q.shape
    out = torch.empty_like(q)
    lse = torch.empty(B, H, Sq, dtype=torch.float32, device="cuda")
    if mode == "bf16":
        ra.fwd_step(q, k, v, out, lse, None, None, None, q_pos0, k_pos0, causal, bias, seg, True, True)
        res = out
    else:
        (q16, sq), (k16, sk), (v16, sv) = [ra.to_f16(t) for t in (q, k, v)]
        res = torch.empty(B, Sq, H, D, dtype=torch.float32, device="cuda")
        ra.fwd_step(q16, k16, v16, out, lse, None, None, None, q_pos0, k_pos0, causal, bias, seg, True, True,
                    scales=(sq, sk, sv), out_f32=res)
    torch.cuda.synchronize()
    return to_np(res), to_np(lse)


def _check(mode, got, q, k, v, rows=None, **kw):
    from oracle.attn_dense import attention_dense
    ref, ref_lse = attention_dense(to_np(q), to_np(k), to_np(v), return_lse=True, **kw)
    out, lse = got
    assert np.isfinite(out).all() and np.isfinite(lse).all()
    if rows is not None:     # [B, Sq] bool: query rows the reference defines
        for b in range(out.shape[0]):
            assert rel_fro(out[b, rows[b]], ref[b, rows[b]]) < TOL_OUT[mode]
            assert np.abs(lse[b][:, rows[b]] - ref_lse[b][:, rows[b]]).max() < TOL_LSE[mode]
        return
    assert rel_fro(out, ref) < TOL_OUT[mode], rel_fro(out, ref)
    assert np.abs(lse - ref_lse).max() < TOL_LSE[mode]


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
@pytest.mark.parametrize("n_kv", [2, 3])
def test_two_and_three_kv_tiles(mode, n_kv):
    q, k, v = make_qkv(1, 256, 128 * n_kv, 2, seed=201 + n_kv)
    _check(mode, _run(mode, q, k, v, False), q, k, v, causal=False)


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
def test_causal_one_to_three_kv_tiles(mode):
    # the three Q tiles see 1, 2 and 3 KV tiles
    q, k, v = make_qkv(1, 384, 384, 2, seed=204)
    _check(mode, _run(mode, q, k, v, True), q, k, v, causal=True)


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
def test_long_loop_one_q_tile(mode):
    # 64 KV tiles stream past one Q tile: every ring slot is reused many times
    q, k, v = make_qkv(1, 128, 8192, 1, seed=205)
    _check(mode, _run(mode, q, k, v, False), q, k, v, causal=False)


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
@pytest.mark.parametrize("q_pos0", [64, 192])
def test_causal_offset_masks_one_warpgroup(mode, q_pos0):
    # the Q tile's first 64 rows end before a KV tile that its last 64 rows reach: on that iteration one
    # warpgroup's rows are all masked and the other's are on the diagonal
    q, k, v = make_qkv(1, 256, 512, 2, seed=206 + q_pos0)
    _check(mode, _run(mode, q, k, v, True, q_pos0=q_pos0), q, k, v, causal=True, q_pos0=q_pos0)


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
def test_bias_and_segments_every_tile_masked(mode):
    from oracle.attn_dense import finfo_min
    B, S, H = 2, 640, 2
    q, k, v = make_qkv(B, S, S, H, seed=207)
    bias = torch.zeros(B, S, dtype=torch.float32)
    bias[0, :70] = finfo_min("bf16")
    bias[1, :200] = finfo_min("bf16")
    seg = torch.zeros(B, S, dtype=torch.int32)
    seg[0, 250:] = 1
    seg[1, 300:450] = 1
    seg[1, 450:] = 2
    got = _run(mode, q, k, v, True, bias=bias.cuda(), seg=seg.cuda())
    _check(mode, got, q, k, v, rows=bias.numpy() == 0, causal=True, attn_bias=bias.numpy(), segment_ids=seg.numpy())


def test_fp16_two_step_carry_matches_one_step():
    """ring order on one GPU in fp16 mode: the diagonal half of K/V first (first=1, last=0), then the earlier half
    (first=0, last=1), from the same fp16 operand copies as one launch over all of K/V"""
    from lwm_b200 import ringattention as ra
    B, S, H, D = 1, 1024, 2, 128
    half = S // 2
    q, k, v = make_qkv(B, half, S, H, seed=208)
    (q16, sq), (k16, sk), (v16, sv) = [ra.to_f16(t) for t in (q, k, v)]
    out = torch.empty_like(q)
    lse = torch.empty(B, H, half, dtype=torch.float32, device="cuda")
    one = torch.empty(B, half, H, D, dtype=torch.float32, device="cuda")
    ra.fwd_step(q16, k16, v16, out, lse, None, None, None, half, 0, True, None, None, True, True,
                scales=(sq, sk, sv), out_f32=one)
    lse2 = torch.empty_like(lse)
    two = torch.empty_like(one)
    acc = (torch.empty(B, half, H, D, dtype=torch.float32, device="cuda"),
           torch.empty(B, H, half, dtype=torch.float32, device="cuda"),
           torch.empty(B, H, half, dtype=torch.float32, device="cuda"))
    ra.fwd_step(q16, k16[:, half:].contiguous(), v16[:, half:].contiguous(), out, lse2, *acc, half, half, True, None,
                None, True, False, scales=(sq, sk, sv), out_f32=two)
    ra.fwd_step(q16, k16[:, :half].contiguous(), v16[:, :half].contiguous(), out, lse2, *acc, half, 0, True, None,
                None, False, True, scales=(sq, sk, sv), out_f32=two)
    torch.cuda.synchronize()
    assert rel_fro(to_np(two), to_np(one)) < 1e-3
    assert np.abs(to_np(lse2) - to_np(lse)).max() < 1e-3
    _check("fp16", (to_np(two), to_np(lse2)), q, k, v, causal=True, q_pos0=half, k_pos0=0)


@pytest.mark.parametrize("mode", ["bf16", "fp16"])
def test_batch2_heads3(mode):
    q, k, v = make_qkv(2, 512, 512, 3, seed=209)
    _check(mode, _run(mode, q, k, v, True), q, k, v, causal=True)
