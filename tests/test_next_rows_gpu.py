"""GPU parity (through the C ABI) of the §8f next rows: rotary embedding of the attention prologue against the
fixture produced by the reference's own `apply_rotary_emb`, and the vision token framing (bit-exact).
Tolerances: fp32 output: |err| <= 1.5e-6 (cos/sin are within 1 ulp of the reference's table, inputs are O(1));
bf16 output: equal to the fp32 oracle rounded to bf16, except one bf16 ulp on rare rounding ties (near-cancelled
results are compared on absolute error, their ulp being arbitrarily small)."""
import os

import numpy as np
import pytest
import torch

from helpers import to_np

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("tag", ("t1e4", "t5e7"))
def test_rope_matches_reference_fixture_fp32(tag):
    from lwm_b200.rope import apply_rotary_emb, precompute_freqs_cis
    g = np.load(os.path.join(GOLD, "rope_reference.npz"))
    table = precompute_freqs_cis(128, int(g[tag + "_max_pos"]), theta=float(g[tag + "_theta"]))
    xq, xk = torch.from_numpy(g[tag + "_xq"]).cuda(), torch.from_numpy(g[tag + "_xk"]).cuda()
    pos = torch.from_numpy(g[tag + "_pos"]).cuda()
    oq, ok = apply_rotary_emb(xq, xk, table, torch.float32, position_ids=pos)
    torch.cuda.synchronize()
    assert np.abs(to_np(oq) - g[tag + "_oq"]).max() <= 1.5e-6
    assert np.abs(to_np(ok) - g[tag + "_ok"]).max() <= 1.5e-6


def test_rope_bf16_io_and_large_shape():
    """bf16 in / bf16 out (the measured mode) on a ragged token count (not a multiple of the CTA's 4 positions) and
    32 heads; reference = the numpy oracle on the bf16-rounded inputs, rounded to bf16."""
    from lwm_b200.rope import apply_rotary_emb, precompute_freqs_cis
    from oracle import rope as R
    B, S, H = 1, 1023, 32
    g = torch.Generator().manual_seed(3)
    xq = torch.randn(B, S, H, 128, generator=g).to(torch.bfloat16)
    xk = torch.randn(B, S, H, 128, generator=g).to(torch.bfloat16)
    pos = torch.randint(0, 1 << 20, (B, S), generator=g, dtype=torch.int32)
    table = precompute_freqs_cis(128, 1 << 20, theta=5e7)
    oq, ok = apply_rotary_emb(xq.cuda(), xk.cuda(), table, torch.bfloat16, position_ids=pos.cuda())
    torch.cuda.synchronize()
    rq, rk = R.rope_reference(xq.float().numpy(), xk.float().numpy(), pos.numpy(), 5e7, 1 << 20)
    for got, ref in ((oq, rq), (ok, rk)):
        ref16 = torch.from_numpy(ref).to(torch.bfloat16)
        differs = (got.cpu() != ref16)
        assert float(differs.float().mean()) < 2e-3        # identical bf16 values except on rare rounding ties ...
        err = np.abs(to_np(got) - ref)
        assert (err <= 2.0 ** -8 * np.abs(ref) + 1e-6).all()  # ... which move by one bf16 ulp at most


def test_rope_backward_is_the_conjugate_rotation():
    from lwm_b200.rope import apply_rotary_emb, precompute_freqs_cis
    from oracle import rope as R
    B, S, H = 2, 64, 2
    g = torch.Generator().manual_seed(4)
    xq = torch.randn(B, S, H, 128, generator=g).cuda().requires_grad_(True)
    xk = torch.randn(B, S, 1, 128, generator=g).cuda().requires_grad_(True)
    gq, gk = torch.randn(B, S, H, 128, generator=g), torch.randn(B, S, 1, 128, generator=g)
    pos = torch.arange(S, dtype=torch.int32)[None].expand(B, S).contiguous() + 777
    table = precompute_freqs_cis(128, 4096, theta=10000.0)
    oq, ok = apply_rotary_emb(xq, xk, table, torch.float32, position_ids=pos.cuda())
    (oq * gq.cuda()).sum().backward(retain_graph=True)
    (ok * gk.cuda()).sum().backward()
    tab = R.precompute_freqs_cis(128, 4096, 10000.0)
    dq, dk = R.apply_rotary_emb(gq.numpy(), gk.numpy(), np.conj(np.take(tab, pos.numpy(), axis=0)))
    assert np.abs(to_np(xq.grad) - dq).max() <= 2e-6 and np.abs(to_np(xk.grad) - dk).max() <= 2e-6


def test_rope_rejects_bad_arguments():
    from lwm_b200 import _lib
    from lwm_b200.rope import apply_rotary_emb, precompute_freqs_cis
    table = precompute_freqs_cis(128, 128)
    x = torch.zeros(1, 8, 1, 128, device="cuda")
    with pytest.raises(_lib.LwmError):
        apply_rotary_emb(x, x, table, torch.float32, position_ids=torch.full((1, 8), 128, device="cuda"))
    with pytest.raises(_lib.LwmError):
        precompute_freqs_cis(64, 128)
    with pytest.raises(_lib.LwmError):
        apply_rotary_emb(x, x, table, torch.float16, position_ids=torch.zeros(1, 8, dtype=torch.int32, device="cuda"))


@pytest.mark.parametrize("tag", ("f1", "f5", "f9sel4"))
def test_frame_tokens_bit_exact_vs_reference_fixture(tag):
    from lwm_b200.vision_tokens import frame_tokens, unframe_tokens
    g = np.load(os.path.join(GOLD, "vision_tokens_reference.npz"))
    codes = torch.from_numpy(g[tag + "_codes"]).cuda().reshape(-1, 16, 16)
    toks = frame_tokens(codes, max_n_frames=int(g[tag + "_max_n_frames"]))
    torch.cuda.synchronize()
    want = g[tag + "_tokens"][2:-3]             # strip bos, <vision> ... </vision> (2 ids), eos of the fixture
    assert toks.dtype == torch.int32 and np.array_equal(toks.cpu().numpy(), want)
    back = unframe_tokens(toks)
    assert back.shape[1:] == (16, 16)
    if int(g[tag + "_max_n_frames"]) < 0:
        assert np.array_equal(back.cpu().numpy().reshape(-1), g[tag + "_codes"])


def test_frame_tokens_batched_clip_of_vqgan_size():
    """[B,T,16,16] clips (16 frames, as in the benchmark clip): round trip + delimiter positions, and chaining from VQGAN.encode"""
    from lwm_b200.vision_tokens import EOF_TOKEN, EOV_TOKEN, frame_tokens, unframe_tokens
    from oracle import vision_tokens as V
    g = torch.Generator().manual_seed(9)
    codes = torch.randint(0, 8192, (3, 16, 16, 16), generator=g, dtype=torch.int32)
    toks = frame_tokens(codes.cuda())
    torch.cuda.synchronize()
    assert toks.shape == (3, 16 * 257)
    for b in range(3):
        assert toks[b].cpu().tolist() == V.frame_tokens(codes[b].reshape(-1).tolist())
    t = toks.view(3, 16, 257)
    assert bool((t[:, :-1, 256] == EOF_TOKEN).all()) and bool((t[:, -1, 256] == EOV_TOKEN).all())
    assert torch.equal(unframe_tokens(toks).cpu(), codes)
    with pytest.raises(Exception):
        frame_tokens(torch.zeros(0, 16, 16, dtype=torch.int32, device="cuda"))
