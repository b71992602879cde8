"""lwm_vq_argmin at its edges, bit for bit against np.argmin over the oracle's float32 distances
(oracle/vqgan_ref.py::vector_quantize): row counts around the 128-row block, codebooks smaller than the 8 slices the
search is split into (so some slices are empty), duplicate codes in the first and last slice, and non-finite rows.

Non-finite semantics are np.argmin's: the first NaN distance wins (a NaN in z makes every distance NaN), and a row
whose distances are all +inf keeps its first code. |z| ~ 1e20 overflows sum z^2 to +inf, and inf - inf gives NaN
distances. The index is always a valid code, so the straight-through value z + (e[idx] - z) reads the codebook in
bounds."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def vr():
    from oracle import vqgan_ref
    return vqgan_ref


def _check(vr, z, emb):
    from lwm_b200.vqgan import Ops
    zq, idx = Ops("fp16x2").vq_argmin(z.cuda(), emb.cuda())
    torch.cuda.synchronize()
    with np.errstate(over="ignore", invalid="ignore"):
        ref_zq, ref_idx = vr.vector_quantize(z.numpy(), emb.numpy())
    got = idx.cpu().numpy()
    assert got.dtype == np.int32 and bool(((got >= 0) & (got < emb.shape[0])).all())
    assert np.array_equal(got, ref_idx), np.argwhere(got != ref_idx)[:8].ravel()
    assert np.array_equal(zq.cpu().numpy(), ref_zq, equal_nan=True)
    return got


@pytest.mark.parametrize("n_e", [1, 7, 8, 1000, 8192])
@pytest.mark.parametrize("N", [1, 127, 129, 4097])
def test_argmin_rows_and_codebook_sizes(vr, N, n_e):
    g = torch.Generator().manual_seed(N * 10007 + n_e)
    emb = torch.randn(n_e, 64, generator=g)
    z = torch.randn(N, 64, generator=g)
    if n_e >= 2:
        per = -(-n_e // 8)                      # codes per slice of the search
        last = n_e - 1                          # in the last non-empty slice
        first = min(per, n_e) - 1               # in the first slice
        emb[last] = emb[first]                  # an exact duplicate: the first index must win
        z[0] = emb[first]
        if N > 1:
            z[N - 1] = emb[last] * 1.0
    got = _check(vr, z, emb)
    if n_e >= 2:
        assert got[0] == first
        if N > 1:
            assert got[N - 1] == first


@pytest.mark.parametrize("n_e", [1, 7, 8, 1000, 8192])
def test_argmin_non_finite_rows(vr, n_e):
    g = torch.Generator().manual_seed(n_e)
    emb = torch.randn(n_e, 64, generator=g)
    z = torch.randn(300, 64, generator=g)
    z[0, 5] = float("nan")                      # every distance NaN: index 0
    z[1] = float("nan")
    z[2, 7] = float("inf")                      # +inf / NaN distances: the first NaN
    z[3, 0] = -float("inf")
    z[4] = float("inf")
    z[5] = -float("inf")
    z[6] = 1e20 * torch.sign(torch.randn(64, generator=g))   # sum z^2 overflows
    z[7] = -1e20
    z[8, :32] = 1e20
    z[128, 3] = float("nan")                     # the same in the second 128-row block
    z[129] = 1e20
    z[299] = float("inf")
    got = _check(vr, z, emb)
    assert got[0] == 0 and got[1] == 0
