"""CPU tests of the `ringattention_inference` backward: the numpy model of its tile map against a brute-force per-element
classification, the float64 VJP against finite differences, the no-cache mask helper, and the argument validation of
the new entry points (rejected with a message before the device check; LWM_ERR_DEVICE without a GPU)."""
import ctypes

import numpy as np
import pytest
import torch

from helpers import FOLDED_ENTRY_POINTS, with_options
from infer_grad_model import attention_inference_vjp, bwd_tilemap_brute, bwd_tilemap_model, pack_bits


def _mask(kind, B, Q, Sk, seed):
    rng = np.random.default_rng(seed)
    if kind == "none":
        return None
    if kind == "all_false":
        return np.zeros((B, Q, Sk), dtype=bool)
    if kind == "all_true":
        return np.ones((B, Q, Sk), dtype=bool)
    if kind == "causal_pad":      # decode-style causal rows over a cache, left padding, fully masked rows
        m = np.arange(Sk)[None, :] <= np.arange(Q)[:, None] + (Sk - Q)
        m = np.repeat(m[None], B, 0)
        m[0, :, :37] = False
        m[:, min(5, Q - 1)] = False
        return m
    if kind == "blocks":          # whole-false / whole-true 64x128 pairs, random elsewhere
        t = rng.integers(0, 3, (B, (Q + 63) // 64, (Sk + 127) // 128))
        t = t.repeat(64, 1).repeat(128, 2)[:, :Q, :Sk]
        rnd = rng.random((B, Q, Sk)) < 0.3
        return np.where(t == 0, False, np.where(t == 1, True, rnd))
    if kind == "broadcast":       # one mask for the whole batch
        m = np.arange(Sk)[None, :] <= np.arange(Q)[:, None] + (Sk - Q) // 2
        return np.broadcast_to(m[None], (B, Q, Sk)).copy()
    raise ValueError(kind)


@pytest.mark.parametrize("Q,Sk", [(1, 1), (7, 300), (64, 128), (65, 129), (200, 333), (130, 256)])
@pytest.mark.parametrize("kind", ["none", "all_false", "all_true", "causal_pad", "blocks", "broadcast"])
def test_backward_map_model_matches_brute_force(Q, Sk, kind):
    B = 2
    vis = _mask(kind, B, Q, Sk, Q * 31 + Sk)
    bits = None if vis is None else pack_bits(vis, Sk)
    row_any = None if vis is None else vis.any(-1).astype(np.int32)
    assert bwd_tilemap_model(bits, row_any, B, Q, Sk) == bwd_tilemap_brute(vis, B, Q, Sk)


def test_backward_map_counts_only_live_rows():
    """a fully masked row neither forces a visit nor stops a tile from being clean"""
    Q, Sk = 64, 256
    vis = np.ones((1, Q, Sk), dtype=bool)
    vis[0, :, 128:] = False
    vis[0, 3] = False
    maps = bwd_tilemap_model(pack_bits(vis, Sk), vis.any(-1).astype(np.int32), 1, Q, Sk)
    assert maps == [[[0], []]]
    # without row_any every row < Q is live: the dead row makes the tile mixed, still correct
    assert bwd_tilemap_model(pack_bits(vis, Sk), None, 1, Q, Sk) == [[[1], []]]


@pytest.mark.parametrize("kind", ["causal_pad", "blocks", "none"])
def test_float64_vjp_matches_finite_differences(kind):
    from oracle.attn_dense import attention_inference_dense
    B, Q, K, H, D = 2, 9, 13, 2, 4
    rng = np.random.default_rng(3)
    q, k, v, g = (rng.standard_normal((B, n, H, D)) for n in (Q, K, K, Q))
    vis = _mask(kind, B, Q, K, 1)
    if vis is not None:
        vis[:, 2] = True
        vis[:, 4, :] = False
        vis[:, 4, 3] = True
        # a fully masked row's output is the uniform average of V, which the contract leaves out of the gradients:
        # finite differences see it only through dout, so its dout is zero here (the GPU tests cover nonzero ones)
        g[~vis.any(-1)] = 0.0
    mask = None if vis is None else vis[:, None]
    dq, dk, dv = attention_inference_vjp(q, k, v, mask, g)
    eps = 1e-6
    for x, dx in ((q, dq), (k, dk), (v, dv)):
        for idx in [(0, 1, 0, 2), (1, 4, 1, 3), (1, 0, 0, 0)]:
            x0 = x[idx]
            x[idx] = x0 + eps
            fp = (attention_inference_dense(q, k, v, mask) * g).sum()
            x[idx] = x0 - eps
            fm = (attention_inference_dense(q, k, v, mask) * g).sum()
            x[idx] = x0
            assert abs((fp - fm) / (2 * eps) - dx[idx]) < 1e-6, (idx, (fp - fm) / (2 * eps), dx[idx])


def test_fully_masked_rows_contribute_nothing_to_the_vjp():
    B, Q, K, H, D = 1, 5, 7, 1, 4
    rng = np.random.default_rng(0)
    q, k, v, g = (rng.standard_normal((B, n, H, D)) for n in (Q, K, K, Q))
    vis = np.ones((B, 1, Q, K), dtype=bool)
    vis[..., 1, :] = False
    dq, dk, dv = attention_inference_vjp(q, k, v, vis, g)
    assert not dq[:, 1].any()
    keep = [0, 2, 3, 4]
    dq2, dk2, dv2 = attention_inference_vjp(q[:, keep], k, v, vis[:, :, keep], g[:, keep])
    np.testing.assert_allclose(dk, dk2, rtol=0, atol=1e-14)
    np.testing.assert_allclose(dv, dv2, rtol=0, atol=1e-14)


def test_causal_attention_mask_is_the_no_cache_branch():
    from lwm_b200.ringattention import causal_attention_mask
    pad = torch.tensor([[0, 0, 1, 1, 1, 1], [1, 1, 1, 1, 1, 0]])
    seg = torch.tensor([[0, 0, 1, 1, 2, 2], [1, 1, 1, 2, 2, 2]])
    m = causal_attention_mask(pad, seg)
    assert m.shape == (2, 1, 6, 6) and m.dtype == torch.bool
    for b in range(2):
        for i in range(6):
            for j in range(6):
                assert bool(m[b, 0, i, j]) == (j <= i and pad[b, j] > 0 and seg[b, i] == seg[b, j])
    assert torch.equal(causal_attention_mask(pad, None, 4), (torch.ones(4, 4).tril() > 0)[None, None] & (pad[:, None, None, :4] > 0))


P = ctypes.c_void_p(0x1000)
N = None
SHAPE, ARG, DEVICE = 2, 3, 1


def _status(lib, name, *args):
    from lwm_b200 import _lib
    _lib.load()
    return getattr(lib, name)(*args), lib.lwm_last_error().decode()


def _bwd_args(**kw):
    ptrs = dict(q=P, k=P, v=P, do=P, sq=P, sk=P, sv=P, sdo=P, lse=P, delta=P, bits=N, tiles=P, counts=P, dq=P, dk=P,
                dv=P)
    ptrs.update({k: v for k, v in kw.items() if k in ptrs})
    dims = dict(B=1, H=2, Q=200, Sk=300, D=128)
    dims.update({k: v for k, v in kw.items() if k in dims})
    return tuple(ptrs.values()) + tuple(dims.values()) + (0.1, N, N)     # softmax_scale, order_ws, stream


BAD_CALLS = [
    ("lwm_attn_infer_bwd_tilemap", (P, P, 1, 4, 64, N, P, N), ARG, "null"),
    ("lwm_attn_infer_bwd_tilemap", (P, P, 1, 4, 64, P, N, N), ARG, "null"),
    ("lwm_attn_infer_bwd_tilemap", (P, P, 1, 0, 64, P, P, N), SHAPE, "bad shape"),
    ("lwm_attn_infer_bwd_tilemap", (P, P, 1, 4, 0, P, P, N), SHAPE, "bad shape"),
    ("lwm_attn_infer_bwd_tilemap", (P, P, 70000, 4, 64, P, P, N), SHAPE, "bad shape"),
    ("lwm_attn_infer_bwd", _bwd_args(D=64), SHAPE, "head_dim"),
    ("lwm_attn_infer_bwd", _bwd_args(q=N), ARG, "null"),
    ("lwm_attn_infer_bwd", _bwd_args(sdo=N), ARG, "null"),
    ("lwm_attn_infer_bwd", _bwd_args(tiles=N), ARG, "null"),
    ("lwm_attn_infer_bwd", _bwd_args(dv=N), ARG, "null"),
    ("lwm_attn_infer_bwd", _bwd_args(Q=0), SHAPE, "bad shape"),
    ("lwm_attn_infer_bwd", _bwd_args(Sk=0), SHAPE, "bad shape"),
    ("lwm_attn_infer_bwd", _bwd_args(H=70000), SHAPE, "bad shape"),
    ("lwm_attn_infer_bwd", _bwd_args(B=60000, Q=2 ** 30, Sk=2 ** 20), SHAPE, "int32"),
]

# the same rows with the options of the folded entry points turned on: no option slot bypasses these checks
BAD_CALLS += [(n, with_options(n, a, P), c, f) for n, a, c, f in BAD_CALLS if n in FOLDED_ENTRY_POINTS]


@pytest.mark.parametrize("name,args,code,frag", BAD_CALLS, ids=["%s-%d" % (c[0][4:], i) for i, c in enumerate(BAD_CALLS)])
def test_bad_arguments_are_rejected_with_a_message(lib, name, args, code, frag):
    status, msg = _status(lib, name, *args)
    assert status == code, (status, msg)
    assert frag in msg, msg


GOOD_CALLS = [
    ("lwm_attn_infer_bwd_tilemap", (N, N, 2, 200, 300, P, P, N)),
    ("lwm_attn_infer_bwd_tilemap", (P, P, 1, 1, 1, P, P, N)),
    ("lwm_attn_infer_bwd", _bwd_args()),
    ("lwm_attn_infer_bwd", _bwd_args(bits=P, Q=1, Sk=1)),
]

GOOD_CALLS += [(n, with_options(n, a, P)) for n, a in GOOD_CALLS if n in FOLDED_ENTRY_POINTS]


@pytest.mark.skipif(torch.cuda.is_available(), reason="fake pointers: only meaningful where the device check fails")
@pytest.mark.parametrize("name,args", GOOD_CALLS, ids=["%s-%d" % (c[0][4:], i) for i, c in enumerate(GOOD_CALLS)])
def test_well_formed_calls_fail_with_device_error_without_gpu(lib, name, args):
    status, msg = _status(lib, name, *args)
    assert status == DEVICE, (status, msg)
    assert "no CPU fallback" in msg or "sm_90" in msg, msg


def test_backward_of_replicated_decode_row_is_not_implemented():
    """Q = 1 replicated along a ring of more than one rank stays forward-only: its backward says so"""
    from lwm_b200 import ringattention as ra

    class Ctx:
        replicated, small_ring = True, False
    with pytest.raises(NotImplementedError, match="replicated"):
        ra._InferAttnFn.backward(Ctx(), torch.zeros(1, 1, 1, 128))
    Ctx.replicated, Ctx.small_ring = False, True
    with pytest.raises(NotImplementedError, match="INFER_MIN_Q"):
        ra._InferAttnFn.backward(Ctx(), torch.zeros(1, 2, 1, 128))
