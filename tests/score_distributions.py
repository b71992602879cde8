"""Seeded attention inputs whose score distributions look like trained LLaMA heads rather than white noise.

With N(0,1) q and k the logits of D = 128 have a standard deviation of about 1, the softmax is close to uniform and
every probability stays far above where fp16 loses precision. Trained heads at long context often put most of a row's
mass on the first token (the attention sink), whose value vector is near zero, and spread the rest over thousands of
keys whose V has non-zero channel means. Then every p of the bulk is e^-gap or less against the row's max. Three kinds:

  sink(gap, sigma)  q: N(0,1) with channel 0 = 4. Bulk k: N(0, sigma^2) with channel 0 = 0. The key at global position
                    0: zero but channel 0 = gap * sqrt(128) / 4. So the sink's logit is `gap` (up to the bf16 rounding
                    of that channel, < 0.4 %) and the bulk's about N(0, sigma^2). v: a fixed per-channel mean of
                    +-0.5 plus N(0,1) for the bulk, 0.01 N(0,1) for the sink. dO: N(0,1).
  recency           (control) k channel 0 rises linearly with the key's global position, from 0 to 20 nats over the
                    sequence, on top of N(0,1) noise: the row max keeps rising, so the alpha rescale runs often,
                    and each p is taken against a running max close to its own tile's.
  peaked            (control) bulk sigma = 3 and no sink: a few keys per row dominate, none by a wide gap.

Every 128-position block of every (tensor, head) comes from its own generator stream, so a value depends only on its
global position and head, never on the sequence length or the sharding: a rank of an emulated ring can rebuild its own
shard and the float64 oracle any head of the whole sequence (the pattern of lwm_b200/synthetic.py). Values are float32
holding bf16-representable numbers."""
import math

import torch

D = 128
BLOCK = 128
TENSOR_IDS = {"q": 0, "k": 1, "v": 2, "do": 3}
RECENCY_NATS = 20.0
PEAKED_SIGMA = 3.0


def _bf16(x):
    return x.to(torch.bfloat16).float()


def _v_mean(seed):
    """the bulk's per-channel mean: +-0.5, fixed by the seed"""
    g = torch.Generator().manual_seed(seed + 7)
    return (torch.randint(0, 2, (D,), generator=g).float() - 0.5)


def _normal(seed, name, head, pos0, rows):
    """[rows, D] N(0,1) for global positions [pos0, pos0 + rows), pos0 a multiple of BLOCK"""
    assert pos0 % BLOCK == 0, pos0
    out = torch.empty(rows, D)
    for b0 in range(0, rows, BLOCK):
        blk = (pos0 + b0) // BLOCK
        g = torch.Generator().manual_seed(seed + 1000003 * TENSOR_IDS[name] + 10007 * head + 101 * blk)
        n = min(BLOCK, rows - b0)
        out[b0:b0 + n] = torch.randn(BLOCK, D, generator=g)[:n]
    return out


def head_rows(kind, name, head, pos0, rows, S, gap=16.0, sigma=1.0, seed=0):
    """[rows, D] of tensor `name` ('q', 'k', 'v', 'do') of one head at global positions [pos0, pos0 + rows) of a
    sequence of S tokens. kind: 'sink' (with gap, sigma), 'recency' or 'peaked'."""
    x = _normal(seed, name, head, pos0, rows)
    pos = torch.arange(pos0, pos0 + rows)
    if name == "q":
        x[:, 0] = 4.0
    elif name == "k":
        if kind == "sink":
            x *= sigma
            x[:, 0] = 0.0
            x[pos == 0] = 0.0
            x[pos == 0, 0] = gap * math.sqrt(D) / 4.0
        elif kind == "recency":
            x[:, 0] = (RECENCY_NATS * pos.float() / S) * math.sqrt(D) / 4.0
        elif kind == "peaked":
            x *= PEAKED_SIGMA
            x[:, 0] = 0.0
        else:
            raise ValueError(kind)
    elif name == "v":
        x += _v_mean(seed)
        if kind == "sink":
            x[pos == 0] = 0.01 * _normal(seed + 1, "v", head, 0, BLOCK)[0]
    return _bf16(x)


def shard(kind, name, pos0, rows, S, H, **kw):
    """[1, rows, H, D] float32: positions [pos0, pos0 + rows) of every head"""
    return torch.stack([head_rows(kind, name, h, pos0, rows, S, **kw) for h in range(H)], dim=1)[None]


def sink_logit(gap):
    """the sink's logit as the bf16 inputs give it (q channel 0 = 4, the rounded key channel)"""
    return 4.0 * float(_bf16(torch.tensor(gap * math.sqrt(D) / 4.0))) / math.sqrt(D)
