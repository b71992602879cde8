"""numpy restatement of the attention-dropout mask (lwm_b200/csrc/attn_dropout.cuh), bit for bit, and the float64
references the dropout tests compare against: dense attention over the surviving pairs, and CPU stand-ins of the
ring step functions (oracle/step_ops.py) that take the same `dropout=(seed, thr)` keyword as the CUDA ones.

The mask: Philox4x32-10 keyed by (seed & 0xffffffff, seed >> 32), counter (((k >> 4) << 2) | ((k >> 1) & 3), q & ~8,
h, b) over GLOBAL query / key positions and the global batch row b; entry (q, k) is the 16-bit half k & 1 of word
2 ((q >> 3) & 1) + ((k >> 3) & 1), dropped iff it is below thr = min(65535, round(p * 65536))."""
import math

import numpy as np
import torch

from oracle.attn_dense import attention_visible, visible_pairs
from oracle.step_ops import CpuOps, LOG2E, MASKED, _logits2

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: 4 uint32 arrays (broadcastable), key: 2 uint32 scalars -> 4 uint32 arrays"""
    c = [np.asarray(x, dtype=np.uint64) & _LO for x in ctr]
    c = np.broadcast_arrays(*c)
    c = [x.copy() for x in c]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for r in range(10):
        if r:
            k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
        p0, p1 = _M0 * c[0], _M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & _LO, (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1),
             p0 & _LO]
    return [x.astype(np.uint32) for x in c]


def seed_key(seed):
    s = int(seed) & (2 ** 64 - 1)
    return s & 0xFFFFFFFF, s >> 32


def threshold(p):
    return min(65535, int(round(float(p) * 65536)))


def drop_u16(seed, b, h, q_pos, k_pos):
    """the 16-bit draws of queries q_pos [n_q] x keys k_pos [n_k] (global positions) of batch row b, head h"""
    q = np.asarray(q_pos, dtype=np.uint64)[:, None]
    k = np.asarray(k_pos, dtype=np.uint64)[None, :]
    one, three = np.uint64(1), np.uint64(3)
    c0 = ((k >> np.uint64(4)) << np.uint64(2)) | ((k >> one) & three)
    w = np.stack(philox4x32_10((c0, q & ~np.uint64(8), np.uint64(h), np.uint64(b)), seed_key(seed)))  # [4, n_q, n_k]
    j = (np.uint64(2) * ((q >> three) & one) + ((k >> three) & one)).astype(np.int64)             # [n_q, n_k]
    wd = np.take_along_axis(w, j[None], axis=0)[0]
    return (wd >> (16 * (k & np.uint64(1))).astype(np.uint32)) & np.uint32(0xFFFF)


def drop_mask(seed, thr, B, H, q_pos0, Sq, k_pos0, Sk):
    """bool [B, H, Sq, Sk]: True = dropped"""
    return drop_mask_rows(seed, thr, 0, B, H, q_pos0, Sq, k_pos0, Sk)


def attention_dropout_ref(q, k, v, dout=None, drop=None, attn_bias=None, segment_ids=None, causal=True, q_pos0=0,
                          k_pos0=0):
    """float64 attention over the visible pairs that survive `drop` [B,H,Sq,Sk]; a row without a surviving pair
    outputs 0 and gets no gradient. -> (out, live [B,H,Sq]) or (out, dq, dk, dv, live)"""
    q, k, v = (np.asarray(t, dtype=np.float64) for t in (q, k, v))
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    vis = visible_pairs(B, Sq, Sk, q_pos0, k_pos0, attn_bias, segment_ids, causal)      # [B,1,Sq,Sk]
    keep = vis & ~drop if drop is not None else np.broadcast_to(vis, (B, H, Sq, Sk))
    live = keep.any(-1)                                                                 # [B,H,Sq]
    outs, grads = np.zeros(q.shape), [np.zeros(q.shape), np.zeros(k.shape), np.zeros(v.shape)]
    for h in range(H):
        sl = slice(h, h + 1)
        if dout is None:
            o, _ = attention_visible(q[:, :, sl], k[:, :, sl], v[:, :, sl], keep[:, h:h + 1])
        else:
            g = np.asarray(dout, dtype=np.float64)[:, :, sl] * live[:, h, :, None, None]
            o, _, dq, dk, dv = attention_visible(q[:, :, sl], k[:, :, sl], v[:, :, sl], keep[:, h:h + 1], g)
            for acc, x in zip(grads, (dq, dk, dv)):
                acc[:, :, sl] = x
        outs[:, :, sl] = o * live[:, h, :, None, None]
    if dout is None:
        return outs, live
    grads[0] *= live.transpose(0, 2, 1)[..., None]
    return (outs, *grads, live)


def drop_mask_rows(seed, thr, b0, B, H, q_pos0, Sq, k_pos0, Sk):
    """drop_mask of global batch rows b0 .. b0 + B - 1"""
    qp, kp = q_pos0 + np.arange(Sq), k_pos0 + np.arange(Sk)
    return np.stack([np.stack([drop_u16(seed, b0 + b, h, qp, kp) < thr for h in range(H)]) for b in range(B)])


def _drop_torch(dropout, B, H, q_pos0, Sq, k_pos0, Sk):
    """dropout: (seed, thr) or (seed, thr, batch0) as the CUDA step functions take it"""
    seed, thr, b0 = tuple(dropout) + (0,) * (3 - len(dropout))
    return torch.from_numpy(drop_mask_rows(seed, thr, b0, B, H, q_pos0, Sq, k_pos0, Sk))


class CpuDropoutOps(CpuOps):
    """oracle.step_ops.CpuOps with the CUDA step functions' `dropout=(seed, thr)` keyword: dropped entries take the
    masked logit, and on the last step a row whose max is still at the masked level outputs 0 with a masked-level lse
    (the tile kernels' epilogue)."""

    @staticmethod
    def fwd_step(q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last, dropout=None):
        B, Sq, H, _ = q.shape
        t = _logits2(q, k, q_pos0, k_pos0, causal, bias, seg)
        if dropout is not None:
            t = torch.where(_drop_torch(dropout, B, H, q_pos0, Sq, k_pos0, k.shape[1]), torch.full_like(t, MASKED), t)
        m_loc = t.max(dim=-1).values
        p = torch.exp2(t - m_loc[..., None])
        l_loc = p.sum(-1)
        o_loc = torch.einsum("bhqk,bkhd->bqhd", p, v.double())
        if first:
            m_new, l_new, o_new = m_loc, l_loc, o_loc
        else:
            m_c, l_c, o_c = acc_m.double(), acc_l.double(), acc_o.double()
            m_new = torch.maximum(m_c, m_loc)
            wa, wb = torch.exp2(m_c - m_new), torch.exp2(m_loc - m_new)
            l_new = wa * l_c + wb * l_loc
            o_new = o_c * wa.transpose(1, 2)[..., None] + o_loc * wb.transpose(1, 2)[..., None]
        if last:
            o = o_new / l_new.transpose(1, 2)[..., None]
            lse_v = (m_new + torch.log2(l_new)) / LOG2E
            if dropout is not None:
                dead = m_new <= MASKED
                o = torch.where(dead.transpose(1, 2)[..., None], torch.zeros_like(o), o)
                lse_v = torch.where(dead, torch.full_like(lse_v, MASKED / LOG2E), lse_v)
            out.copy_(o.to(out.dtype))
            lse.copy_(lse_v.to(lse.dtype))
        else:
            acc_o.copy_(o_new.to(acc_o.dtype))
            acc_m.copy_(m_new.to(acc_m.dtype))
            acc_l.copy_(l_new.to(acc_l.dtype))

    @staticmethod
    def bwd_step(q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg, dropout=None):
        B, Sq, H, D = q.shape
        t = _logits2(q, k, q_pos0, k_pos0, causal, bias, seg)
        if dropout is not None:
            t = torch.where(_drop_torch(dropout, B, H, q_pos0, Sq, k_pos0, k.shape[1]), torch.full_like(t, MASKED), t)
        dead = (lse.double() < -1.0e29)[..., None]
        p = torch.where(dead, torch.zeros_like(t), torch.exp2(t - lse.double()[..., None] * LOG2E))
        g = dout.double()
        dv_acc += torch.einsum("bhqk,bqhd->bkhd", p, g).to(dv_acc.dtype)
        dp = torch.einsum("bqhd,bkhd->bhqk", g, v.double())
        ds = p * (dp - delta.double()[..., None]) / math.sqrt(D)
        dq_acc += torch.einsum("bhqk,bkhd->bqhd", ds, k.double()).to(dq_acc.dtype)
        dk_acc += torch.einsum("bhqk,bqhd->bkhd", ds, q.double()).to(dk_acc.dtype)
