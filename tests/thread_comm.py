"""In-process stand-in for the collectives of the q-sharded `ringattention_inference` protocol: `world` threads,
one per emulated rank, exchange tensors through a shared table (the interface of lwm_b200.ringattention.TorchComm)."""
import threading

import torch


class ThreadRing:
    def __init__(self, world):
        self.world = world
        self.barrier = threading.Barrier(world)
        self.slots = [None] * world

    def comm(self, rank):
        return ThreadComm(self, rank)


class ThreadComm:
    def __init__(self, ring, rank):
        self.ring, self.rank, self.world = ring, rank, ring.world

    def _exchange(self, x):
        self.ring.slots[self.rank] = x
        self.ring.barrier.wait()
        got = list(self.ring.slots)
        self.ring.barrier.wait()
        return got

    def all_gather(self, x):
        return torch.stack([t.clone() for t in self._exchange(x.contiguous())])

    def all_to_all(self, x):
        got = self._exchange(x.contiguous())
        return torch.stack([t[self.rank].clone() for t in got])


def run_ranks(world, fn):
    """fn(rank, comm) on `world` threads; returns the per-rank results (re-raises the first failure)"""
    ring = ThreadRing(world)
    res, err = [None] * world, []

    def body(r):
        try:
            res[r] = fn(r, ring.comm(r))
        except BaseException as e:      # noqa: BLE001 - surfaced below
            err.append(e)
            ring.barrier.abort()

    ts = [threading.Thread(target=body, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if err:
        raise err[0]
    return res
