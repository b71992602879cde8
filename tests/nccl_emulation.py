"""Thread emulation of the two-sided transport of lwm_b200/ring_exec.py, so that the NCCL executor runs with the REAL
CUDA step functions (ringattention.CudaOps / CudaOpsF16) with P ranks as threads on one GPU
(tests/test_ring_nccl_emulated_gpu.py). All of the executor's communication goes through `ring_exec._Comm`; a test
installs EmuComm in its place (monkeypatch.setattr(rx, "_Comm", EmuComm)) and passes each rank thread its handle
EmuGroup(emu, rank) as the executor's `group`.

EmuP2P(world) holds one FIFO mailbox per (src, dst, channel) and a log of every message. `exchange` clones each send
tensor at post time and deposits the clone; `wait` pops the messages of the token's receives in posting order, asserts
that shape and dtype match exactly, and copies them into the receive buffers. NCCL matches the sends and receives of
one (src, dst) pair of one communicator in posting order, and this is the order the mailboxes keep.

Ordering (the argument of tests/peer_emulation.py): every rank thread enqueues ALL its device work on the one default
stream of the device, so the host order of the enqueues is their device order. A clone is enqueued before it is
deposited, and the copy out of it is enqueued only after the receiver has popped it, so the copy runs after the clone
on the device. There is no device-side wait anywhere: a protocol mistake ends as a host timeout and a failed assertion
naming the rank, peer and channel, never as a stalled GPU. EmuComm.cuda is False, so run_backward records no event.

This orders work more strictly than the real transport, whose transfers run on side streams of their own: the
emulation tests matching, ordering and numerics, not overlap races between the streams. TEST INFRASTRUCTURE ONLY."""
import collections
import threading

import torch

TIMEOUT_S = 120

Msg = collections.namedtuple("Msg", "src dst channel shape dtype nbytes tag")


class EmuP2P:
    def __init__(self, world):
        self.world = world
        self.boxes = collections.defaultdict(collections.deque)     # (src, dst, channel) -> deque of tensors
        self.cv = threading.Condition()
        self.log = []            # Msg of every deposit, in posting order per sender
        self.received = []       # (src, dst, channel, tag) of every pop
        self.barrier = threading.Barrier(world, timeout=TIMEOUT_S)
        self.failed = False      # set when a rank thread fails: the others stop waiting for its messages

    def pending(self):
        """{(src, dst, channel): count} of the messages deposited and not yet received"""
        with self.cv:
            return {key: len(q) for key, q in self.boxes.items() if q}

    def end_pass(self, rank):
        """every rank calls this after a pass: once all ranks are here, every mailbox must be empty"""
        self.barrier.wait()
        left = self.pending()
        self.barrier.wait()
        assert not left, "rank %d: messages left unmatched after the pass: %s" % (rank, left)


class EmuGroup:
    """one rank's handle on the emulated world: what the executor receives as its `group`. `tag` labels the messages
    this rank sends (the test sets it per pass, so the log can be split by pass)."""

    def __init__(self, emu, rank):
        self.emu, self.rank = emu, rank
        self.tag = None


class EmuComm:
    """ring_exec._Comm over EmuP2P mailboxes"""

    def __init__(self, group, device, channel=0):
        assert isinstance(group, EmuGroup), "EmuComm needs the rank's EmuGroup as the executor's group"
        self.group, self.device, self.channel = group, device, channel
        self.emu, self.rank = group.emu, group.rank
        self.cuda = False
        self.stream = None

    def exchange(self, sends, recvs, after_event=None):
        if not sends and not recvs:
            return None
        assert after_event is None
        for t, peer in sends:
            assert 0 <= peer < self.emu.world and peer != self.rank, (self.rank, peer)
            c = t.clone()            # on the current (default) stream, before the deposit
            with self.emu.cv:
                self.emu.boxes[(self.rank, peer, self.channel)].append(c)
                self.emu.log.append(Msg(self.rank, peer, self.channel, tuple(t.shape), t.dtype,
                                        t.numel() * t.element_size(), self.group.tag))
                self.emu.cv.notify_all()
        return list(recvs)

    def wait(self, token):
        if token is None:
            return
        for buf, peer in token:
            key = (peer, self.rank, self.channel)
            with self.emu.cv:
                ok = self.emu.cv.wait_for(lambda: self.emu.boxes[key] or self.emu.failed, timeout=TIMEOUT_S)
                assert not self.emu.failed, "rank %d: another rank failed" % self.rank
                assert ok, "rank %d: no message from peer %d on channel %d within %d s" % (
                    self.rank, peer, self.channel, TIMEOUT_S)
                msg = self.emu.boxes[key].popleft()
                self.emu.received.append((peer, self.rank, self.channel, self.group.tag))
            assert msg.shape == buf.shape and msg.dtype == buf.dtype, (
                "rank %d: message from peer %d on channel %d is %s %s, the receive buffer %s %s" % (
                    self.rank, peer, self.channel, tuple(msg.shape), msg.dtype, tuple(buf.shape), buf.dtype))
            buf.copy_(msg)


def run_threads(world, emu, fn, timeout=900):
    """fn(rank) on `world` threads; returns {rank: result}. A failing rank aborts the barrier, so the others stop at
    their next one; the first failure is re-raised with its traceback."""
    results, fails = {}, []

    def body(rank):
        try:
            results[rank] = fn(rank)
        except BaseException:   # noqa: BLE001  (reported by the main thread)
            import traceback
            fails.append((rank, traceback.format_exc()))
            with emu.cv:
                emu.failed = True
                emu.cv.notify_all()
            emu.barrier.abort()

    ts = [threading.Thread(target=body, args=(r,)) for r in range(world)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=timeout)
    torch.cuda.synchronize()
    assert not any(t.is_alive() for t in ts), "rank threads did not finish"
    assert not fails, "rank %d failed:\n%s" % fails[0]
    return results
