"""CPU emulation of the peer-memory transport and of the step functions, so that lwm_b200/ring_peer.py — the very
executor that runs on the GPUs — is exercised in the CPU test-suite: P rank THREADS of one process share P uint8
"heaps" and a flag table; pulls / puts are tensor copies, remote flag writes take effect immediately, waits block on a
condition variable. Streams do not exist here (every operation completes before the next one is issued), which is a
stricter ordering than the GPU's, so a protocol that deadlocks here may still be correct — but one that passes here has
no circular cross-rank wait. Numerics come from the oracle-backed step functions (oracle/step_ops.py).

EmuWorld(world, device=cuda_device) puts the heaps on one GPU instead, so that the executor can run with the real CUDA
step functions (ringattention.PeerOpsF16 / PeerOpsBf16; tests/test_ring_peer_emulated_gpu.py). Pulls and puts are then
device-to-device copies, while the flags stay on the host. This is sound because every rank thread issues ALL of its
device work — staging, copies, kernels — on the one default stream of that device: the host order of the enqueues is
their device order. A rank signals a flag only after it has enqueued the work the flag announces, and the consumer
enqueues its dependent copies or kernels only after it has seen the flag on the host, so they run after the producer's
work on the device. There is no device-side wait anywhere in the emulation: a protocol mistake ends as a host timeout
and a failed assertion, never as a stalled GPU.
TEST INFRASTRUCTURE ONLY."""
import contextlib
import threading

import torch

from oracle.step_ops import CpuOps


class EmuWorld:
    def __init__(self, world, n_flags=4096, device=None):
        self.world = world
        self.device = torch.device("cpu") if device is None else torch.device(device)
        self.heaps = [torch.zeros(0, dtype=torch.uint8, device=self.device) for _ in range(world)]
        self.flags = [[0] * n_flags for _ in range(world)]
        self.cv = threading.Condition()
        self.barrier = threading.Barrier(world)


class EmuTransport:
    def __init__(self, emu, rank):
        self.emu, self.rank, self.world = emu, rank, emu.world
        self.pass_id = 0
        self.log = []

    def ensure(self, nbytes):
        if self.emu.heaps[self.rank].numel() < nbytes:
            self.emu.barrier.wait()
            self.emu.heaps[self.rank] = torch.zeros(nbytes + 256, dtype=torch.uint8, device=self.emu.device)
            self.pass_id = 0
            self.emu.barrier.wait()

    def next_pass(self):
        self.pass_id += 1
        return self.pass_id

    def _view(self, peer, off, shape, dtype):
        n = 1
        for s in shape:
            n *= s
        nb = n * torch.empty((), dtype=dtype).element_size()
        return self.emu.heaps[peer][off:off + nb].view(dtype).view(*shape)

    def heap_view(self, off, shape, dtype):
        return self._view(self.rank, off, shape, dtype)

    def pull(self, dst, peer, off, stream):
        assert dst.is_contiguous() and peer != self.rank
        dst.copy_(self._view(peer, off, tuple(dst.shape), dst.dtype))
        self.log.append(("pull", peer, dst.numel() * dst.element_size()))

    def put(self, src, peer, off, stream):
        assert src.is_contiguous() and peer != self.rank
        self._view(peer, off, tuple(src.shape), src.dtype).copy_(src)
        self.log.append(("put", peer, src.numel() * src.element_size()))

    def signal(self, peer, flag, value, stream):
        with self.emu.cv:
            self.emu.flags[peer][flag] = value
            self.emu.cv.notify_all()

    def wait(self, flag, value, stream):
        with self.emu.cv:
            ok = self.emu.cv.wait_for(lambda: self.emu.flags[self.rank][flag] >= value, timeout=120)
        assert ok, "rank %d: flag %d never reached %d" % (self.rank, flag, value)

    def record(self, stream):
        return None

    def wait_event(self, stream, event):
        pass

    def on(self, stream):
        return contextlib.nullcontext()


class EmuOps:
    """Step functions with the signatures ring_peer.py expects. scaled=True emulates the fp16 operand mode's
    bookkeeping (per-tensor power-of-two scales shared by all ranks; operands stored divided by the scale) in float32."""
    op_dtype, op_itemsize = torch.float32, 4

    def __init__(self, scaled):
        self.scaled = scaled

    def absmax(self, x, bits):
        m = x.detach().abs().max().to(torch.float32).reshape(1)
        bits.copy_(torch.maximum(bits, m.view(torch.int32)))

    def make_scale(self, table, col):
        m = table[:, col].max().reshape(1).view(torch.float32)
        if float(m) == 0.0:
            return torch.ones(1)
        e = torch.floor(torch.log2(m))
        return torch.pow(torch.tensor(2.0), e - 12).reshape(1)

    def scale_of(self, x, out):
        m = float(x.detach().abs().max())
        out.fill_(1.0 if m == 0.0 else 2.0 ** (int(torch.floor(torch.log2(torch.tensor(m)))) - 12))

    def stage(self, x, dst, scale):
        dst.copy_(x.to(torch.float32) / (scale if scale is not None else 1.0))

    def fwd_step(self, q, k, v, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last, scales, out_f32):
        sq, sk, sv = [1.0 if s is None else s for s in scales]
        CpuOps.fwd_step(q * sq, k * sk, v * sv, out, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last)
        if last and out_f32 is not None:
            # the emulated kernel's bf16 `out` is what CpuOps wrote; recompute the un-rounded value for the fp32 readout
            tmp = torch.empty(out.shape, dtype=torch.float64)
            CpuOps.fwd_step(q * sq, k * sk, v * sv, tmp, lse, acc_o, acc_m, acc_l, q_pos0, k_pos0, causal, bias, seg, first, last)
            out_f32.copy_(tmp)

    def bwd_prep(self, out, dout, sdo, delta):
        CpuOps.bwd_prep(out, dout * (1.0 if sdo is None else sdo), delta)

    def lse_for_bwd(self, lse):
        return lse

    def bwd_step(self, q, k, v, dout, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg, scales, init):
        sq, sk, sv, sdo = [1.0 if s is None else s for s in scales]
        if init:
            dk_acc.zero_()
            dv_acc.zero_()
        CpuOps.bwd_step(q * sq, k * sk, v * sv, dout * sdo, lse, delta, dq_acc, dk_acc, dv_acc, q_pos0, k_pos0, causal, bias, seg)

    def reduce_cast(self, srcs, dst):
        acc = srcs[0].double().clone()
        for s in srcs[1:]:
            acc += s.double()
        dst.copy_(acc.to(dst.dtype))

    def cast(self, src, dst):
        dst.copy_(src.to(dst.dtype))
