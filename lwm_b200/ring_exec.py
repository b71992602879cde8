"""Executor of a ring Plan (ring_schedule.py): posts the NCCL transfers of step idx+1 on a side
stream while the tile kernels of step idx run, and sequences the per-(q chunk, kv block)
kernel launches with their first/last carry flags.

The step functions are injected (`ops`), so the very same sequencing code is exercised on CPU
with the gloo backend and an oracle-backed `ops` in tests/test_ring_gloo.py, and on H100s with
the CUDA C-ABI calls of lwm_b200.ringattention.

The rotary embedding of `ringattention(..., freqs_cis=, position_ids=)` is not folded into this executor's staging:
on this path the op runs the composition, `apply_rotary_emb` on q and k and then this executor on the rotated tensors,
which is bit-identical to the fused passes of the one-GPU and peer-memory paths by construction.
"""
import os
from typing import List

import torch
import torch.distributed as dist


_HP_GROUPS = {}
_TRACE = None     # debug: list of (label, start_event, end_event, stream_name) when LWM_RING_TRACE=1


def trace_begin():
    global _TRACE
    _TRACE = []


def trace_end(t0_event):
    """-> list of (label, stream, start_ms, end_ms) relative to t0_event; synchronises the device."""
    global _TRACE
    torch.cuda.synchronize()
    out = [(lab, st, t0_event.elapsed_time(a), t0_event.elapsed_time(b)) for (lab, a, b, st) in _TRACE]
    _TRACE = None
    return out


class _Span:
    def __init__(self, label, stream_name):
        self.label, self.stream_name = label, stream_name

    def __enter__(self):
        if _TRACE is not None:
            self.a = torch.cuda.Event(enable_timing=True)
            self.a.record()
        return self

    def __exit__(self, *exc):
        if _TRACE is not None:
            b = torch.cuda.Event(enable_timing=True)
            b.record()
            _TRACE.append((self.label, self.a, b, self.stream_name))


def _high_priority_group(group, channel=0):
    """A clone of `group` whose NCCL kernels run on HIGH-PRIORITY streams (created once per (group, channel)).
    The attention tile kernels occupy every SM (1 CTA/SM, all of the register file and shared memory), and
    ProcessGroupNCCL's default streams have normal priority: its send/recv kernels then only get SMs when an
    attention grid drains, i.e. the K/V prefetch does not overlap at all (measured: 83 ms/step at 8 GPUs vs
    63 ms for the same per-rank work without communication). With priority the copy CTAs are placed as soon
    as any attention CTA retires (~0.2 ms).
    The clone is made with use_local_synchronization=True: only the MEMBERS of `group` take part, so an 'sp' axis that
    is a proper subgroup of WORLD (dp x sp meshes) can create its clone inside its first forward without the other
    subgroups calling new_group with the same arguments. $LWM_RING_HP_GROUP=0 keeps the caller's group."""
    key = (id(group) if group is not None else 0, channel)
    if key not in _HP_GROUPS:
        hp = group
        if os.environ.get("LWM_RING_HP_GROUP", "1") != "0" and dist.get_backend(group) == "nccl":
            opts = dist.ProcessGroupNCCL.Options(is_high_priority_stream=True)
            ranks = dist.get_process_group_ranks(group if group is not None else dist.group.WORLD)
            hp = dist.new_group(ranks=ranks, backend="nccl", pg_options=opts, use_local_synchronization=True)
        _HP_GROUPS[key] = hp
    return _HP_GROUPS[key]


class _Comm:
    """send/recv helper: batches P2P ops per step; on CUDA they run on a dedicated stream."""

    def __init__(self, group, device, channel=0):
        """channel: independent communicator + stream (0: K/V prefetch and Q/O permutations; 1: dK/dV partial
        returns) so that a group waiting for a late peer on one channel cannot block the other."""
        self.device = device
        self.cuda = device.type == "cuda"
        self.group = _high_priority_group(group, channel) if self.cuda else group
        self.stream = torch.cuda.Stream(device=device, priority=-1) if self.cuda else None

    def _peer(self, r):
        return r if self.group is None or self.group is dist.group.WORLD else dist.get_global_rank(self.group, r)

    def exchange(self, sends, recvs, after_event=None):
        """sends: [(tensor, peer)], recvs: [(tensor, peer)]. Returns a token to wait on."""
        if not sends and not recvs:
            return None
        ops = []
        # a deterministic global order (by peer) keeps gloo's blocking pairs matched
        for t, peer in recvs:
            ops.append(dist.P2POp(dist.irecv, t, self._peer(peer), self.group))
        for t, peer in sends:
            ops.append(dist.P2POp(dist.isend, t, self._peer(peer), self.group))
        if self.cuda:
            self.stream.wait_stream(torch.cuda.current_stream(self.device))
            if after_event is not None:
                self.stream.wait_event(after_event)
            with torch.cuda.stream(self.stream):
                nb = sum(t.numel() * t.element_size() for t, _ in recvs)
                with _Span("xfer %d MiB in, %d ops" % (nb >> 20, len(ops)), "comm"):
                    works = dist.batch_isend_irecv(ops)
                    for w in works:
                        w.wait()
                ev = self.stream.record_event()
            # keep the tensors alive until the stream is done with them
            return (ev, [t for t, _ in sends] + [t for t, _ in recvs])
        works = dist.batch_isend_irecv(ops)
        return (works, None)

    def wait(self, token):
        if token is None:
            return
        if self.cuda:
            torch.cuda.current_stream(self.device).wait_event(token[0])
        else:
            for w in token[0]:
                w.wait()


def _rows(t, start, length):
    return t[:, start:start + length].contiguous()


def _gather_q_like(plan, comm, x):
    """Build this rank's compute chunks of a [B,S_loc,H,D] tensor laid out contiguously over ranks
    (entry permutation of the zigzag layout; identity for the contiguous layout)."""
    sends = [(_rows(x, s, l), peer) for (s, l, peer) in plan.q_sends]
    chunks, recvs = [], []
    for qc in plan.q_chunks:
        if qc.owner == plan.rank:
            chunks.append(_rows(x, qc.start, qc.length))
        else:
            buf = torch.empty((x.shape[0], qc.length) + tuple(x.shape[2:]), dtype=x.dtype, device=x.device)
            chunks.append(buf)
            recvs.append((buf, qc.owner))
    comm.wait(comm.exchange(sends, recvs))
    return chunks


def _scatter_q_like(plan, comm, chunks, out):
    """Inverse of _gather_q_like: return computed chunks to the contiguous owners' `out`."""
    sends, recvs, stage = [], [], []
    for qc, c in zip(plan.q_chunks, chunks):
        if qc.owner == plan.rank:
            out[:, qc.start:qc.start + qc.length].copy_(c)
        else:
            sends.append((c.contiguous(), qc.owner))
    for (s, l, peer) in plan.q_sends:
        buf = torch.empty((out.shape[0], l) + tuple(out.shape[2:]), dtype=out.dtype, device=out.device)
        recvs.append((buf, peer))
        stage.append((s, l, buf))
    comm.wait(comm.exchange(sends, recvs))
    for s, l, buf in stage:
        out[:, s:s + l].copy_(buf)
    return out


def _post_step_kv(plan, comm, idx, k, v, after_event=None):
    """Post the K/V traffic of step idx: my rows other ranks need, and the blocks I need."""
    st = plan.steps[idx]
    sends = []
    for (s, l, peer) in st.sends:
        sends.append((_rows(k, s, l), peer))
        sends.append((_rows(v, s, l), peer))
    bufs, recvs = [], []
    for kv in st.kv:
        if kv.owner == plan.rank:
            bufs.append((_rows(k, kv.start, kv.length), _rows(v, kv.start, kv.length)))
        else:
            kb = torch.empty((k.shape[0], kv.length) + tuple(k.shape[2:]), dtype=k.dtype, device=k.device)
            vb = torch.empty_like(kb)
            bufs.append((kb, vb))
            recvs.append((kb, kv.owner))
            recvs.append((vb, kv.owner))
    token = comm.exchange(sends, recvs, after_event)
    return bufs, token


def _prefetch_depth(n_steps):
    """How many steps ahead the K/V exchange is posted. 1 (default, the measured configuration): step idx+1 is posted
    when step idx starts. $LWM_RING_PREFETCH=all (or an integer): K/V are immutable during a pass, so every exchange
    can be posted at the start of the pass — the transfers then no longer depend on each rank's host timing; costs the
    whole remote K/V resident at once. Not yet measured on hardware."""
    v = os.environ.get("LWM_RING_PREFETCH", "1")
    return n_steps if v == "all" else max(1, min(int(v), n_steps))


def run_forward(plan, q, k, v, bias, seg, causal, group, ops):
    """Returns (out [B,Sq,H,D] like q, residuals) with residuals = dict(q_chunks, out_chunks, lse_chunks)."""
    dev = q.device
    comm = _Comm(group, dev)
    B, Sq, H, D = q.shape
    q_chunks = _gather_q_like(plan, comm, q)
    n_q = len(q_chunks)
    out_chunks = [torch.empty_like(c) for c in q_chunks]
    lse_chunks = [torch.empty((B, H, c.shape[1]), dtype=torch.float32, device=dev) for c in q_chunks]
    acc = [None] * n_q
    # first / last visit of every q chunk over the whole schedule
    visits = [[] for _ in range(n_q)]
    for idx, st in enumerate(plan.steps):
        for (qi, ki) in st.pairs:
            visits[qi].append((idx, ki))
    for qi in range(n_q):
        if len(visits[qi]) > 1:
            c = q_chunks[qi]
            acc[qi] = (torch.empty(c.shape, dtype=torch.float32, device=dev),
                       torch.empty((B, H, c.shape[1]), dtype=torch.float32, device=dev),
                       torch.empty((B, H, c.shape[1]), dtype=torch.float32, device=dev))
    depth = _prefetch_depth(len(plan.steps))
    posted = [_post_step_kv(plan, comm, i, k, v) for i in range(depth)]
    for idx, st in enumerate(plan.steps):
        bufs, token = posted.pop(0)
        if idx + depth < len(plan.steps):
            posted.append(_post_step_kv(plan, comm, idx + depth, k, v))   # prefetch while this step computes
        comm.wait(token)
        for (qi, ki) in st.pairs:
            kb, vb = bufs[ki]
            first = visits[qi][0] == (idx, ki)
            last = visits[qi][-1] == (idx, ki)
            a = acc[qi] or (None, None, None)
            with _Span("fwd step %d pair(%d,%d)" % (idx, qi, ki), "main"):
                ops.fwd_step(q_chunks[qi], kb, vb, out_chunks[qi], lse_chunks[qi], a[0], a[1], a[2],
                             plan.q_chunks[qi].pos0, st.kv[ki].pos0, causal, bias, seg, first, last)
    out = torch.empty_like(q)
    _scatter_q_like(plan, comm, out_chunks, out)
    return out, dict(q_chunks=q_chunks, out_chunks=out_chunks, lse_chunks=lse_chunks)


def run_backward(plan, res, k, v, dout, bias, seg, causal, group, ops):
    """dq, dk, dv (contiguous shards, input dtype). `res` are the residuals of run_forward."""
    dev = k.device
    comm = _Comm(group, dev)
    comm_pr = _Comm(group, dev, channel=1)     # partial returns: own communicator + stream
    q_chunks, out_chunks, lse_chunks = res["q_chunks"], res["out_chunks"], res["lse_chunks"]
    B, Sk, H, D = k.shape
    do_chunks = _gather_q_like(plan, comm, dout)
    n_q = len(q_chunks)
    delta = [torch.empty_like(l) for l in lse_chunks]
    dq_acc = [torch.zeros(c.shape, dtype=torch.float32, device=dev) for c in q_chunks]
    for qi in range(n_q):
        ops.bwd_prep(out_chunks[qi], do_chunks[qi], delta[qi])
    lse_chunks = [ops.lse_for_bwd(l) for l in lse_chunks]   # pre-scaled once; the tile kernel is exp-bound
    dk_acc = torch.zeros(k.shape, dtype=torch.float32, device=dev)
    dv_acc = torch.zeros(v.shape, dtype=torch.float32, device=dev)

    pending = []   # (token, [(start, length, dk_buf, dv_buf)]) partials received from peers
    depth = _prefetch_depth(len(plan.steps))
    posted = [_post_step_kv(plan, comm, i, k, v) for i in range(depth)]
    for idx, st in enumerate(plan.steps):
        bufs, token = posted.pop(0)
        if idx + depth < len(plan.steps):
            posted.append(_post_step_kv(plan, comm, idx + depth, k, v))
        comm.wait(token)
        parts = []
        for ki, kv in enumerate(st.kv):
            if kv.owner == plan.rank:   # accumulate straight into my own dk/dv rows
                parts.append(None)
            else:
                shape = (B, kv.length, H, D)
                parts.append((torch.zeros(shape, dtype=torch.float32, device=dev),
                              torch.zeros(shape, dtype=torch.float32, device=dev)))
        own_views = {}
        for (qi, ki) in st.pairs:
            kv = st.kv[ki]
            kb, vb = bufs[ki]
            if parts[ki] is None:
                if ki not in own_views:
                    if kv.start == 0 and kv.length == Sk:
                        own_views[ki] = (dk_acc, dv_acc, False)
                    else:   # row slice of my accumulator: stage through a contiguous buffer
                        own_views[ki] = (_rows(dk_acc, kv.start, kv.length), _rows(dv_acc, kv.start, kv.length), True)
                dkb, dvb = own_views[ki][0], own_views[ki][1]
            else:
                dkb, dvb = parts[ki]
            with _Span("bwd step %d pair(%d,%d)" % (idx, qi, ki), "main"):
                ops.bwd_step(q_chunks[qi], kb, vb, do_chunks[qi], lse_chunks[qi], delta[qi], dq_acc[qi], dkb, dvb,
                             plan.q_chunks[qi].pos0, kv.pos0, causal, bias, seg)
        for ki, (a, b2, staged) in own_views.items():
            if staged:
                kv = st.kv[ki]
                dk_acc[:, kv.start:kv.start + kv.length].copy_(a)
                dv_acc[:, kv.start:kv.start + kv.length].copy_(b2)
        # push the partials of remote blocks to their owners; receive the partials peers computed for
        # the rows they fetched from me at this step (the mirror image of st.sends)
        sends, recvs, incoming = [], [], []
        for ki, kv in enumerate(st.kv):
            if parts[ki] is not None:
                sends.append((parts[ki][0], kv.owner))
                sends.append((parts[ki][1], kv.owner))
        for (s, l, peer) in st.sends:
            dkb = torch.empty((B, l, H, D), dtype=torch.float32, device=dev)
            dvb = torch.empty_like(dkb)
            recvs.append((dkb, peer))
            recvs.append((dvb, peer))
            incoming.append((s, l, dkb, dvb))
        ev = torch.cuda.current_stream(dev).record_event() if comm.cuda else None
        pending.append((comm_pr.exchange(sends, recvs, ev), incoming))
        # fold in partials whose transfer was posted one step ago (overlapped with this step's kernels)
        while len(pending) > 1:
            tok, inc = pending.pop(0)
            comm_pr.wait(tok)
            for (s, l, dkb, dvb) in inc:
                ops.accumulate(dk_acc, s, l, dkb)
                ops.accumulate(dv_acc, s, l, dvb)
    for tok, inc in pending:
        comm_pr.wait(tok)
        for (s, l, dkb, dvb) in inc:
            ops.accumulate(dk_acc, s, l, dkb)
            ops.accumulate(dv_acc, s, l, dvb)

    dq_chunks = []
    for qi in range(n_q):
        c = torch.empty_like(q_chunks[qi])
        ops.cast(dq_acc[qi], c)
        dq_chunks.append(c)
    dq = torch.empty((B,) + tuple(dout.shape[1:]), dtype=q_chunks[0].dtype, device=dev)
    _scatter_q_like(plan, comm, dq_chunks, dq)
    dk = torch.empty_like(k)
    dv = torch.empty_like(v)
    ops.cast(dk_acc, dk)
    ops.cast(dv_acc, dv)
    return dq, dk, dv
