"""Peer-memory executor of the sequence-parallel attention op — the default multi-GPU path.

What the reference does with `lax.ppermute(k, v)` hop by hop (un-vendored `ringattention` package, entered at
lwm/llama.py:539-569; SURVEY.md Appendix A) is done here the NVSwitch way: every rank STAGES its K/V (and Q or dO) once
per pass in a heap all peers map (include/lwm_b200.h: lwm_ring_ctx_*), every rank PULLS the chunks it needs with
copy-engine transfers (no SMs, no matching call on the owner) into a position-ordered local copy of K/V, and runs the
tile kernels over whatever contiguous range has arrived. Results that belong to another rank — O / dQ chunks of the
zigzag work assignment, dK/dV partials — are PUT into landing slots of the owner's heap. All ordering is done with
32-bit flags in the heaps (remote flag write behind the payload on the same stream; cuStreamWaitValue32 on the local
flag): there is no host synchronisation and no two-sided rendezvous anywhere on the data path.

Protocol of one pass (forward or backward; `pid` = pass counter, identical on all ranks; `set` = pid & 1 selects one of
two copies of every heap region, so a rank may start pass n+1 while slower peers still read its pass-n data):
  1. (fp16 operand mode) every rank derives the power-of-two scales of ITS OWN shards and writes them next to the data
     (a launch only ever combines one Q-side owner with one K/V owner, so no cross-rank agreement is needed).
  2. stage K, V (own rows of the position-ordered K/V arrays) and Q (forward) / dO (backward); flag STAGED[rank] = pid
     on every peer.
  3. pull streams: wait STAGED[owner] once per owner and fetch its scale row, the Q/dO chunks first, then one copy per
     (K|V chunk), enqueued a couple of groups ahead of the compute loop; one event per group of chunks.
  4. main stream: per group, wait for its event, launch the tile kernels (carries merged in the kernels' epilogues).
  5. push stream (backward): after a remote chunk's launches, put its fp32 dK/dV partial into the owner's landing slot,
     flag PART[slot] = pid. Exit: put O / dQ chunks computed for other ranks, flag RES[rank] = pid.
  6. owner: wait PART[*] / RES[*], fold partials (one fused sum + cast pass), copy landed chunks into the outputs.
Heap reuse is safe without an end-of-pass barrier: a rank signals STAGED(pid) only after everything of its pass pid-1
has been enqueued before it on the same stream, every rank waits for all peers' STAGED(pid) during pass pid, and pass
pid+1 touches the other region set.

The transport (`tr`) and the step functions (`ops`) are injected: tests/peer_emulation.py runs this very file on CPU
with shared-memory heaps and oracle-backed step functions (tests/test_ring_peer_cpu.py).
"""
import ctypes
import os

import torch
import torch.distributed as dist

from . import _lib

FLAG_STAGED, FLAG_RES, FLAG_PART = 16, 32, 64
_ALIGN = 256


def _al(n):
    return (n + _ALIGN - 1) // _ALIGN * _ALIGN


class Layout:
    """Byte offsets inside every rank's heap payload — a pure function of the GLOBAL call shape, so a rank can address
    any region of any peer. Two sets (pass parity) of: |max| table, K array, V array (position-ordered, [B, P*Sk, H, D]),
    Q/dO stage [B, Sq, H, D], two landing areas for O/dQ rows computed elsewhere (4-byte and 2-byte elements) and the
    dK/dV partial landing slots (chunks_per_rank * world slots of one chunk, dK then dV, fp32)."""

    def __init__(self, B, Sq, Sk, H, D, world, chunks_per_rank, op_itemsize):
        row = H * D
        self.B, self.Sq, self.Sk, self.row, self.world, self.isz = B, Sq, Sk, row, world, op_itemsize
        self.chunk_rows = Sk // chunks_per_rank
        self.n_slots = chunks_per_rank * world
        off = 0
        self.abs = off; off += _al(world * 16)
        self.kg = off; off += _al(B * world * Sk * row * op_itemsize)
        self.vg = off; off += _al(B * world * Sk * row * op_itemsize)
        self.qs = off; off += _al(B * Sq * row * op_itemsize)
        self.lq4 = off; off += _al(B * Sq * row * 4)
        self.lq2 = off; off += _al(B * Sq * row * 2)
        self.slot_bytes = _al(B * self.chunk_rows * row * 4)
        self.lp = off; off += self.n_slots * 2 * self.slot_bytes
        self.set_bytes = off
        self.total = 2 * off

    def base(self, which):
        return which * self.set_bytes

    def kv_row_off(self, region, which, b, pos, itemsize=None):
        """byte offset of global key row `pos` of batch b in the K (region='kg') or V array; itemsize: of the array's
        elements when they are narrower than the operand itemsize the region is sized for (the fp8 mode's e4m3 K)"""
        isz = self.isz if itemsize is None else itemsize
        return self.base(which) + getattr(self, region) + (b * self.world * self.Sk + pos) * self.row * isz

    def q_row_off(self, region, which, b, row, itemsize):
        return self.base(which) + getattr(self, region) + (b * self.Sq + row) * self.row * itemsize

    def slot_off(self, which, slot, tensor):
        return self.base(which) + self.lp + (slot * 2 + tensor) * self.slot_bytes


# ------------------------------------------------------------------------------------------------
# CUDA transport over the C-ABI ring context
# ------------------------------------------------------------------------------------------------
class PeerTransportUnavailable(RuntimeError):
    """raised by every rank of the group together when the peer-memory heaps cannot be set up on this box"""


class _RawCuda:
    def __init__(self, addr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (addr, False), "version": 2}


class CudaPeerTransport:
    """One per (process group, device). Owns the lwm_ring_ctx, two side streams and the pass counter."""
    _instances = {}

    @classmethod
    def get(cls, group, device):
        key = (id(group) if group is not None else 0, device.index)
        if key not in cls._instances:
            cls._instances[key] = cls(group, device)
        return cls._instances[key]

    def __init__(self, group, device):
        self.group, self.device = group, device
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.ctx, self.capacity, self.pass_id = None, 0, 0
        self.heap_addr, self.own = [], None
        self.signal_mode = int(os.environ.get("LWM_RING_SIGNAL", "0"))
        # "pull" / "push" each fan out over several streams, so that independent transfers can ride different copy
        # engines; a batch that must stay ordered (payload then flag) takes ONE of them with pick()
        self.fan = max(1, int(os.environ.get("LWM_RING_COPY_STREAMS", "4")))
        self.side = {"%s#%d" % (n, i): torch.cuda.Stream(device=device) for n in ("pull", "push") for i in range(self.fan)}
        self._rr = {"pull": 0, "push": 0}

    def ensure(self, nbytes):
        """(Re)create the heap collectively when the call needs more than is mapped. Every rank sees the same sizes
        (the layout is a function of the global shape), so all of them take this branch together."""
        if self.ctx is not None and nbytes <= self.capacity:
            return
        torch.cuda.synchronize(self.device)
        if self.ctx is not None:
            dist.barrier(group=self.group)
            _lib.call("lwm_ring_ctx_destroy", self.ctx)
            self.ctx = None
        want = int(nbytes * 1.05) + (1 << 20)
        lib = _lib.load()
        # Bootstrap: every step that can fail on a box (heap allocation, IPC export / mapping of the peers) is tried by all
        # ranks, and the ranks AGREE on the outcome before anybody relies on it: if one rank cannot map its peers, all of
        # them raise PeerTransportUnavailable together (ringattention.py then switches the process group to the two-sided
        # NCCL executor, loudly) instead of one rank raising while the others wait for its flags forever.
        ctx, err = ctypes.c_void_p(), None
        handle = (ctypes.c_ubyte * 64)()
        try:
            _lib.call("lwm_ring_ctx_create", self.rank, self.world, want, self.signal_mode, ctypes.byref(ctx))
            _lib.call("lwm_ring_ctx_get_handle", ctx, handle)
        except _lib.LwmError as e:
            err = str(e)
        mine = torch.tensor(list(handle), dtype=torch.uint8, device=self.device)
        allh = torch.empty(self.world * 64, dtype=torch.uint8, device=self.device)
        dist.all_gather_into_tensor(allh, mine, group=self.group)
        if err is None:
            try:
                buf = (ctypes.c_ubyte * (self.world * 64))(*allh.cpu().tolist())
                _lib.call("lwm_ring_ctx_open_peers", ctx, buf)
            except _lib.LwmError as e:
                err = str(e)
        ok = torch.tensor([0 if err else 1], dtype=torch.int32, device=self.device)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=self.group)
        if int(ok.item()) == 0:
            if ctx.value:
                _lib.call("lwm_ring_ctx_destroy", ctx)
            raise PeerTransportUnavailable(err or "a peer rank could not set up its peer-memory heap")
        self.ctx, self.capacity, self.pass_id = ctx, want, 0
        self.heap_addr = [int(lib.lwm_ring_ctx_heap(ctx, p)) for p in range(self.world)]
        self.own = torch.as_tensor(_RawCuda(self.heap_addr[self.rank], want), device=self.device)
        dist.barrier(group=self.group)      # nobody signals into a heap that is not mapped yet

    def next_pass(self):
        self.pass_id += 1
        return self.pass_id

    def heap_view(self, off, shape, dtype):
        n = 1
        for s in shape:
            n *= s
        nb = n * torch.empty((), dtype=dtype).element_size()
        return self.own[off:off + nb].view(dtype).view(*shape)

    def pick(self, name):
        """one concrete stream of the fan-out `name` (round robin) for a batch that must stay ordered"""
        if name not in self._rr:
            return name
        self._rr[name] = (self._rr[name] + 1) % self.fan
        return "%s#%d" % (name, self._rr[name])

    def _members(self, name):
        return ["%s#%d" % (name, i) for i in range(self.fan)] if name in self._rr else [name]

    def _stream(self, name):
        if name == "main":
            return torch.cuda.current_stream(self.device)
        return self.side[name if "#" in name else name + "#0"]

    def _sp(self, name):
        return ctypes.c_void_p(self._stream(name).cuda_stream)

    def pull(self, dst, peer, off, stream):
        assert dst.is_contiguous()
        _lib.call("lwm_ring_copy", ctypes.c_void_p(dst.data_ptr()), ctypes.c_void_p(self.heap_addr[peer] + off),
                  dst.numel() * dst.element_size(), self._sp(stream))

    def put(self, src, peer, off, stream):
        assert src.is_contiguous()
        _lib.call("lwm_ring_copy", ctypes.c_void_p(self.heap_addr[peer] + off), ctypes.c_void_p(src.data_ptr()),
                  src.numel() * src.element_size(), self._sp(stream))

    def signal(self, peer, flag, value, stream):
        _lib.call("lwm_ring_signal", self.ctx, peer, flag, value, self._sp(stream))

    def wait(self, flag, value, stream):
        for m in self._members(stream):
            _lib.call("lwm_ring_wait", self.ctx, flag, value, self._sp(m))

    def record(self, stream):
        return [self._stream(m).record_event() for m in self._members(stream)]

    def wait_event(self, stream, event):
        for m in self._members(stream):
            for ev in event:
                self._stream(m).wait_event(ev)

    def on(self, stream):
        return torch.cuda.stream(self._stream(stream))

    # -- optional timeline (tools/ring_trace_peer.py): CUDA events around labelled pieces of a pass
    trace = None

    @staticmethod
    def span_times(t0, spans):
        """[(label, stream, start_ms, end_ms)] relative to event t0 (earliest start / latest end over a fan-out)"""
        return [(lab, st, min(t0.elapsed_time(e) for e in a), max(t0.elapsed_time(e) for e in b)) for (lab, st, a, b) in spans]

    def span(self, label, stream):
        return _Span(self, label, stream)


class _Span:
    def __init__(self, tr, label, stream):
        self.tr, self.label, self.stream = tr, label, stream

    def _events(self):
        evs = []
        for m in self.tr._members(self.stream):
            e = torch.cuda.Event(enable_timing=True)
            e.record(self.tr._stream(m))
            evs.append(e)
        return evs

    def __enter__(self):
        if self.tr.trace is not None:
            self.a = self._events()
        return self

    def __exit__(self, *exc):
        if self.tr.trace is not None:
            self.tr.trace.append((self.label, self.stream, self.a, self._events()))


class _NoSpan:
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        pass


def _pick(tr, name):
    f = getattr(tr, "pick", None)
    return f(name) if f is not None else name


def _pull_striped(tr, dst, peer, off):
    """Pull the rows of `dst` ([rows, ...], contiguous) from `peer`'s heap at byte offset `off`, striped over the members
    of the 'pull' fan-out: every member carries a slice of EVERY transfer, in issue order — transfers complete in the
    order they are needed at the aggregate bandwidth, with no cross-stream dependency between them."""
    f = getattr(tr, "_members", None)
    members = f("pull") if f is not None else ["pull"]
    rows = dst.shape[0]
    n = min(len(members), rows)
    row_bytes = dst[0].numel() * dst.element_size()
    for i in range(n):
        a, b = rows * i // n, rows * (i + 1) // n
        if b > a:
            tr.pull(dst[a:b], peer, off + a * row_bytes, members[i])


def _span(tr, label, stream):
    f = getattr(tr, "span", None)
    return f(label, stream) if f is not None else _NoSpan()


# ------------------------------------------------------------------------------------------------
# executor
# ------------------------------------------------------------------------------------------------
def v_ops(ops):
    """the ops that stage V: ops itself, except in the fp8 mode, whose V is the fp16 mode's copy (ops.v_ops)"""
    return getattr(ops, "v_ops", ops)


def _layout_for(plan, q_shape, Sk, ops):
    B, Sq, H, D = q_shape
    return Layout(B, Sq, Sk, H, D, plan.world, plan.chunks_per_rank, ops.op_itemsize)


def _stage_and_announce(tr, lay, which, pid, ops, k, v, x, cols, known=None, rope=None, rope_x=False, rope_k=True):
    """Scales of the local shards -> my row of the scale table (in the heap: peers pull it with the data); K/V -> own
    rows of the position-ordered arrays, x (Q or dO) -> the stage; then STAGED[rank] = pid on every peer.
    cols = (column of k, of v, of x) in the table row [sq, sk, sv, sdo]; known = {column: scale tensor} to reuse (the
    backward re-stages K/V with the forward's scales). Every operand has its OWNER's scale: no cross-rank agreement and
    therefore no exchange is needed — a launch only ever combines one Q-side owner with one K/V owner.
    k, v may be the 8-bit cache (kv_cache.QuantizedKV, the forward only): ops stage it from its codes, batch row by batch
    row, into the same heap regions and with the same bytes as its dequantized values would give.
    rope: None, or (positions int32 [B,Sk], inv_freq): k (unless not rope_k) and x (when rope_x) are un-rotated, and their
    scales and staged copies are those of the rotated rows. Every rank stages its own rows, so only local positions are
    needed (rope_k=False: x's positions [B,Sq])."""
    P, r = tr.world, tr.rank
    B, Sk = k.shape[0], k.shape[1]
    vops = v_ops(ops)
    table = tr.heap_view(lay.base(which) + lay.abs, (P, 4), torch.float32)
    KG = tr.heap_view(lay.base(which) + lay.kg, (B, P * Sk) + tuple(k.shape[2:]), ops.op_dtype)
    VG = tr.heap_view(lay.base(which) + lay.vg, (B, P * Sk) + tuple(k.shape[2:]), vops.op_dtype)
    QS = tr.heap_view(lay.base(which) + lay.qs, tuple(x.shape), ops.op_dtype)
    rot = (rope is not None and rope_k, False, rope is not None and rope_x)
    sc = []
    for t, c, rt, o in zip((k, v, x), cols, rot, (ops, vops, ops)):
        dst = table[r, c:c + 1]
        if not o.scaled:
            sc.append(None)
        elif known is not None and c in known:
            dst.copy_(known[c])
            sc.append(dst)
        elif rt:
            o.scale_of_rope(t, dst, *rope)
            sc.append(dst)
        else:
            o.scale_of(t, dst)
            sc.append(dst)
    for b in range(B):
        if rot[0]:
            ops.stage_rope(k[b], KG[b, r * Sk:(r + 1) * Sk], sc[0], rope[0][b], rope[1])
        else:
            ops.stage(k[b], KG[b, r * Sk:(r + 1) * Sk], sc[0])
        vops.stage(v[b], VG[b, r * Sk:(r + 1) * Sk], sc[1])
    if rot[2]:
        ops.stage_rope(x, QS, sc[2], *rope)
    else:
        ops.stage(x, QS, sc[2])
    for p in range(P):
        if p != r:
            tr.signal(p, FLAG_STAGED + r, pid, "main")
    return KG, VG, QS, table


def _close_pass(tr, pid):
    """Every rank has seen every peer ENTER pass pid before it leaves it. A peer signals STAGED(pid) only after its
    whole pass pid-1 (pulls from my heap, consumption of what I put into its heap) was enqueued before it, so when I
    overwrite this parity's regions again in pass pid+1 ... pid+2 nobody can still be reading them. Costs nothing:
    by the end of a pass the peers have long staged."""
    for p in range(tr.world):
        if p != tr.rank:
            tr.wait(FLAG_STAGED + p, pid, "main")


class _OwnerGate:
    """Before the first transfer from an owner: wait for STAGED[owner] (once per stream fan-out) and fetch the owner's
    scale row (16 bytes) into the local table the kernels read."""

    def __init__(self, tr, pid, lay, which, scales):
        self.tr, self.pid, self.lay, self.which, self.scales, self.seen = tr, pid, lay, which, scales, set()

    def __call__(self, owner, stream):
        if owner != self.tr.rank and (stream, owner) not in self.seen:
            self.tr.wait(FLAG_STAGED + owner, self.pid, stream)
            self.seen.add((stream, owner))
            if self.scales is not None and stream == "pull":
                self.tr.pull(self.scales[owner], owner, self.lay.base(self.which) + self.lay.abs + owner * 16, "pull")


def _gather_q_chunks(tr, lay, which, plan, QS, gate, ops):
    """-> this rank's compute chunks of the staged Q-like tensor (views of the local stage or pulled copies)"""
    B = QS.shape[0]
    chunks = []
    for qc in plan.q_chunks:
        if qc.owner == tr.rank:
            c = QS[:, qc.start:qc.start + qc.length]
            # (B > 1: a row slice of the stage is strided over the batch; the step functions take contiguous tensors)
            chunks.append(c if c.is_contiguous() else c.contiguous())
        else:
            buf = torch.empty((B, qc.length) + tuple(QS.shape[2:]), dtype=QS.dtype, device=QS.device)
            gate(qc.owner, "pull")
            for b in range(B):
                _pull_striped(tr, buf[b], qc.owner, lay.q_row_off("qs", which, b, qc.start, QS.element_size()))
            chunks.append(buf)
    return chunks


def _pull_group(tr, lay, which, group, KG, VG, gate):
    B = KG.shape[0]
    if all(c.owner == tr.rank for c in group.chunks):
        return []                       # local rows are already in place: nothing to wait for
    for c in group.chunks:
        if c.owner == tr.rank:
            continue
        gate(c.owner, "pull")
        for b in range(B):
            for region, arr in (("kg", KG), ("vg", VG)):
                _pull_striped(tr, arr[b, c.pos0:c.pos0 + c.length], c.owner,
                              lay.kv_row_off(region, which, b, c.pos0, arr.element_size()))
    return tr.record("pull")


def _return_rows(tr, lay, which, pid, plan, chunks, out, region, itemsize, ops=None, rope=None):
    """Exit permutation: rows computed here for other ranks go to the owner's landing area, mine come back the same way.
    chunks[i] belongs to plan.q_chunks[i]; `out` [B, Sq, H, D] is this rank's contiguous result. rope: None, or
    (positions int32 [B,Sq], inv_freq): the rows are gradients w.r.t. rotated rows, and the owner's copies into `out`
    are the conjugate rotations (ops.rope_conj) that make them gradients w.r.t. the un-rotated ones."""
    B, r = out.shape[0], tr.rank

    def place(s, l, src):
        if rope is None:
            out[:, s:s + l].copy_(src)
            return
        for b in range(B):
            ops.rope_conj(src[b], out[b, s:s + l], rope[0][b, s:s + l], rope[1])

    ev = tr.record("main")
    tr.wait_event("push", ev)
    dests = {}
    for qc, c in zip(plan.q_chunks, chunks):
        if qc.owner == r:
            place(qc.start, qc.length, c)
        else:
            st = dests.setdefault(qc.owner, _pick(tr, "push"))     # a destination's payloads and its flag: one stream
            for b in range(B):
                tr.put(c[b], qc.owner, lay.q_row_off(region, which, b, qc.start, itemsize), st)
    for p in sorted(dests):
        tr.signal(p, FLAG_RES + r, pid, dests[p])
    land = tr.heap_view(lay.base(which) + getattr(lay, region), tuple(out.shape), out.dtype)
    for peer in sorted({peer for (_, _, peer) in plan.q_sends}):
        tr.wait(FLAG_RES + peer, pid, "main")
    for (s, l, peer) in plan.q_sends:
        place(s, l, land[:, s:s + l])
    return out


class _Puller:
    """Enqueues the K/V pulls group by group, a couple of groups ahead of the compute loop: the first tile kernel is
    launched as soon as ITS operands are on their way instead of after the whole pass's transfer list was enqueued."""

    def __init__(self, tr, lay, which, groups, KG, VG, gate, tag, lookahead=1):
        self.tr, self.lay, self.which, self.groups, self.KG, self.VG, self.gate = tr, lay, which, groups, KG, VG, gate
        self.tag, self.lookahead, self.events = tag, lookahead, []

    def event(self, gi):
        upto = min(len(self.groups), gi + 1 + self.lookahead)
        while len(self.events) < upto:
            i = len(self.events)
            with _span(self.tr, "%s pull group %d" % (self.tag, i), "pull"):
                self.events.append(_pull_group(self.tr, self.lay, self.which, self.groups[i], self.KG, self.VG, self.gate))
        return self.events[gi]


def _sc(table, owner, col):
    return None if table is None else table[owner, col:col + 1]


def _batch_kw(ops, b):
    """The steps launch one batch row at a time; with attention dropout (ops carries a `dropout`) they say which global
    row it is, so that every batch row draws its own mask"""
    return {"batch0": b} if getattr(ops, "dropout", None) is not None else {}


def run_forward(plan, q, k, v, bias, seg, causal, ops, tr, want_f32=False, rope=None, rope_k=True):
    """-> (out [B,Sq,H,D] in bf16 or fp32, residuals). q/k/v: bf16 or fp32 shards (contiguous sharding).
    rope: None, or (positions int32 [B,Sq], inv_freq): q (and k when rope_k, Sq == Sk) are un-rotated and are rotated
    while staged."""
    B, Sq, H, D = q.shape
    Sk = k.shape[1]
    dev = q.device
    r = tr.rank
    lay = _layout_for(plan, q.shape, Sk, ops)
    tr.ensure(lay.total)
    pid = tr.next_pass()
    which = pid & 1
    # (result / carry buffers are allocated up front: nothing but enqueues stands between staging and the first kernel)
    n_q = len(plan.q_chunks)
    n_launch = [sum(1 for g in plan.fwd_groups for l in g.launches if l[0] == i) for i in range(n_q)]
    lens = [qc.length for qc in plan.q_chunks]
    out_chunks = [torch.empty((B, L, H, D), dtype=torch.bfloat16, device=dev) for L in lens]
    need32 = want_f32 or ops.scaled     # fp16 mode keeps the un-rounded output as the backward's residual
    out32 = [torch.empty((B, L, H, D), dtype=torch.float32, device=dev) if need32 else None for L in lens]
    lse_chunks = [torch.empty((B, H, L), dtype=torch.float32, device=dev) for L in lens]
    acc = [None] * n_q
    for i in range(n_q):
        if n_launch[i] > 1:
            acc[i] = (torch.empty((B, lens[i], H, D), dtype=torch.float32, device=dev),
                      torch.empty((B, H, lens[i]), dtype=torch.float32, device=dev),
                      torch.empty((B, H, lens[i]), dtype=torch.float32, device=dev))
    with _span(tr, "fwd stage q,k,v", "main"):
        KG, VG, QS, table = _stage_and_announce(tr, lay, which, pid, ops, k, v, q, (1, 2, 0), rope=rope, rope_x=True,
                                                rope_k=rope_k)
    # scale rows [sq, sk, sv, sdo] of every owner, local copy (mine straight from the heap row I just wrote)
    scales = None
    if ops.scaled:
        scales = torch.empty((tr.world, 4), dtype=torch.float32, device=dev)
        scales[r].copy_(table[r])
    tr.wait_event("pull", tr.record("main"))            # after everything that still reads this set (pass pid-2) and my staging
    gate = _OwnerGate(tr, pid, lay, which, scales)
    with _span(tr, "fwd pull q chunks", "pull"):
        q_chunks = _gather_q_chunks(tr, lay, which, plan, QS, gate, ops)
    ev_q = tr.record("pull")        # (every pull member carries its slice of the Q chunks before any K/V slice)
    puller = _Puller(tr, lay, which, plan.fwd_groups, KG, VG, gate, "fwd")

    done = [0] * n_q
    first_wait = True
    for gi, g in enumerate(plan.fwd_groups):
        ev = puller.event(gi)
        if first_wait:
            tr.wait_event("main", ev_q)
            first_wait = False
        tr.wait_event("main", ev)
        for (qi, p0, rows, owner) in g.launches:
            with _span(tr, "fwd kernel g%d q%d x %d keys" % (gi, qi, rows), "main"):
                first, last = done[qi] == 0, done[qi] == n_launch[qi] - 1
                done[qi] += 1
                a = acc[qi] or (None, None, None)
                sc = (_sc(scales, plan.q_chunks[qi].owner, 0), _sc(scales, owner, 1), _sc(scales, owner, 2))
                for b in range(B):
                    sl = slice(b, b + 1)
                    ops.fwd_step(q_chunks[qi][sl], KG[sl, p0:p0 + rows], VG[sl, p0:p0 + rows], out_chunks[qi][sl],
                                 lse_chunks[qi][sl], None if a[0] is None else a[0][sl],
                                 None if a[1] is None else a[1][sl], None if a[2] is None else a[2][sl],
                                 plan.q_chunks[qi].pos0, p0, causal, None if bias is None else bias[sl],
                                 None if seg is None else seg[sl], first, last, sc,
                                 None if out32[qi] is None else out32[qi][sl], **_batch_kw(ops, b))
    for i in range(n_q):
        if n_launch[i] == 0:     # a chunk that sees no key at all cannot occur with Sq == Sk causal; keep it defined
            out_chunks[i].zero_()
            lse_chunks[i].fill_(float("-inf"))
            if out32[i] is not None:
                out32[i].zero_()
    with _span(tr, "fwd return O rows", "main"):
        if want_f32:
            out = _return_rows(tr, lay, which, pid, plan, out32, torch.empty((B, Sq, H, D), dtype=torch.float32, device=dev),
                               "lq4", 4)
        else:
            out = _return_rows(tr, lay, which, pid, plan, out_chunks,
                               torch.empty((B, Sq, H, D), dtype=torch.bfloat16, device=dev), "lq2", 2)
        tr.wait_event("main", tr.record("push"))
        _close_pass(tr, pid)
    # the local Q chunk is a view of the heap stage, which the next pass of this parity overwrites: keep a copy
    q_res = [c.clone() if qc.owner == r else c for qc, c in zip(plan.q_chunks, q_chunks)]
    q_scales = tuple(_sc(scales, qc.owner, 0) for qc in plan.q_chunks)
    own = (_sc(scales, r, 1), _sc(scales, r, 2))
    res = dict(q_chunks=q_res, out_chunks=[o32 if ops.scaled else ob for o32, ob in zip(out32, out_chunks)],
               lse_chunks=lse_chunks, scales=q_scales + own)
    return out, res


def run_backward(plan, res, k, v, dout, bias, seg, causal, ops, tr, want_f32=False, rope=None, rope_k=True):
    """-> dq, dk, dv (contiguous shards; bf16, or fp32 when want_f32). `res`: residuals of run_forward
    (scales = one Q scale per compute chunk, then this rank's own K and V scales). rope, rope_k: as run_forward's; K is
    re-staged rotated when rope_k, and dq (and dk when rope_k) are the gradients w.r.t. the un-rotated q (and k)."""
    B, Sk, H, D = k.shape
    Sq = dout.shape[1]
    dev = k.device
    P, r = tr.world, tr.rank
    lay = _layout_for(plan, dout.shape, Sk, ops)
    tr.ensure(lay.total)
    pid = tr.next_pass()
    which = pid & 1
    q_chunks, out_chunks, lse_chunks = res["q_chunks"], res["out_chunks"], res["lse_chunks"]
    n_q = len(q_chunks)
    q_scales, (sk_own, sv_own) = res["scales"][:n_q], res["scales"][n_q:n_q + 2]
    with _span(tr, "bwd stage k,v,dO", "main"):
        KG, VG, DS, table = _stage_and_announce(tr, lay, which, pid, ops, k, v, dout, (1, 2, 3),
                                                known={1: sk_own, 2: sv_own} if ops.scaled else None,
                                                rope=rope if rope_k else None)
    scales = None
    if ops.scaled:
        scales = torch.empty((P, 4), dtype=torch.float32, device=dev)
        scales[r].copy_(table[r])
    tr.wait_event("pull", tr.record("main"))
    gate = _OwnerGate(tr, pid, lay, which, scales)
    with _span(tr, "bwd pull dO chunks", "pull"):
        do_chunks = _gather_q_chunks(tr, lay, which, plan, DS, gate, ops)
    ev_q = tr.record("pull")
    puller = _Puller(tr, lay, which, plan.bwd_groups, KG, VG, gate, "bwd")
    puller.event(0)

    tr.wait_event("main", ev_q)
    delta = [torch.empty_like(l) for l in lse_chunks]
    with _span(tr, "bwd prep (delta, lse, zero dq)", "main"):
        for i in range(n_q):
            ops.bwd_prep(out_chunks[i], do_chunks[i], _sc(scales, plan.q_chunks[i].owner, 3), delta[i])
        nlse = [ops.lse_for_bwd(l) for l in lse_chunks]
        dq_acc = [torch.zeros((B, c.shape[1], H, D), dtype=torch.float32, device=dev) for c in q_chunks]
    # position-ordered fp32 accumulators; every chunk's rows are initialised by its first launch (dkv_init)
    dKG = torch.empty((B, P * Sk, H, D), dtype=torch.float32, device=dev)
    dVG = torch.empty((B, P * Sk, H, D), dtype=torch.float32, device=dev)
    for gi, g in enumerate(plan.bwd_groups):
        tr.wait_event("main", puller.event(gi))
        seen = set()
        for (qi, p0, rows, owner) in g.launches:
            with _span(tr, "bwd kernel g%d q%d" % (gi, qi), "main"):
                init = p0 not in seen
                seen.add(p0)
                sc = (q_scales[qi], _sc(scales, owner, 1), _sc(scales, owner, 2), _sc(scales, plan.q_chunks[qi].owner, 3))
                for b in range(B):
                    sl = slice(b, b + 1)
                    ops.bwd_step(q_chunks[qi][sl], KG[sl, p0:p0 + rows], VG[sl, p0:p0 + rows], do_chunks[qi][sl],
                                 nlse[qi][sl], delta[qi][sl], dq_acc[qi][sl], dKG[sl, p0:p0 + rows],
                                 dVG[sl, p0:p0 + rows], plan.q_chunks[qi].pos0, p0, causal,
                                 None if bias is None else bias[sl], None if seg is None else seg[sl], sc, init,
                                 **_batch_kw(ops, b))
        c = g.chunks[0]
        if c.owner != r and g.launches:
            tr.wait_event("push", tr.record("main"))
            slot = plan.slot(c.index, r)
            st = _pick(tr, "push")
            with _span(tr, "bwd put partial g%d -> rank %d" % (gi, c.owner), st):
                for t, arr in enumerate((dKG, dVG)):
                    for b in range(B):
                        tr.put(arr[b, c.pos0:c.pos0 + c.length], c.owner,
                               lay.slot_off(which, slot, t) + b * c.length * lay.row * 4, st)
                tr.signal(c.owner, FLAG_PART + slot, pid, st)

    # dQ: cast and return to the rows' owners
    res_dtype = torch.float32 if want_f32 else torch.bfloat16
    if want_f32:
        dq_chunks = dq_acc
    else:
        dq_chunks = []
        for i in range(n_q):
            c = torch.empty(dq_acc[i].shape, dtype=torch.bfloat16, device=dev)
            ops.cast(dq_acc[i], c)
            dq_chunks.append(c)
    with _span(tr, "bwd return dQ rows", "main"):
        dq = _return_rows(tr, lay, which, pid, plan, dq_chunks, torch.empty((B, Sq, H, D), dtype=res_dtype, device=dev),
                          "lq4" if want_f32 else "lq2", 4 if want_f32 else 2, ops, rope)
    # dK/dV: own partial + landed partials -> one fused sum + cast per chunk
    dk = torch.empty((B, Sk, H, D), dtype=res_dtype, device=dev)
    dv = torch.empty((B, Sk, H, D), dtype=res_dtype, device=dev)
    with _span(tr, "bwd wait incoming partials", "main"):
        for (ci, peer) in plan.incoming:
            tr.wait(FLAG_PART + plan.slot(ci, peer), pid, "main")
    L = lay.chunk_rows
    with _span(tr, "bwd fold partials", "main"):
        for ci in range(plan.chunks_per_rank):
            for t, (acc_g, dst) in enumerate(((dKG, dk), (dVG, dv))):
                for b in range(B):
                    srcs = []
                    if ci in plan.own_computed:
                        srcs.append(acc_g[b, r * Sk + ci * L:r * Sk + (ci + 1) * L])
                    for (cj, peer) in plan.incoming:
                        if cj == ci:
                            off = lay.slot_off(which, plan.slot(ci, peer), t) + b * L * lay.row * 4
                            srcs.append(tr.heap_view(off, (L, H, D), torch.float32))
                    if srcs and rope is not None and rope_k and t == 0:
                        ops.reduce_cast_rope(srcs, dst[b, ci * L:(ci + 1) * L], rope[0][b, ci * L:(ci + 1) * L], rope[1])
                    elif srcs:
                        ops.reduce_cast(srcs, dst[b, ci * L:(ci + 1) * L])
                    else:
                        dst[b, ci * L:(ci + 1) * L].zero_()
    tr.wait_event("main", tr.record("push"))
    tr.wait_event("main", tr.record("pull"))
    _close_pass(tr, pid)
    return dq, dk, dv
