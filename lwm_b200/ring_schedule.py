"""Ring schedules for the sequence-parallel attention op (host logic only — no numerics here).

The reference rotates K/V one hop per step with lax.ppermute (SURVEY.md Appendix A), because a
TPU torus only has neighbour links. On an NVSwitch box every peer is one hop away at full
bandwidth, so the "ring" is only a SCHEDULE: at step `idx` rank r needs the K/V block that
originated on rank (r - idx) mod P. We fetch it straight from its owner (one NCCL send/recv
pair per block, posted one step ahead on a side stream, double-buffered against the tile
kernels) instead of forwarding it hop by hop; K/V are never modified, so there is no chained
dependency between steps. In the backward the dK/dV partial of a block is pushed straight back
to the block's owner, which accumulates it (the reference lets dk/dv ride the ring instead).

Two schedules, identical inputs/outputs (contiguous sequence shards, lwm/llama.py:559-566):
  contiguous  the reference's work assignment: rank r computes its own rows against blocks
              0..r. Causal work is unbalanced (rank P-1 does 2P-1 times the work of rank 0).
  zigzag      the sequence is cut in 2P half-chunks; rank r COMPUTES query chunks r and
              2P-1-r, which makes every rank's causal work identical at every step. Only Q
              (and dO) are permuted on entry and O (and dQ) on exit; K/V half-chunks are pulled
              from their contiguous owners directly and dK/dV partials pushed back to them.

The plan is a pure function of (world, rank, sizes, causal, layout): every rank derives the
same global picture, so sends and receives always match without negotiation.
"""
import os
from dataclasses import dataclass, field
from typing import List, Tuple


def visible(q_pos0, q_len, k_pos0, causal):
    """Does any query of the chunk see any key of the chunk (token-level causal mask)?"""
    return (not causal) or (q_pos0 + q_len - 1 >= k_pos0)


@dataclass
class KvRef:
    owner: int      # rank holding the block in the contiguous layout
    start: int      # local row offset inside the owner's shard
    length: int
    pos0: int       # global token position of its first row


@dataclass
class QRef:
    owner: int      # rank whose contiguous shard holds these rows
    start: int
    length: int
    pos0: int


@dataclass
class Step:
    kv: List[KvRef] = field(default_factory=list)              # blocks this rank consumes
    sends: List[Tuple[int, int, int]] = field(default_factory=list)  # (start, length, peer) of my shard
    pairs: List[Tuple[int, int]] = field(default_factory=list)  # (q chunk idx, kv idx in `kv`)


@dataclass
class Plan:
    world: int
    rank: int
    layout: str
    q_chunks: List[QRef]             # query chunks this rank computes
    q_sends: List[Tuple[int, int, int]]  # (start, length, peer): rows of MY shard computed elsewhere
    steps: List[Step]
    params: Tuple = ()               # (Sq, Sk, causal, n_sub_first, n_sub_last): lets a rank re-derive a peer's plan


def choose_layout(world, Sq, Sk, causal, layout):
    if layout == "auto":
        layout = "zigzag" if (causal and world > 1 and Sq == Sk and Sq % 256 == 0) else "contiguous"
    if layout == "zigzag" and not (Sq == Sk and Sq % 256 == 0):
        raise ValueError("zigzag layout needs Sq == Sk and a shard length divisible by 256")
    if layout not in ("contiguous", "zigzag"):
        raise ValueError("unknown layout %r" % (layout,))
    return layout


def _zig(c, P):
    """rank that COMPUTES half-chunk c (0 <= c < 2P) in the zigzag assignment."""
    return c if c < P else 2 * P - 1 - c


def compute_chunks(world, rank, Sq, layout):
    """Query chunks computed by `rank` (as references into the contiguous shards)."""
    if layout == "contiguous":
        return [QRef(rank, 0, Sq, rank * Sq)]
    h = Sq // 2
    return [QRef(c // 2, (c % 2) * h, h, c * h) for c in (rank, 2 * world - 1 - rank)]


def step_kv(world, rank, idx, Sk, layout, sub=(0, 1)):
    """K/V blocks rank `rank` consumes at step idx (before visibility filtering). sub=(j, n): only the
    j-th of n equal row pieces of every block (sub-block pipelining of a step)."""
    src = (rank - idx) % world
    if layout == "contiguous":
        blocks = [KvRef(src, 0, Sk, src * Sk)]
    else:
        h = Sk // 2
        blocks = [KvRef(c // 2, (c % 2) * h, h, c * h) for c in (src, 2 * world - 1 - src)]
    j, n = sub
    if n == 1:
        return blocks
    return [KvRef(b.owner, b.start + j * (b.length // n), b.length // n, b.pos0 + j * (b.length // n)) for b in blocks]


def auto_sub(world, Sk, layout, min_piece=2048):
    """How many pieces to cut the first / last step's blocks into so that their transfer pipelines with the
    tile kernels instead of being exposed (nothing precedes step 0; nothing follows the last dK/dV return)."""
    # sub-stepping trades extra, smaller launches for less exposed transfer; it is opt-in (LWM_RING_SUBSTEPS=1)
    if world == 1 or os.environ.get("LWM_RING_SUBSTEPS", "0") != "1":
        return 1
    block = Sk if layout == "contiguous" else Sk // 2
    n = 1
    while n < 4 and block % (2 * n * 128) == 0 and block // (2 * n) >= min_piece:
        n *= 2
    return n


def make_plan(world, rank, Sq, Sk, causal, layout="auto", n_sub_first=1, n_sub_last=1):
    """n_sub_first / n_sub_last: split step 0 / step world-1 into that many sub-steps (same on every rank)."""
    layout = choose_layout(world, Sq, Sk, causal, layout)
    q_chunks = compute_chunks(world, rank, Sq, layout)
    # rows of my contiguous shard that another rank computes
    q_sends = []
    for peer in range(world):
        if peer == rank:
            continue
        for qc in compute_chunks(world, peer, Sq, layout):
            if qc.owner == rank:
                q_sends.append((qc.start, qc.length, peer))
    steps = []
    for idx in range(world):
        n_sub = n_sub_first if idx == 0 else (n_sub_last if idx == world - 1 else 1)
        if world == 1:
            n_sub = 1
        for j in range(n_sub):
            st = Step()
            for kv in step_kv(world, rank, idx, Sk, layout, (j, n_sub)):
                needed = [qi for qi, qc in enumerate(q_chunks) if visible(qc.pos0, qc.length, kv.pos0, causal)]
                if needed:
                    st.kv.append(kv)
                    st.pairs.extend((qi, len(st.kv) - 1) for qi in needed)
            # what do the OTHER ranks need from my shard at this (sub-)step?
            for peer in range(world):
                if peer == rank:
                    continue
                peer_q = compute_chunks(world, peer, Sq, layout)
                for kv in step_kv(world, peer, idx, Sk, layout, (j, n_sub)):
                    if kv.owner == rank and any(visible(qc.pos0, qc.length, kv.pos0, causal) for qc in peer_q):
                        st.sends.append((kv.start, kv.length, peer))
            steps.append(st)
    return Plan(world, rank, layout, q_chunks, q_sends, steps, (Sq, Sk, causal, n_sub_first, n_sub_last))


def work_units(plan, causal):
    """Causal work (in units of full chunk x chunk tiles; a diagonal pair counts 1/2) per step —
    used by the tests to assert the balance property of the zigzag schedule."""
    out = []
    for st in plan.steps:
        w = 0.0
        for qi, ki in st.pairs:
            qc, kv = plan.q_chunks[qi], st.kv[ki]
            if causal and kv.pos0 + kv.length - 1 > qc.pos0:   # straddles the diagonal
                w += 0.5 * qc.length * kv.length
            else:
                w += 1.0 * qc.length * kv.length
        out.append(w)
    return out


# ------------------------------------------------------------------------------------------------
# Peer-memory schedule (ring_peer.py): no lock-step ring — every rank pulls the K/V chunks it needs
# straight out of their owners' heaps, in a rank-staggered ("ring") order so that every owner serves
# about one puller at a time, and processes them in groups.
# ------------------------------------------------------------------------------------------------
@dataclass
class Chunk:
    owner: int      # rank holding the rows (contiguous sharding)
    index: int      # which of the owner's chunks (0 .. chunks_per_rank-1)
    start: int      # row offset inside the owner's shard
    length: int
    pos0: int       # global token position of the first row


@dataclass
class Group:
    chunks: List[Chunk] = field(default_factory=list)          # K/V chunks that must have arrived
    launches: List[Tuple[int, int, int, int]] = field(default_factory=list)   # (q chunk idx, first global key row, rows, K/V owner)


@dataclass
class PeerPlan:
    world: int
    rank: int
    layout: str
    chunks_per_rank: int
    q_chunks: List[QRef]                      # query chunks this rank computes (references into the owners' shards)
    q_sends: List[Tuple[int, int, int]]       # (start, length, peer): rows of MY shard that `peer` computes
    fwd_groups: List[Group]                   # coarse groups (few launches, few carry round trips)
    bwd_groups: List[Group]                   # one K/V chunk per launch (dK/dV partials leave chunk by chunk)
    incoming: List[Tuple[int, int]]           # (my chunk index, peer): dK/dV partials that will land in my heap
    own_computed: List[int]                   # my chunk indices I compute a partial for myself

    def slot(self, chunk_index, peer):
        """landing slot (in the OWNER's heap) of the partial `peer` computes for the owner's chunk `chunk_index`"""
        return chunk_index * self.world + peer


def kv_chunks_of(world, rank, Sk, layout):
    """the chunks rank `rank` OWNS (contiguous sharding): one per rank, or two half-shards under zigzag"""
    if layout == "contiguous":
        return [Chunk(rank, 0, 0, Sk, rank * Sk)]
    h = Sk // 2
    return [Chunk(rank, 0, 0, h, rank * Sk), Chunk(rank, 1, h, h, rank * Sk + h)]


def _merge_ranges(chunks):
    """contiguous global-position ranges [(pos0, rows)] covered by `chunks`"""
    out = []
    for c in sorted(chunks, key=lambda c: c.pos0):
        if out and out[-1][0] + out[-1][1] == c.pos0:
            out[-1] = (out[-1][0], out[-1][1] + c.length)
        else:
            out.append((c.pos0, c.length))
    return out


_PLAN_CACHE = {}


def make_peer_plan(world, rank, Sq, Sk, causal, layout="auto", fwd_group_chunks=4):
    """cached: the plan is a pure function of its arguments and is asked for twice per layer and step"""
    key = (world, rank, Sq, Sk, bool(causal), layout, fwd_group_chunks)
    if key not in _PLAN_CACHE:
        _PLAN_CACHE[key] = _make_peer_plan(*key)
    return _PLAN_CACHE[key]


def _make_peer_plan(world, rank, Sq, Sk, causal, layout, fwd_group_chunks):
    layout = choose_layout(world, Sq, Sk, causal, layout)
    q_chunks = compute_chunks(world, rank, Sq, layout)
    q_sends = []
    for peer in range(world):
        if peer != rank:
            q_sends += [(qc.start, qc.length, peer) for qc in compute_chunks(world, peer, Sq, layout) if qc.owner == rank]

    def sees(qc, c):
        return visible(qc.pos0, qc.length, c.pos0, causal)

    def needed_by(r):
        qs = compute_chunks(world, r, Sq, layout)
        return [c for o in range(world) for c in kv_chunks_of(world, o, Sk, layout) if any(sees(qc, c) for qc in qs)]

    need = needed_by(rank)
    local = [c for c in need if c.owner == rank]
    # ring order: owners rank-1, rank-2, ... (every owner then serves ~one puller at a time)
    remote = []
    for d in range(1, world):
        o = (rank - d) % world
        remote += [c for c in need if c.owner == o]

    def launches_for(chunks):
        # one launch per (q chunk, K/V owner): every operand carries its OWNER's fp16 scale (ring_peer.py), and the
        # chunks of one owner are adjacent in position, so they merge into one range
        ls = []
        for qi, qc in enumerate(q_chunks):
            for o in sorted({c.owner for c in chunks}, key=lambda o_: [c.owner for c in chunks].index(o_)):
                for (p0, rows) in _merge_ranges([c for c in chunks if c.owner == o and sees(qc, c)]):
                    ls.append((qi, p0, rows, o))
        return ls

    # forward: local chunks first (their compute hides the first pulls), then the remote chunks in a few big groups
    fwd_groups = []
    if local:
        fwd_groups.append(Group(local, launches_for(local)))
    first = 1 if not local else fwd_group_chunks
    i = 0
    while i < len(remote):
        n = first if i == 0 else fwd_group_chunks
        g = remote[i:i + n]
        fwd_groups.append(Group(g, launches_for(g)))
        i += n
    # backward: one chunk per launch; a local chunk first (hides the first pulls) and a local chunk last (hides the
    # last partial's flight) when there are any
    order = (local[:1] + remote + local[1:]) if local else remote
    bwd_groups = []
    for c in order:
        bwd_groups.append(Group([c], [(qi, c.pos0, c.length, c.owner) for qi, qc in enumerate(q_chunks) if sees(qc, c)]))
    incoming = []
    for c in kv_chunks_of(world, rank, Sk, layout):
        for peer in range(world):
            if peer != rank and any(n.owner == rank and n.index == c.index for n in needed_by(peer)):
                incoming.append((c.index, peer))
    return PeerPlan(world, rank, layout, 1 if layout == "contiguous" else 2, q_chunks, q_sends, fwd_groups, bwd_groups,
                    incoming, [c.index for c in local])
