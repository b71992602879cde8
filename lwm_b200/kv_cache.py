"""Sequence-sharded KV cache — host mirror of `FlaxLLaMAAttention._concatenate_to_cache` (lwm/llama.py:440-492) in the
process-per-GPU model: every rank of the 'sp' group holds the rows [rank*L, (rank+1)*L) of cached_key / cached_value
(L = max_length / sp; in_specs PS(('dp','fsdp'), 'sp', 'tp', None), llama.py:468-469).

  * decode step (query length 1, llama.py:452-483): the new key/value row is written by the ONE rank that owns slot
    `cache_index` (`cur_index - axis_index * sp_size` in range), everybody else leaves its shard untouched;
  * prefill (query length > 1, llama.py:485-487: `dynamic_update_slice` at `cache_index`): the new rows are sharded like
    the queries (rank r holds rows [r*q_loc, (r+1)*q_loc) of them), their destination slots generally belong to other
    ranks, so the shards are all-gathered once and every rank copies the slice that falls into its own cache rows.
Without the rotary keywords this is pure data movement (copies and one all-gather). With them (freqs_cis, position_ids)
the new keys arrive un-rotated and are rotated as they are written (lwm_kv_cache_write_rope: one launch for k and v), so
the cache holds what apply_rotary_emb followed by the plain update would leave in it, bit for bit. The cache shards are
exactly the k / v arguments `ringattention` (prefill: "K/V = whole cache") and `ringattention_inference` (decode) take
(with rotate_k=False when q is rotated inside the op).

dtype=torch.int8 is the 8-bit cache (QuantizedKV below; DESIGN.md §5): every new row is quantized as it is written
(lwm_kv_cache_write_q8, the keys rotated first when the rotary keywords are given), and both attention ops read it.
It is lossy and meant for generation only."""
import torch
import torch.distributed as dist

from . import _lib
from . import rope as _rope
from .ringattention import TorchComm, _dt


def kv_cache_write_rope(k_src, v_src, src0, n, cache_k, cache_v, dst0, pos, inv_freq):
    """rows [src0, src0+n) of k_src / v_src [B,n_src,H,128] -> rows [dst0, dst0+n) of cache_k / cache_v [B,L,H,128]
    (one dtype), k rotated at pos int32 [B,n_src] and rounded to the cache dtype, v copied (lwm_kv_cache_write_rope)"""
    B, n_src, H, D = k_src.shape
    _lib.call("lwm_kv_cache_write_rope", _lib.ptr(k_src), _lib.ptr(v_src), _dt(cache_k), _lib.ptr(cache_k),
              _lib.ptr(cache_v), _lib.ptr(pos), _lib.ptr(inv_freq), B, n_src, int(src0), int(n), cache_k.shape[1],
              int(dst0), H, D, _lib.stream_ptr())


def kv_cache_write_q8(k_src, v_src, src0, n, cache_k, cache_v, dst0, pos=None, inv_freq=None):
    """rows [src0, src0+n) of k_src / v_src [B,n_src,H,128] (bf16 or fp32, one dtype) quantized into rows
    [dst0, dst0+n) of the QuantizedKV caches cache_k / cache_v; pos int32 [B,n_src] and inv_freq given: k is rotated at
    pos and rounded to its dtype first, as kv_cache_write_rope stores it (lwm_kv_cache_write_q8)"""
    B, n_src, H, D = k_src.shape
    _lib.call("lwm_kv_cache_write_q8", _lib.ptr(k_src), _lib.ptr(v_src), _dt(k_src), _lib.ptr(cache_k.data),
              _lib.ptr(cache_k.exp), _lib.ptr(cache_v.data), _lib.ptr(cache_v.exp), _lib.ptr(pos), _lib.ptr(inv_freq),
              B, n_src, int(src0), int(n), cache_k.shape[1], int(dst0), H, D, _lib.stream_ptr())


class QuantizedKV:
    """One tensor (keys or values) of the 8-bit KV cache, [B,L,H,128] rows: data int8 [B,L,H,128] holds the codes and
    exp int8 [B,H,L,4] one power-of-two exponent per 32-element group, head-major (lwm_b200/csrc/kv_q8.cuh). A value is
    code * 2^e, exact in fp32 and bf16; code -128 is NaN. It stands where a cache shard goes: ringattention_inference
    and ringattention(..., rotate_k=False) accept it for k and v (generation only, no gradient) and stage their operand
    copies straight from the codes."""
    dtype = torch.int8
    requires_grad = False

    def __init__(self, data, exp):
        if data.dtype != torch.int8 or exp.dtype != torch.int8:
            raise TypeError("QuantizedKV: data and exp must be int8, got %s and %s" % (data.dtype, exp.dtype))
        if data.dim() != 4 or data.shape[-1] != 128:
            raise ValueError("QuantizedKV: data must be [B,L,H,128], got %s" % (tuple(data.shape),))
        B, L, H, _ = data.shape
        if tuple(exp.shape) != (B, H, L, 4):
            raise ValueError("QuantizedKV: exp must be [B,H,L,4] = %s, got %s" % ((B, H, L, 4), tuple(exp.shape)))
        if not (data.is_contiguous() and exp.is_contiguous()) or data.device != exp.device:
            raise ValueError("QuantizedKV: data and exp must be contiguous and on one device")
        self.data, self.exp = data, exp

    @classmethod
    def zeros(cls, batch, length, num_heads, device="cuda"):
        """an all-zero cache (the value of a bf16 / fp32 cache of zeros)"""
        return cls(torch.zeros((batch, length, num_heads, 128), dtype=torch.int8, device=device),
                   torch.zeros((batch, num_heads, length, 4), dtype=torch.int8, device=device))

    @property
    def shape(self):
        return self.data.shape

    @property
    def device(self):
        return self.data.device

    @property
    def is_cuda(self):
        return self.data.is_cuda

    @property
    def nbytes(self):
        return self.data.numel() + self.exp.numel()

    def contiguous(self):
        return self

    def __getitem__(self, b):
        """batch row b as a cache of one row, [1,L,H,128] (views of data[b] and exp[b]): the peer-memory executor
        stages a shard one batch row at a time"""
        b = range(self.shape[0])[b]
        return QuantizedKV(self.data[b:b + 1], self.exp[b:b + 1])

    def dequantize(self, dtype):
        """-> the rows' values [B,L,H,128] in bf16 or fp32 (exact; lwm_kv_dequant_q8)"""
        if dtype not in (torch.bfloat16, torch.float32):
            raise ValueError("QuantizedKV.dequantize: dtype must be bfloat16 or float32, got %s" % dtype)
        if not self.is_cuda:
            raise _lib.LwmError("QuantizedKV.dequantize: the cache must live on an sm_90 GPU (no CPU fallback)")
        B, L, H, D = self.shape
        out = torch.empty(self.shape, dtype=dtype, device=self.device)
        _lib.call("lwm_kv_dequant_q8", _lib.ptr(self.data), _lib.ptr(self.exp), _lib.ptr(out), _dt(out), B, L, H, D,
                  _lib.stream_ptr())
        return out


def kv_cache_write_at(key, value, cache_k, cache_v, cursor, lo, max_length, pos=None, inv_freq=None, max_position=0):
    """the decode write of key / value [B,1,H,128] (bf16 or fp32, contiguous) into this rank's shards cache_k / cache_v
    [B,L,H,128] of a max_length-row cache (tensors of key's dtype, or QuantizedKV) at the global slot cursor[0]
    (cursor: int32 [2] on the GPU, the slot and a zero word), which it advances by one on the device. Only the owner of
    the slot (lo <= slot < lo + L) writes, as kv_cache_write_rope / kv_cache_write_q8 / a row copy at that row would.
    pos int32 [B,1] and inv_freq: k is rotated first. A slot >= max_length or a position outside [0, max_position)
    writes nothing and sets a bit of the device error word (rope.error_word). No host synchronisation: the call can be
    captured in a CUDA graph (lwm_kv_cache_write_at)."""
    B, _, H, D = key.shape
    q8 = isinstance(cache_k, QuantizedKV)
    _lib.call("lwm_kv_cache_write_at", _lib.ptr(key), _lib.ptr(value), _dt(key),
              _lib.ptr(cache_k.data if q8 else cache_k), _lib.ptr(cache_v.data if q8 else cache_v),
              _lib.ptr(cache_k.exp if q8 else None), _lib.ptr(cache_v.exp if q8 else None), _lib.ptr(pos),
              _lib.ptr(inv_freq), int(max_position), _lib.ptr(cursor), int(lo), cache_k.shape[1], int(max_length), B,
              H, D, _lib.ptr(_rope.error_word(key.device)), _lib.stream_ptr())


class ShardedKVCache:
    """comm: None (torch.distributed over `group`, or a ring of one), or an object with TorchComm's all_gather and
    `world` / `rank` attributes (e.g. an in-process stand-in that runs the real kernels on emulated ranks).

    On a GPU the write slot is kept twice: cache_index on the host and `cursor`, an int32 on the device. Every decode
    write goes through kv_cache_write_at, which reads the slot from the cursor and advances it on the device, eager or
    captured, so the decode step can be recorded once in a CUDA graph and replayed token after token (INTEGRATION.md
    "Decode in a CUDA graph"). The prefill stays eager. A CPU cache (host bookkeeping) writes at the host index."""
    write_rope = staticmethod(kv_cache_write_rope)
    write_q8 = staticmethod(kv_cache_write_q8)
    write_at = staticmethod(kv_cache_write_at)

    def __init__(self, batch, max_length, num_heads, head_dim, dtype=torch.bfloat16, device="cuda", group=None,
                 comm=None):
        self.group = group
        self.world, self.rank = 1, 0
        if comm is not None:
            self.world, self.rank = comm.world, comm.rank
        elif dist.is_available() and dist.is_initialized():
            self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
            comm = TorchComm(group, self.world)
        self.comm = comm
        if max_length % self.world:
            raise ValueError("max_length %d must be divisible by the ring size %d" % (max_length, self.world))
        self.max_length = max_length
        self.shard_len = max_length // self.world
        shape = (batch, self.shard_len, num_heads, head_dim)
        self.quantized = dtype == torch.int8
        if self.quantized:
            if head_dim != 128:
                raise ValueError("ShardedKVCache: the 8-bit cache needs head_dim 128, got %d" % head_dim)
            self.cached_key = QuantizedKV.zeros(batch, self.shard_len, num_heads, device)
            self.cached_value = QuantizedKV.zeros(batch, self.shard_len, num_heads, device)
        else:
            self.cached_key = torch.zeros(shape, dtype=dtype, device=device)       # jnp.zeros (llama.py:444-445)
            self.cached_value = torch.zeros(shape, dtype=dtype, device=device)
        self._on_gpu = self.cached_key.device.type == "cuda"
        self._index = 0
        self._cursor = None             # made on first use (_device_cursor): the cache allocates only its rows here
        self._captured = False          # a decode write was captured: replays move the cursor without the host

    def _device_cursor(self):
        """[the slot, the write kernel's arrival counter (zero between writes)], int32 on the cache's device; made by the
        first eager decode write or `cursor` read, with the GPU's error word. Not inside a capture: the fill would be
        recorded and every replay would rewind the slot."""
        if self._cursor is None:
            if _rope.capturing():
                raise RuntimeError("ShardedKVCache: the device cursor does not exist yet; run the decode step once "
                                   "eagerly (the warm-up) before capturing it")
            cursor = torch.zeros(2, dtype=torch.int32, device=self.cached_key.device)
            cursor[0].fill_(self._index)
            if self._on_gpu:
                _rope.error_word(cursor.device)
            self._cursor = cursor
        return self._cursor

    @property
    def cursor(self):
        """the slot of the next write as a 0-d int32 device tensor (a view of the cursor). A decode write advances it,
        so whatever a step derives from it (decode_attention_mask, position_ids) is computed before concatenate."""
        return self._device_cursor()[0]

    @property
    def cache_index(self):
        """the global slot of the next write (the reference's cache_index). Once a decode write has been captured in a
        CUDA graph, replays advance the device cursor behind the host's back, and each read synchronises once to fetch
        it."""
        if self._captured:
            if _rope.capturing():
                raise RuntimeError("ShardedKVCache.cache_index cannot be read while capturing a CUDA graph (it would "
                                   "need a synchronisation); use the device tensor `cursor`")
            self._index = int(self._cursor[0].item())
        return self._index

    @cache_index.setter
    def cache_index(self, value):
        value = int(value)
        if value < 0:
            raise ValueError("ShardedKVCache.cache_index must be >= 0, got %d" % value)
        self._index = value
        if self._cursor is not None:
            self._cursor[0].fill_(value)

    def take_errors(self):
        """-> the bits the device checks have set since the last call, and clears them: rope.ERR_SLOT (a decode write at
        a slot >= max_length: nothing was written) and rope.ERR_POSITION (a position outside [0, max_position) of the
        rotary table: nothing was written, or a captured ringattention_inference rotated q at it). The word belongs to
        the GPU: every cache and capturing op on it shares it. One synchronisation."""
        if not self._on_gpu:
            return 0
        return _rope.take_errors(self.cached_key.device)

    def concatenate(self, key, value, *, freqs_cis=None, position_ids=None):
        """key/value: the new rows. Decode: [B,1,H,D], replicated along the ring. Prefill: this rank's shard
        [B,q_loc,H,D] of the q_loc*world new rows. Returns (cached_key, cached_value) shards after the update and
        advances cache_index by the number of new rows (llama.py:488-491).
        freqs_cis, position_ids: both None (key is already rotated), or key is the un-rotated head-split projection and
        position_ids [B,1] (decode, replicated) or [B,q_loc] (prefill, this rank's rows) are the positions of the new
        rows (checked as ringattention checks them); key and value must then have the cache's dtype. Decode: the owner
        of the slot makes one write launch. Prefill: the positions travel with the rows through the all-gather and
        every rank rotates only the slice it keeps, straight into its shard.
        The 8-bit cache (dtype=torch.int8): key and value are bf16 or fp32, of one dtype, and every write goes through
        write_q8 (one launch for k and v, rotating the keys first when the rotary keywords are given); each rank
        quantizes only the rows it keeps. The returned pair is QuantizedKV.
        On a GPU the decode write is one kv_cache_write_at launch on every rank (only the owner writes) at the device
        cursor, and it can be captured in a CUDA graph: key, value and position_ids are then device tensors, and a slot
        past max_length or a position outside the table writes nothing and sets a bit that take_errors reports (the
        eager decode past max_length writes nothing either). The prefill cannot be captured."""
        decode = key.shape[1] == 1 and value.shape[1] == 1 and self._is_decode(key)
        capturing = _rope.capturing()
        if capturing and not decode:
            raise RuntimeError("ShardedKVCache.concatenate: only the decode step (one new row) can be captured in a CUDA "
                               "graph; run the prefill eagerly before capturing")
        # (the decode write on a GPU checks its positions on the device itself)
        rope = _rope.check_position_ids("ShardedKVCache.concatenate", freqs_cis, position_ids,
                                        (key.shape[0], key.shape[1]), key.device, device_check=False)
        if self.quantized:
            if not (key.dtype == value.dtype and key.dtype in (torch.bfloat16, torch.float32)):
                raise ValueError("ShardedKVCache.concatenate: the 8-bit cache takes bfloat16 or float32 key and value "
                                 "of one dtype, got %s and %s" % (key.dtype, value.dtype))
        elif rope is not None and not (key.dtype == value.dtype == self.cached_key.dtype):
            raise ValueError("ShardedKVCache.concatenate: with the rotary keywords key and value must have the cache "
                             "dtype %s, got %s and %s" % (self.cached_key.dtype, key.dtype, value.dtype))
        if decode and self._on_gpu:
            self._write_decode(key, value, rope, freqs_cis, capturing)
            return self.cached_key, self.cached_value
        if self.quantized:
            return self._concatenate_q8(key, value, rope)
        lo = self.rank * self.shard_len
        ci = self.cache_index
        if decode:
            cur = ci - lo
            if 0 <= cur < self.shard_len:
                if rope is None:
                    self.cached_key[:, cur].copy_(key[:, -1])
                    self.cached_value[:, cur].copy_(value[:, -1])
                else:
                    self.write_rope(key.contiguous(), value.contiguous(), 0, 1, self.cached_key, self.cached_value, cur,
                                    *rope)
            n_new = 1
        else:
            n_new = key.shape[1] * self.world
            if ci + n_new > self.max_length:
                raise ValueError("cache overflow: %d + %d > %d" % (ci, n_new, self.max_length))
            # global slots [ci, ci + n_new) intersected with my rows [lo, lo + shard_len)
            a, b = max(ci, lo), min(ci + n_new, lo + self.shard_len)
            if rope is not None:
                k_all, v_all, p_all = (self._gather_rows(t.contiguous()) for t in (key, value, rope[0]))
                if b > a:
                    self.write_rope(k_all.contiguous(), v_all.contiguous(), a - ci, b - a,
                                    self.cached_key, self.cached_value, a - lo, p_all.contiguous(), rope[1])
                self.cache_index = ci + n_new
                return self.cached_key, self.cached_value
            for new, cache in ((key, self.cached_key), (value, self.cached_value)):
                full = self._gather_rows(new.contiguous())
                if b > a:
                    cache[:, a - lo:b - lo].copy_(full[:, a - ci:b - ci])
        self.cache_index = ci + n_new
        return self.cached_key, self.cached_value

    def _write_decode(self, key, value, rope, freqs_cis, capturing):
        """the decode write of a GPU cache at the device cursor (eager and captured alike)"""
        B, _, H, D = self.cached_key.shape
        if tuple(key.shape) != (B, 1, H, D) or tuple(value.shape) != (B, 1, H, D):
            raise ValueError("ShardedKVCache.concatenate: the decode rows must be [B,1,H,D] = %s, got %s and %s"
                             % ((B, 1, H, D), tuple(key.shape), tuple(value.shape)))
        if capturing and not (key.is_cuda and value.is_cuda):
            raise ValueError("ShardedKVCache.concatenate: while capturing a CUDA graph key and value must be device "
                             "tensors")
        cursor = self._device_cursor()
        dev = cursor.device
        if self.quantized:
            key, value = key.to(device=dev).contiguous(), value.to(device=dev).contiguous()
        else:       # (a row copy casts to the cache dtype)
            dt = self.cached_key.dtype
            key = key.to(device=dev, dtype=dt).contiguous()
            value = value.to(device=dev, dtype=dt).contiguous()
        pos, inv_freq = rope if rope is not None else (None, None)
        self.write_at(key, value, self.cached_key, self.cached_value, cursor, self.rank * self.shard_len,
                      self.max_length, pos, inv_freq, 0 if rope is None else freqs_cis.max_position)
        if capturing:
            self._captured = True
        else:
            self._index += 1

    def _concatenate_q8(self, key, value, rope):
        pos, inv_freq = rope if rope is not None else (None, None)
        lo = self.rank * self.shard_len
        ci = self.cache_index
        if key.shape[1] == 1 and value.shape[1] == 1 and self._is_decode(key):
            cur = ci - lo
            if 0 <= cur < self.shard_len:
                self.write_q8(key.contiguous(), value.contiguous(), 0, 1, self.cached_key, self.cached_value, cur,
                              None if pos is None else pos.contiguous(), inv_freq)
            self.cache_index = ci + 1
            return self.cached_key, self.cached_value
        n_new = key.shape[1] * self.world
        if ci + n_new > self.max_length:
            raise ValueError("cache overflow: %d + %d > %d" % (ci, n_new, self.max_length))
        a, b = max(ci, lo), min(ci + n_new, lo + self.shard_len)
        k_all, v_all = self._gather_rows(key.contiguous()), self._gather_rows(value.contiguous())
        p_all = None if pos is None else self._gather_rows(pos.contiguous()).contiguous()
        if b > a:
            self.write_q8(k_all.contiguous(), v_all.contiguous(), a - ci, b - a, self.cached_key,
                          self.cached_value, a - lo, p_all, inv_freq)
        self.cache_index = ci + n_new
        return self.cached_key, self.cached_value

    def _is_decode(self, key):
        # a one-row prefill on a one-rank "ring" is the same write; on a real ring a [B,1,...] argument is the
        # replicated decode row (the reference switches on query.shape[1] == 1, llama.py:451)
        return True

    def _gather_rows(self, x):
        if self.world == 1:
            return x
        B, n = x.shape[0], x.shape[1]
        g = self.comm.all_gather(x)                                 # [world, B, n, ...], rank-major
        return g.transpose(0, 1).reshape((B, self.world * n) + tuple(x.shape[2:]))
