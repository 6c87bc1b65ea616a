"""KV cache objects with the reference's Python-visible behaviour
(mlx_vlm/models/cache.py:337-439 `KVCache`, :45-70 `make_prompt_cache`).

Storage is device-first: ONE device pool per request (`KVPool`, laid out
(n_layers, 2, batch, n_kv_heads, capacity, head_dim) bf16) that the CUDA engine
writes directly (K is rotated and appended inside the QKV kernels), instead of
per-layer arrays grown by concatenation.  Each layer's `KVCache` is a view of the
pool that keeps `offset / keys / values / state / trim / update_and_fetch /
is_trimmable / size / empty / nbytes` semantics; capacity still grows in
`step = 256` multiples (cache.py:338).

`kv_bits=8` swaps the request's pool for a `QuantizedKVPool` (codes + bf16 scales / biases, the format of
csrc/kvq.cuh) viewed per layer by `QuantizedKVCache` (cache.py:233-335).
"""
from __future__ import annotations

from contextlib import nullcontext
from typing import Any, List, Optional

import torch


class KVPool:
    step = 256

    def __init__(self, n_layers: int, n_kv_heads: int, head_dim: int, device, batch: int = 1,
                 capacity: int = 0, dtype=torch.bfloat16, stream=None):
        self.n_layers, self.n_kv, self.hd = n_layers, n_kv_heads, head_dim
        self.batch = batch
        self.device = device
        self.dtype = dtype
        self.stream = stream  # the stream the engine writes this pool on (None: the current stream)
        self.buf: Optional[torch.Tensor] = None
        self.capacity = 0
        self.generation = 0  # bumped whenever the buffer moves (engine must re-bind)
        if capacity:
            self.reserve(capacity)

    def reserve(self, n_tokens: int, live_tokens: int = 0) -> bool:
        """Make room for n_tokens positions; returns True if the buffer moved."""
        if n_tokens <= self.capacity:
            return False
        cap = ((max(n_tokens, 2 * self.capacity) + self.step - 1) // self.step) * self.step
        new = torch.zeros((self.n_layers, 2, self.batch, self.n_kv, cap, self.hd),
                          dtype=self.dtype, device=self.device)
        if self.buf is not None and live_tokens > 0:
            new[..., :live_tokens, :].copy_(self.buf[..., :live_tokens, :])
        self.buf = new
        self.capacity = cap
        self.generation += 1
        return True


def _kvq_check(group_size: int, bits, head_dim: Optional[int] = None):
    if bits != 8:
        raise NotImplementedError(f"{bits}-bit KV cache: only kv_bits=8 is built")
    if group_size not in (32, 64, 128) or (head_dim is not None and head_dim % group_size):
        raise ValueError(f"kv_group_size={group_size}: must be 32, 64 or 128 and divide head_dim={head_dim}")


class QuantizedKVPool:
    """8-bit twin of `KVPool` (format and arithmetic: csrc/kvq.cuh): codes (n_layers, 2, batch, n_kv, capacity,
    head_dim) uint8 plus scales and biases (..., capacity, head_dim / group_size) bf16.  The one owner of the
    allocation, growth and bulk conversion of 8-bit pools."""
    step = 256
    bits = 8

    def __init__(self, n_layers: int, n_kv_heads: int, head_dim: int, device, group_size: int = 64,
                 batch: int = 1, capacity: int = 0, stream=None):
        _kvq_check(group_size, 8, head_dim)
        self.n_layers, self.n_kv, self.hd = n_layers, n_kv_heads, head_dim
        self.group_size = group_size
        self.batch = batch
        self.device = device
        self.stream = stream
        self.codes: Optional[torch.Tensor] = None
        self.scales: Optional[torch.Tensor] = None
        self.biases: Optional[torch.Tensor] = None
        self.capacity = 0
        self.generation = 0
        if capacity:
            self.reserve(capacity)

    @property
    def planes(self) -> int:
        return self.n_layers * 2 * self.batch * self.n_kv

    def bytes_per_position(self) -> int:
        """bytes of one position of one row over all layers: codes + bf16 scales and biases"""
        return self.n_layers * 2 * self.n_kv * (self.hd + 2 * 2 * (self.hd // self.group_size))

    def reserve(self, n_tokens: int, live_tokens: int = 0) -> bool:
        if n_tokens <= self.capacity:
            return False
        cap = ((max(n_tokens, 2 * self.capacity) + self.step - 1) // self.step) * self.step
        lead = (self.n_layers, 2, self.batch, self.n_kv, cap)
        ng = self.hd // self.group_size
        with torch.cuda.stream(self.stream) if self.stream is not None else nullcontext():
            new = (torch.zeros(lead + (self.hd,), dtype=torch.uint8, device=self.device),
                   torch.zeros(lead + (ng,), dtype=torch.bfloat16, device=self.device),
                   torch.zeros(lead + (ng,), dtype=torch.bfloat16, device=self.device))
            if self.codes is not None and live_tokens > 0:
                for n_, o_ in zip(new, (self.codes, self.scales, self.biases)):
                    n_[..., :live_tokens, :].copy_(o_[..., :live_tokens, :])
        self.codes, self.scales, self.biases = new
        self.capacity = cap
        self.generation += 1
        return True

    @classmethod
    def from_pool(cls, pool: KVPool, n_tokens: int, group_size: int) -> "QuantizedKVPool":
        """Quantize the first n_tokens positions of every plane of a bf16 pool (same capacity)."""
        from .. import _native as N
        q = cls(pool.n_layers, pool.n_kv, pool.hd, pool.device, group_size=group_size, batch=pool.batch,
                capacity=max(pool.capacity, 1), stream=pool.stream)
        if pool.buf is not None and n_tokens > 0:
            N.check(N.lib().b200_kvq_quantize(pool.buf.data_ptr(), pool.capacity, q.codes.data_ptr(),
                                              q.scales.data_ptr(), q.biases.data_ptr(), q.capacity, q.planes,
                                              int(n_tokens), q.hd, group_size, _stream_handle(q)), "kvq_quantize")
        return q

    def to_bf16_pool(self, n_tokens: int) -> KVPool:
        """A bf16 pool of the same capacity holding the dequantized first n_tokens positions (the prefix a
        prefill chunk over this cache attends to)."""
        from .. import _native as N
        with torch.cuda.stream(self.stream) if self.stream is not None else nullcontext():
            out = KVPool(self.n_layers, self.n_kv, self.hd, self.device, batch=self.batch, capacity=self.capacity,
                         stream=self.stream)
        assert out.capacity == self.capacity
        if n_tokens > 0:
            N.check(N.lib().b200_kvq_dequantize(self.codes.data_ptr(), self.scales.data_ptr(),
                                                self.biases.data_ptr(), self.capacity, out.buf.data_ptr(),
                                                out.capacity, self.planes, int(n_tokens), self.hd, self.group_size,
                                                _stream_handle(self)), "kvq_dequantize")
        return out


def _stream_handle(pool) -> int:
    s = pool.stream if pool.stream is not None else torch.cuda.current_stream(pool.device)
    return s.cuda_stream


def should_quantize_kv_layer(layer_idx: int, num_layers: int) -> bool:
    """models/cache.py:8-21: the lock-step batch rule of kv_bits.  Stacks of more than two layers keep the last
    layer in bf16; shallower stacks quantize every layer."""
    if num_layers <= 2:
        return True
    return layer_idx < num_layers - 1


class BatchKVQPool:
    """The lock-step batch pool of kv_bits=8 (DESIGN §3).  The layers where `should_quantize_kv_layer` holds are a
    prefix 0 .. n_q-1; they live in a `QuantizedKVPool` of n_q layers, the remaining layers in a bf16 `KVPool` of
    n_layers - n_q layers (None when every layer is 8-bit).  Both have the same rows and capacity and grow together,
    so an 8-bit layer takes no bf16 storage."""
    step = 256
    bits = 8

    def __init__(self, n_layers: int, n_kv_heads: int, head_dim: int, device, group_size: int = 64, batch: int = 1,
                 capacity: int = 0, stream=None):
        self.n_layers, self.n_kv, self.hd = n_layers, n_kv_heads, head_dim
        self.n_q = sum(should_quantize_kv_layer(i, n_layers) for i in range(n_layers))
        self.group_size, self.batch, self.device, self.stream = group_size, batch, device, stream
        self.q = QuantizedKVPool(self.n_q, n_kv_heads, head_dim, device, group_size=group_size, batch=batch,
                                 capacity=capacity, stream=stream)
        self.bf = (KVPool(n_layers - self.n_q, n_kv_heads, head_dim, device, batch=batch, capacity=capacity,
                          stream=stream) if self.n_q < n_layers else None)

    @property
    def capacity(self) -> int:
        return self.q.capacity

    @property
    def generation(self) -> int:
        return self.q.generation

    @generation.setter
    def generation(self, v):
        self.q.generation = v

    def reserve(self, n_tokens: int, live_tokens: int = 0) -> bool:
        moved = self.q.reserve(n_tokens, live_tokens=live_tokens)
        if self.bf is not None:
            with torch.cuda.stream(self.stream) if self.stream is not None else nullcontext():
                self.bf.reserve(n_tokens, live_tokens=live_tokens)
            assert self.bf.capacity == self.q.capacity
        return moved

    def like(self, batch: int, capacity: int) -> "BatchKVQPool":
        return BatchKVQPool(self.n_layers, self.n_kv, self.hd, self.device, group_size=self.group_size, batch=batch,
                            capacity=capacity, stream=self.stream)

    def bytes_per_position(self) -> int:
        """bytes of one position of one row over all layers"""
        return self.q.bytes_per_position() + (self.n_layers - self.n_q) * 2 * self.n_kv * self.hd * 2

    def row_caches(self, row: int) -> list:
        """per-layer views of row `row`: QuantizedKVCache on the 8-bit layers, KVCache on the bf16 one"""
        out = [QuantizedKVCache(self.group_size, 8, pool=self.q, layer=l, row=row) for l in range(self.n_q)]
        out += [KVCache(self.bf, l - self.n_q, row=row) for l in range(self.n_q, self.n_layers)]
        for c in out:
            c._batch_pool = self
        return out


class _BaseCache:
    @property
    def state(self):
        return []

    def is_trimmable(self):
        return False

    def size(self):
        return 0

    def empty(self):
        raise NotImplementedError


class KVCache(_BaseCache):
    step = 256

    def __init__(self, pool: Optional[KVPool] = None, layer: int = 0, row: Optional[int] = None):
        self._pool = pool
        self._layer = layer
        self._row = row   # None: the whole (batch-1) pool; r: row r of a batched pool
        self.offset = 0
        self._own = None  # standalone storage when used without a pool (API parity)

    # --- reference attribute surface ---------------------------------------
    @property
    def keys(self):
        if self._pool is not None:
            if self._pool.buf is None:
                return None
            k = self._pool.buf[self._layer, 0]
            return k if self._row is None else k[self._row:self._row + 1]
        return None if self._own is None else self._own[0]

    @property
    def values(self):
        if self._pool is not None:
            if self._pool.buf is None:
                return None
            v = self._pool.buf[self._layer, 1]
            return v if self._row is None else v[self._row:self._row + 1]
        return None if self._own is None else self._own[1]

    def update_and_fetch(self, keys: torch.Tensor, values: torch.Tensor):
        """cache.py:345-367.  Generic (non-fused) append used by callers that
        bring their own K/V; the engine's kernels append in place instead."""
        prev = self.offset
        L = keys.shape[2]
        if self._pool is not None:
            self._pool.reserve(prev + L, live_tokens=prev)
            k, v = self.keys, self.values
        else:
            B, nkv, _, hd = keys.shape
            need = prev + L
            cap = 0 if self._own is None else self._own.shape[3]
            if need > cap:
                n_steps = (self.step + need - 1) // self.step
                new = torch.zeros((2, B, nkv, n_steps * self.step, hd), dtype=keys.dtype,
                                  device=keys.device)
                if self._own is not None:
                    new[:, :, :, :prev].copy_(self._own[:, :, :, :prev])
                self._own = new
            k, v = self._own[0], self._own[1]
        self.offset += L
        k[..., prev:self.offset, :] = keys
        v[..., prev:self.offset, :] = values
        return k[..., :self.offset, :], v[..., :self.offset, :]

    def size(self):
        return self.offset

    @property
    def state(self):
        return self.keys[..., :self.offset, :], self.values[..., :self.offset, :]

    @state.setter
    def state(self, v):
        k, vv = v
        self.offset = 0
        if self._pool is None:
            self._own = None
        self.update_and_fetch(k, vv)

    def is_trimmable(self):
        return True

    def trim(self, n):
        n = min(self.offset, n)
        self.offset -= n
        return n

    def extract(self, idx):
        cache = KVCache()
        if self.keys is None:
            if idx not in (0, -1):
                raise IndexError("KVCache row index out of range")
            return cache
        batch_size = int(self.keys.shape[0])
        if idx < 0:
            idx += batch_size
        if idx < 0 or idx >= batch_size:
            raise IndexError(f"KVCache row index {idx} out of range for batch size {batch_size}")
        cache.update_and_fetch(self.keys[idx:idx + 1, :, :self.offset, :].contiguous(),
                               self.values[idx:idx + 1, :, :self.offset, :].contiguous())
        return cache

    def make_mask(self, N: int, return_array: bool = False, window_size=None):
        # create_attention_mask (cache.py:73-83): "causal" for N>1, None for N==1
        if N == 1:
            return None
        return "causal"

    def to_quantized(self, group_size: int = 64, bits: int = 4) -> "QuantizedKVCache":
        """cache.py:415-423.  The layers of one request share a pool, so the first layer converted quantizes
        the whole pool (one kernel) and the other layers of the same pool become views of that 8-bit pool."""
        hd = self._pool.hd if self._pool is not None else (None if self._own is None else self._own.shape[-1])
        _kvq_check(group_size, bits, hd)
        if self._pool is None or self._pool.buf is None:
            raise NotImplementedError("to_quantized: only engine (pool-backed) caches with content are converted")
        pool = self._pool
        q = getattr(pool, "_q8", None)
        if q is None or q[0] != (pool.generation, self.offset, group_size):
            q = ((pool.generation, self.offset, group_size), QuantizedKVPool.from_pool(pool, self.offset, group_size))
            pool._q8 = q
        out = QuantizedKVCache(group_size=group_size, bits=bits, pool=q[1], layer=self._layer, row=self._row)
        out.offset = self.offset
        return out

    def empty(self):
        return self.keys is None or self.offset == 0 and self._pool is None and self._own is None

    @property
    def nbytes(self):
        k = self.keys
        if k is None:
            return 0
        return 2 * k.numel() * k.element_size()


class QuantizedKVCache(_BaseCache):
    """One layer's view of a `QuantizedKVPool` with the reference surface (cache.py:233-335): `keys` / `values`
    are (codes as uint32 (B, n_kv, S, head_dim / 4), scales, biases) with mx.quantize's packing (element 4i+j in
    bits 8j of word i).  The engine appends to the pool in its decode kernels."""
    step = 256

    def __init__(self, group_size: int = 64, bits: int = 8, pool: Optional[QuantizedKVPool] = None,
                 layer: int = 0, row: Optional[int] = None):
        _kvq_check(group_size, bits)
        self.group_size, self.bits = group_size, bits
        self._pool = pool
        self._layer = layer
        self._row = row
        self.offset = 0

    def _side(self, side: int):
        p = self._pool
        if p is None or p.codes is None:
            return None
        sl = slice(None) if self._row is None else slice(self._row, self._row + 1)
        return (p.codes[self._layer, side, sl].view(torch.uint32), p.scales[self._layer, side, sl],
                p.biases[self._layer, side, sl])

    @property
    def keys(self):
        return self._side(0)

    @property
    def values(self):
        return self._side(1)

    @property
    def state(self):
        k, v = self.keys, self.values
        if self.offset == k[0].shape[2]:
            return k, v
        return tuple(x[..., :self.offset, :] for x in k), tuple(x[..., :self.offset, :] for x in v)

    @state.setter
    def state(self, v):
        """(keys, values) triples of one row; written into this layer's planes of the pool (grown if needed)"""
        k, vv = v
        n = int(k[0].shape[2])
        if self._pool is None:
            raise NotImplementedError("QuantizedKVCache.state: only pool-backed caches are assigned")
        self._pool.reserve(n, live_tokens=self.offset)
        for side, trip in ((0, k), (1, vv)):
            for dst, src in zip(self._side(side), trip):
                dst[..., :n, :].copy_(src.view(dst.dtype))
        self.offset = n

    @property
    def meta_state(self):
        return tuple(map(str, (self.offset, self.group_size, self.bits)))

    @meta_state.setter
    def meta_state(self, v):
        self.offset, self.group_size, self.bits = map(int, v)

    def is_trimmable(self):
        return True

    def trim(self, n):
        n = min(self.offset, n)
        self.offset -= n
        return n

    def size(self):
        return self.offset

    def make_mask(self, N: int, return_array: bool = False, window_size=None):
        return None if N == 1 else "causal"

    def empty(self):
        return self.keys is None

    @property
    def nbytes(self):
        k, v = self.keys, self.values
        if k is None:
            return 0
        return sum(x.numel() * x.element_size() for x in (*k, *v))


def make_prompt_cache(model: Any, max_kv_size: Optional[int] = None) -> List[Any]:
    """cache.py:45-70: defer to model.make_cache() when present."""
    if max_kv_size is not None:
        raise NotImplementedError("RotatingKVCache (max_kv_size) is out of scope (SURVEY §2.1 #6)")
    if hasattr(model, "make_cache"):
        return model.make_cache()
    return [KVCache() for _ in range(len(model.layers))]


def create_causal_mask(N: int, offset: int = 0, window_size: Optional[int] = None,
                       left_padding=None) -> torch.Tensor:
    """Boolean (…, N, offset+N) mask, True = attend (reference cache.py:24-42): query i (absolute
    position offset+i) sees key j iff j <= offset+i, within `window_size` if given, and, per
    row, j >= left_padding[row]."""
    rinds = torch.arange(offset + N)
    linds = torch.arange(offset, offset + N) if offset else rinds
    linds, rinds = linds[:, None], rinds[None]
    mask = linds >= rinds
    if window_size is not None:
        mask = mask & (linds < rinds + window_size)
    if left_padding is not None:
        lp = torch.as_tensor(left_padding).reshape(-1, 1, 1, 1)
        mask = mask & (rinds >= lp)
    return mask


class BatchKVCache(_BaseCache):
    """Left-padded batch of KV rows (reference cache.py:972-1201): rows of different lengths are
    right-aligned at the shared write index `_idx`; `left_padding[b]` positions at the front of
    row b are dead, `offset[b] = _idx - left_padding[b]` is the row's real length.

    Host-side container with the reference's observable behaviour (merge / extract / filter /
    extend / trim / state); the CUDA engine decodes each row from its own `KVCache` pool
    (`generate_batch.BatchGenerator`), this class is the interchange format."""
    step = 256

    def __init__(self, left_padding: List[int]):
        self.keys: Optional[torch.Tensor] = None
        self.values: Optional[torch.Tensor] = None
        self.left_padding = torch.as_tensor(list(left_padding), dtype=torch.int64)
        self.offset = -self.left_padding.clone()
        self._idx = 0
        self._right_padding: Optional[torch.Tensor] = None

    # -- append ----------------------------------------------------------------
    def update_and_fetch(self, keys: torch.Tensor, values: torch.Tensor):
        L = keys.shape[2]
        start, end = self._idx, self._idx + L
        cap = 0 if self.keys is None else self.keys.shape[2]
        if end > cap:
            grow = ((L + self.step - 1) // self.step) * self.step
            B, H, _, Dk = keys.shape
            extra_k = torch.zeros((B, H, grow, Dk), dtype=keys.dtype, device=keys.device)
            extra_v = torch.zeros((B, H, grow, values.shape[3]), dtype=values.dtype, device=values.device)
            if self.keys is None:
                self.keys, self.values = extra_k, extra_v
            else:
                live_k = self.keys if start % self.step == 0 else self.keys[..., :start, :]
                live_v = self.values if start % self.step == 0 else self.values[..., :start, :]
                self.keys = torch.cat([live_k, extra_k], dim=2)
                self.values = torch.cat([live_v, extra_v], dim=2)
        self.keys[..., start:end, :] = keys
        self.values[..., start:end, :] = values
        self.offset = self.offset + L
        self._idx = end
        return self.keys[..., :end, :], self.values[..., :end, :]

    def prepare(self, *, left_padding=None, lengths=None, right_padding=None):
        if left_padding is not None:
            if self.keys is not None:
                raise ValueError("Left padding can only be added to an empty BatchKVCache")
            lp = torch.as_tensor(list(left_padding), dtype=torch.int64)
            self.left_padding = self.left_padding + lp
            self.offset = self.offset - lp
        if right_padding is not None and max(right_padding) > 0:
            self._right_padding = torch.as_tensor(list(right_padding), dtype=torch.int64)

    def finalize(self):
        """Turn right padding (rows shorter than the processed chunk) into left padding by
        rotating each row to the right by its padding."""
        if self._right_padding is None:
            return
        pad = self._right_padding
        n = self.keys.shape[2]
        idx = (torch.arange(n)[None, :] - pad[:, None]) % n           # (B, n)
        gather = idx[:, None, :, None]
        self.keys = torch.take_along_dim(self.keys, gather.to(self.keys.device), dim=2)
        self.values = torch.take_along_dim(self.values, gather.to(self.values.device), dim=2)
        self.offset = self.offset - pad
        self.left_padding = self.left_padding + pad
        self._right_padding = None

    # -- reference attribute surface ----------------------------------------------
    @property
    def state(self):
        k, v = self.keys, self.values
        if k is not None and self._idx < k.shape[2]:
            k, v = k[..., :self._idx, :], v[..., :self._idx, :]
        return k, v, self.offset, self.left_padding

    @state.setter
    def state(self, v):
        self.keys, self.values, self.offset, self.left_padding = v
        self._idx = self.keys.shape[2]

    def is_trimmable(self):
        return True

    def trim(self, n):
        n = min(self._idx, n)
        self._idx -= n
        self.offset = self.offset - n
        return n

    def make_mask(self, N: int, return_array: bool = False, **kwargs):
        return create_causal_mask(N, offset=self._idx, left_padding=self.left_padding, **kwargs)

    def filter(self, batch_indices):
        """Keep the given rows (in place); drop the padding no remaining row needs."""
        sel = torch.as_tensor(batch_indices, dtype=torch.int64).reshape(-1)
        if self.keys is not None:
            self.keys = self.keys[sel.to(self.keys.device)]
            self.values = self.values[sel.to(self.values.device)]
        self.offset = self.offset[sel]
        self.left_padding = self.left_padding[sel]
        if self._right_padding is not None:
            self._right_padding = self._right_padding[sel]
        shift = int(self.left_padding.min()) if self.left_padding.numel() else 0
        if shift > 0:
            if self.keys is not None:
                self.keys = self.keys[..., shift:, :]
                self.values = self.values[..., shift:, :]
            self._idx -= shift
            self.left_padding = self.left_padding - shift

    def extend(self, other: "BatchKVCache"):
        """Append the rows of `other` (in place): both are right-aligned at the larger write index."""
        if self.keys is None and other.keys is None:
            self.left_padding = torch.cat([self.left_padding, other.left_padding])
            self.offset = torch.cat([self.offset, other.offset])
            return
        ref = self.keys if self.keys is not None else other.keys
        refv = self.values if self.values is not None else other.values
        H, Dk, Dv = ref.shape[1], ref.shape[3], refv.shape[3]
        new_idx = max(self._idx, other._idx)
        size = max(0 if c.keys is None else c.keys.shape[2] for c in (self, other))

        def aligned(c):
            rows = int(c.offset.shape[0])
            k = c.keys if c.keys is not None else torch.zeros((rows, H, 0, Dk), dtype=ref.dtype, device=ref.device)
            v = c.values if c.values is not None else torch.zeros((rows, H, 0, Dv), dtype=refv.dtype, device=refv.device)
            left = new_idx - c._idx
            right = size - k.shape[2] - left
            if right < 0:
                k, v = k[..., :right, :], v[..., :right, :]
                right = 0
            if left or right:
                k = torch.nn.functional.pad(k, (0, 0, left, right))
                v = torch.nn.functional.pad(v, (0, 0, left, right))
            return k, v, c.offset, c.left_padding + left

        ka, va, oa, la = aligned(self)
        kb, vb, ob, lb = aligned(other)
        self.keys, self.values = torch.cat([ka, kb]), torch.cat([va, vb])
        self.offset, self.left_padding = torch.cat([oa, ob]), torch.cat([la, lb])
        self._idx = new_idx

    def extract(self, idx: int) -> "KVCache":
        pad = int(self.left_padding[idx])
        out = KVCache()
        out.update_and_fetch(self.keys[idx:idx + 1, :, pad:self._idx].contiguous(),
                             self.values[idx:idx + 1, :, pad:self._idx].contiguous())
        return out

    @classmethod
    def merge(cls, caches: List["KVCache"]) -> "BatchKVCache":
        lengths = [int(c.size()) for c in caches]
        longest = max(lengths)
        if longest == 0:
            return cls([0] * len(caches))
        padding = [longest - n for n in lengths]
        src = next(c for c in caches if c.keys is not None)
        H, Dk, Dv = src.keys.shape[1], src.keys.shape[3], src.values.shape[3]
        keys = torch.zeros((len(caches), H, longest, Dk), dtype=src.keys.dtype, device=src.keys.device)
        values = torch.zeros((len(caches), H, longest, Dv), dtype=src.values.dtype, device=src.values.device)
        for b, (pad, c, n) in enumerate(zip(padding, caches, lengths)):
            if c.keys is None or n == 0:
                continue
            keys[b, :, pad:pad + n] = c.keys[0, :, :n]
            values[b, :, pad:pad + n] = c.values[0, :, :n]
        out = cls(padding)
        out.keys, out.values = keys, values
        out.offset = out.offset + longest
        out._idx = longest
        return out

    def size(self):
        return self._idx

    def empty(self):
        return self.keys is None

    @property
    def batch_size(self) -> int:
        return int(self.keys.shape[0]) if self.keys is not None else int(self.left_padding.shape[0])

    def is_single_row(self) -> bool:
        return self.batch_size == 1

    @property
    def nbytes(self):
        if self.keys is None:
            return 0
        return self.keys.numel() * self.keys.element_size() + self.values.numel() * self.values.element_size()


# ------------------------------------------------------------------------------------------------
# Device-resident batch cache of the lock-step decoder (csrc/decode_batch.cu)
# ------------------------------------------------------------------------------------------------
class BatchRows:
    """Row bookkeeping of ONE batched device pool (layers, 2, rows, kv heads, capacity, head_dim)
    shared by the per-layer `RowBatchKVCache` views.  Row b of the logical batch is row b of the
    pool (live rows are kept compact); every row has its own length — there is no left padding
    and no common write index, the kernels read the per-row lengths from device arrays.

    `filter / extend / extract / trim` are the reference's BatchKVCache operations
    (cache.py:1077-1201) as row copies inside / between pools (`b200_kv_copy_row`)."""

    def __init__(self, pool: KVPool, engine, lengths: Optional[List[int]] = None):
        self.pool = pool
        self.eng = engine
        self.lengths: List[int] = list(lengths or [])
        self.version = 0   # bumped by every structural change (the decoder re-arms its rows)

    @property
    def B(self) -> int:
        return len(self.lengths)

    def _touch(self):
        self.version += 1

    def ensure(self, rows: int, tokens: int):
        """room for `rows` rows of `tokens` positions (re-allocates and copies the live part)"""
        p = self.pool
        if rows > p.batch:
            if isinstance(p, BatchKVQPool):
                new = p.like(rows, max(p.capacity, tokens))
            else:
                new = KVPool(p.n_layers, p.n_kv, p.hd, p.device, batch=rows, capacity=max(p.capacity, tokens),
                             dtype=p.dtype)
            with torch.cuda.stream(self.eng.stream):
                for b, n in enumerate(self.lengths):
                    self.eng.kv_copy_row(new, b, p, b, n)
            new.generation = p.generation + 1
            self.pool.__dict__.update(new.__dict__)
            self._touch()
        elif tokens > p.capacity:
            self.eng.stream.synchronize()
            with torch.cuda.stream(self.eng.stream):
                p.reserve(tokens, live_tokens=max(self.lengths) if self.lengths else 0)
            self._touch()

    def filter(self, keep):
        keep = [int(i) for i in keep]
        assert keep == sorted(keep) and len(set(keep)) == len(keep), "filter: ascending unique row indices"
        for new_i, old_i in enumerate(keep):
            if new_i != old_i:
                self.eng.kv_copy_row(self.pool, new_i, self.pool, old_i, self.lengths[old_i])
        self.lengths = [self.lengths[i] for i in keep]
        self._touch()

    def extend(self, other: "BatchRows"):
        n = max(self.lengths + other.lengths + [0])
        self.ensure(self.B + other.B, n)
        for b, ln in enumerate(other.lengths):
            self.eng.kv_copy_row(self.pool, self.B + b, other.pool, b, ln)
        self.lengths = self.lengths + list(other.lengths)
        self._touch()

    def append_row(self, src_pool: KVPool, src_row: int, length: int) -> int:
        self.ensure(self.B + 1, max(self.lengths + [length]))
        self.eng.kv_copy_row(self.pool, self.B, src_pool, src_row, length)
        self.lengths.append(int(length))
        self._touch()
        return self.B - 1

    def trim(self, n: int) -> int:
        n = min([n] + self.lengths) if self.lengths else 0
        self.lengths = [ln - n for ln in self.lengths]
        self._touch()
        return n

    def layer_caches(self) -> list:
        p = self.pool
        if isinstance(p, BatchKVQPool):   # the batch rule: BatchQuantizedKVCache where the layer is 8-bit
            return ([BatchQuantizedKVCache(self, l) for l in range(p.n_q)] +
                    [RowBatchKVCache(self, l) for l in range(p.n_q, p.n_layers)])
        return [RowBatchKVCache(self, l) for l in range(p.n_layers)]

    def key(self) -> tuple:
        """identifies the device allocation behind the rows (changes whenever it moves)"""
        p = self.pool
        if isinstance(p, BatchKVQPool):
            return (p.q.codes.data_ptr() if p.q.codes is not None else 0, p.capacity)
        return (p.buf.data_ptr() if p.buf is not None else 0,)


class RowBatchKVCache(_BaseCache):
    """One layer's view of a `BatchRows` pool with the reference batch-cache surface
    (`offset`, `keys`, `values`, `state`, `filter`, `extend`, `extract`, `trim`, `merge`, `size`,
    `empty`, `nbytes`).  The pool is shared by all layers, so the structural operations act on the
    WHOLE pool when invoked on layer 0 and are no-ops on the other layers (the reference calls them
    on every layer's object in a loop; the net effect is the same)."""

    def __init__(self, rows: BatchRows, layer: int):
        self._rows = rows
        self._layer = layer

    @property
    def offset(self):
        import numpy as np
        return np.asarray(self._rows.lengths, dtype=np.int64)

    @property
    def left_padding(self):
        import numpy as np
        return np.zeros(self._rows.B, dtype=np.int64)

    def _planes(self):
        p = self._rows.pool
        return p.bf.buf[self._layer - p.n_q] if isinstance(p, BatchKVQPool) else p.buf[self._layer]

    @property
    def keys(self):
        return self._planes()[0][:self._rows.B]

    @property
    def values(self):
        return self._planes()[1][:self._rows.B]

    @property
    def state(self):
        n = self.size()
        return self.keys[..., :n, :], self.values[..., :n, :], self.offset, self.left_padding

    def size(self):
        return max(self._rows.lengths) if self._rows.lengths else 0

    def empty(self):
        return self._rows.B == 0

    def is_trimmable(self):
        return True

    @property
    def batch_size(self) -> int:
        return self._rows.B

    def trim(self, n):
        if self._layer == 0:
            self._trimmed = self._rows.trim(n)
            return self._trimmed
        return min([n] + [ln + n for ln in self._rows.lengths]) if self._rows.lengths else 0

    def filter(self, batch_indices):
        if self._layer == 0:
            idx = batch_indices.tolist() if hasattr(batch_indices, "tolist") else list(batch_indices)
            self._rows.filter(idx)

    def extend(self, other: "RowBatchKVCache"):
        if self._layer == 0:
            self._rows.extend(other._rows)

    def extract(self, idx: int) -> KVCache:
        """row `idx` as a standalone single-request KVCache of this layer (a copy)"""
        n = self._rows.lengths[idx]
        out = KVCache()
        out.update_and_fetch(self.keys[idx:idx + 1, :, :n].clone(), self.values[idx:idx + 1, :, :n].clone())
        return out

    def make_mask(self, N: int, return_array: bool = False, **kwargs):
        return None if N == 1 else "causal"   # per-row lengths are applied by the kernels

    @property
    def nbytes(self):
        k = self.keys
        return 2 * k.numel() * k.element_size()

    @classmethod
    def merge(cls, caches: List[KVCache], engine=None, rows: Optional[BatchRows] = None):
        """Batch cache from single-request caches (cache.py:1180-1201).  `caches` are this layer's
        pool-backed KVCache objects of the requests; the rows of ALL layers are copied when the
        layer-0 caches are merged (one shared pool).  Returns this layer's view."""
        c0 = caches[0]
        if rows is None:
            assert c0._pool is not None and engine is not None, "merge needs pool-backed caches and the engine"
            p = c0._pool
            cap = max(int(c.offset) for c in caches)
            pool = KVPool(p.n_layers, p.n_kv, p.hd, p.device, batch=max(len(caches), 1), capacity=max(cap, 1),
                          dtype=p.dtype)
            rows = BatchRows(pool, engine)
            with torch.cuda.stream(engine.stream):
                for c in caches:
                    rows.append_row(c._pool, c._row or 0, int(c.offset))
        return cls(rows, c0._layer)


class BatchQuantizedKVCache(_BaseCache):
    """One 8-bit layer's view of a `BatchRows` over a `BatchKVQPool`, with the reference's observable surface
    (models/cache.py:1747-1960): `keys` / `values` are (codes as uint32 (B, n_kv, S, head_dim / 4), scales, biases)
    in mx.quantize's packing, `offset` the per-row lengths, `left_padding` zeros (rows here are not padded).  Rows
    sit on the pool rows exactly as for `RowBatchKVCache`; `filter` / `extend` act on the whole pool from layer 0 and
    move every plane byte for byte.  `extract` returns a single-request `QuantizedKVCache`."""

    def __init__(self, rows: BatchRows, layer: int):
        self._rows = rows
        self._layer = layer
        self.bits = 8

    @property
    def group_size(self) -> int:
        return self._rows.pool.group_size

    @property
    def offset(self):
        import numpy as np
        return np.asarray(self._rows.lengths, dtype=np.int64)

    @property
    def left_padding(self):
        import numpy as np
        return np.zeros(self._rows.B, dtype=np.int64)

    def _side(self, side: int):
        q = self._rows.pool.q
        B = self._rows.B
        return (q.codes[self._layer, side, :B].view(torch.uint32), q.scales[self._layer, side, :B],
                q.biases[self._layer, side, :B])

    @property
    def keys(self):
        return self._side(0)

    @property
    def values(self):
        return self._side(1)

    @property
    def state(self):
        n = self.size()
        k, v = self.keys, self.values
        return (tuple(x[..., :n, :] for x in k), tuple(x[..., :n, :] for x in v), self.offset, self.left_padding)

    def size(self):
        return max(self._rows.lengths) if self._rows.lengths else 0

    def empty(self):
        return self._rows.B == 0

    def is_trimmable(self):
        return True

    @property
    def batch_size(self) -> int:
        return self._rows.B

    def trim(self, n):
        if self._layer == 0:
            return self._rows.trim(n)
        return min([n] + [ln + n for ln in self._rows.lengths]) if self._rows.lengths else 0

    def filter(self, batch_indices):
        if self._layer == 0:
            idx = batch_indices.tolist() if hasattr(batch_indices, "tolist") else list(batch_indices)
            self._rows.filter(idx)

    def extend(self, other: "BatchQuantizedKVCache"):
        if self._layer == 0:
            self._rows.extend(other._rows)

    def extract(self, idx: int) -> QuantizedKVCache:
        """row `idx` as a single-request QuantizedKVCache of this layer (a byte copy of its first offset[idx]
        positions).  The reference calls extract on every layer in turn; as the layers of a request share one pool
        here, the extract of layer 0 copies the row's 8-bit layers into a FRESH single-request pool and the extracts
        of the other 8-bit layers of that same sweep (same rows state, row and length) view it.  Every sweep gets its
        own pool, so caches extracted twice never share storage."""
        rows = self._rows
        key = (rows.version, rows.key(), idx, rows.lengths[idx])
        cached = getattr(rows, "_extracted", None)
        if self._layer == 0 or cached is None or cached[0] != key or self._layer in cached[2]:
            bp, n = rows.pool, rows.lengths[idx]
            one = QuantizedKVPool(bp.n_q, bp.n_kv, bp.hd, bp.device, group_size=bp.group_size, batch=1,
                                  capacity=max(n, 1), stream=rows.eng.stream)
            with torch.cuda.stream(rows.eng.stream) if rows.eng.stream is not None else nullcontext():
                rows.eng.kvq_copy_row(one, 0, bp.q, idx, n)
            cached = (key, one, set())
            rows._extracted = cached
        cached[2].add(self._layer)
        out = QuantizedKVCache(self.group_size, 8, pool=cached[1], layer=self._layer)
        out.offset = rows.lengths[idx]
        return out

    def make_mask(self, N: int, return_array: bool = False, **kwargs):
        return None if N == 1 else "causal"

    @property
    def nbytes(self):
        return sum(x.numel() * x.element_size() for x in (*self.keys, *self.values))
