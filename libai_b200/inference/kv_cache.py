"""Preallocated KV cache for incremental decoding.

``StaticKVCache`` keeps one K and one V buffer ``[batch, heads, capacity, head_dim]`` per layer this pipeline stage owns
(``heads`` = the key/value heads, fewer than the query heads under grouped-query attention; under tensor parallelism the
rank's local ones).  New tokens are written in place at rows ``seqlens[b] + i``
(:func:`libai_b200.ops.functional.kv_cache_append`) and the decode attention reads the buffers directly, so a decoding
step copies nothing but the new rows.  ``seqlens`` and ``kv_start`` (the left padding of each sample) are int32 device
tensors read inside the kernels; ``length`` is their host-side mirror (every sample holds the same number of rows, the
left padding included), which sizes the windows and decides when the buffers must grow.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Tuple

import torch

from libai_b200.utils import distributed as dutil


def left_padding(attention_mask: torch.Tensor) -> Optional[torch.Tensor]:
    """``kv_start`` (int32 ``[b]``, the number of leading zeros) of a 2-D padding mask whose rows are "zeros, then ones"
    with at least one one; None for any other mask.  One small host sync."""
    m = attention_mask.to(torch.int8)
    if m.shape[1] > 1 and not bool((m[:, 1:] >= m[:, :-1]).all()):
        return None
    if not bool((m[:, -1] == 1).all()):
        return None
    return (m.shape[1] - m.to(torch.int32).sum(dim=1)).to(torch.int32)


def padding_window(attention_mask: torch.Tensor) -> Optional[Tuple[torch.Tensor, torch.Tensor]]:
    """``(kv_start, kv_end)`` (int32 ``[b]``) of a 2-D padding mask whose rows are each one run of ones — "ones, then
    zeros" (right padding), "zeros, then ones" (left padding) or all ones: the keys ``kv_start[b] <= j < kv_end[b]``.
    None for any other mask (a row with a hole, or without a one).  One small host sync."""
    m = attention_mask.to(torch.int32)
    n = m.shape[1]
    j = torch.arange(n, dtype=torch.int32, device=m.device)[None, :]
    ones = m.sum(dim=1, dtype=torch.int32)
    start = torch.where(m > 0, j, n).amin(dim=1)
    end = torch.where(m > 0, j + 1, 0).amax(dim=1)
    if not bool(((m == 0) | (m == 1)).all() & (ones > 0).all() & (end - start == ones).all()):
        return None
    return start.to(torch.int32), end.to(torch.int32)


class KVCacheLayer:
    """The cache of one layer, handed to its attention module in place of the ``(key, value)`` tuple."""

    __slots__ = ("cache", "idx")

    def __init__(self, cache: "StaticKVCache", idx: int):
        self.cache, self.idx = cache, idx

    @property
    def k(self) -> torch.Tensor:
        return self.cache.k[self.idx]

    @property
    def v(self) -> torch.Tensor:
        return self.cache.v[self.idx]

    @property
    def seqlens(self) -> torch.Tensor:
        return self.cache.seqlens

    @property
    def kv_start(self) -> torch.Tensor:
        return self.cache.kv_start

    @property
    def length(self) -> int:
        return self.cache.length


class StaticKVCache:
    def __init__(self, num_layers: int, batch: int, heads: int, head_dim: int, capacity: int,
                 dtype=torch.bfloat16, device=None, layers: Optional[Iterable[int]] = None):
        self.num_layers, self.batch, self.heads, self.head_dim = num_layers, batch, heads, head_dim
        self.dtype, self.device = dtype, torch.device(device) if device is not None else torch.device("cpu")
        self.owned = sorted(range(num_layers) if layers is None else layers)
        self.capacity = max(int(capacity), 1)
        self.k: List[Optional[torch.Tensor]] = [None] * num_layers
        self.v: List[Optional[torch.Tensor]] = [None] * num_layers
        for i in self.owned:
            self.k[i], self.v[i] = self._buffer(self.capacity), self._buffer(self.capacity)
        self.seqlens = torch.zeros(batch, dtype=torch.int32, device=self.device)
        self.kv_start = torch.zeros(batch, dtype=torch.int32, device=self.device)
        self.length = 0
        self.dense_mask = False   # the cached prompt's padding is not "zeros, then ones": kv_start cannot carry it

    def _buffer(self, capacity):
        # uninitialised: the attention reads rows below the current length only (the decode kernel repeats the last
        # row of the window to fill its last tile), and every such row has been written by an append
        return torch.empty(self.batch, self.heads, capacity, self.head_dim, dtype=self.dtype, device=self.device)

    def layer(self, i: int) -> KVCacheLayer:
        return KVCacheLayer(self, i)

    def matches(self, batch: int, dtype, device) -> bool:
        return self.batch == batch and self.dtype == dtype and self.device == torch.device(device)

    def reserve(self, n: int) -> None:
        """Make room for ``n`` more rows: the buffers are reallocated at twice their capacity (or more, when needed) and
        the held rows copied over."""
        need = self.length + n
        if need <= self.capacity:
            return
        cap = max(2 * self.capacity, need)
        for i in self.owned:
            for bufs in (self.k, self.v):
                new = self._buffer(cap)
                new[:, :, : self.length] = bufs[i][:, :, : self.length]
                bufs[i] = new
        self.capacity = cap

    def advance(self, n: int) -> None:
        """Count ``n`` appended rows (on the device in place, and in the host mirror)."""
        self.seqlens.add_(n)
        self.length += n

    def reorder_(self, beam_idx: torch.Tensor) -> None:
        """Gather the samples along the batch dimension in place (beam search)."""
        idx = beam_idx.to(device=self.device, dtype=torch.long)
        L = self.length
        for i in self.owned:
            for buf in (self.k[i], self.v[i]):
                buf[:, :, :L] = buf[:, :, :L].index_select(0, idx)
        self.seqlens.copy_(self.seqlens.index_select(0, idx))
        self.kv_start.copy_(self.kv_start.index_select(0, idx))

    def reset(self) -> None:
        self.seqlens.zero_()
        self.kv_start.zero_()
        self.length = 0
        self.dense_mask = False


class KVCacheOwner:
    """The model side of a :class:`StaticKVCache` for decoder-only models: ``generate`` sizes it through
    ``allocate_kv_cache``, ``set_cache`` / ``past_key_values`` / ``past_length`` keep the generator's cache protocol.
    The model lists its self-attention modules (``query_key_value``, ``head_size``, and ``local_kv_heads`` — the rank's
    key/value heads — or, for modules without grouped-query attention, ``local_heads``)."""

    kv_cache: Optional[StaticKVCache] = None
    past_length = 0

    def _cache_attention_modules(self) -> list:
        raise NotImplementedError

    @property
    def past_key_values(self):
        return self.kv_cache

    def allocate_kv_cache(self, batch: int, max_length: int) -> StaticKVCache:
        """Size the cache for ``batch`` sequences of up to ``max_length`` tokens (``generate`` calls this before the
        first step); an existing cache of that batch that is large enough is reused."""
        mods = self._cache_attention_modules()
        topo = dutil.get_dist_util()
        owned = [i for i in range(len(mods)) if topo.owns_layer(i)]   # this pipeline stage's layers
        w = mods[0].query_key_value.weight
        c = self.kv_cache
        if c is None or not c.matches(batch, w.dtype, w.device) or c.capacity < max_length:
            heads = getattr(mods[0], "local_kv_heads", mods[0].local_heads)
            c = StaticKVCache(len(mods), batch, heads, mods[0].head_size, max_length, w.dtype, w.device, owned)
        c.reset()
        self.kv_cache, self.past_length = c, 0
        return c

    def _prepare_cache(self, input_ids, max_positions: Optional[int] = None) -> StaticKVCache:
        """The cache for this step's ``input_ids`` ``[b, s]``: allocated for a new batch, grown to fit ``s`` more rows."""
        bsz, s_len = input_ids.shape
        c = self.kv_cache
        if c is None or (c.length == 0 and c.batch != bsz):
            c = self.allocate_kv_cache(bsz, s_len)
        if max_positions is not None and c.length + s_len > max_positions:
            raise ValueError(f"The maximum supported length is {max_positions}, "
                             f"and the current length is {c.length + s_len}.")
        c.reserve(s_len)
        return c

    def set_cache(self, past_key_values):
        """``None`` empties the cache (its buffers are kept); a :class:`StaticKVCache` becomes the model's cache."""
        if past_key_values is None:
            if self.kv_cache is not None:
                self.kv_cache.reset()
        else:
            assert isinstance(past_key_values, StaticKVCache), "set_cache expects a StaticKVCache"
            self.kv_cache = past_key_values
        self.past_length = 0 if self.kv_cache is None else self.kv_cache.length
