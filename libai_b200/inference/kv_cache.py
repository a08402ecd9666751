"""Preallocated KV cache for incremental decoding.

``StaticKVCache`` keeps one K and one V buffer ``[batch, heads, capacity, head_dim]`` per layer this pipeline stage owns
(``heads`` = the key/value heads, fewer than the query heads under grouped-query attention; under tensor parallelism the
rank's local ones).  New tokens are written in place at rows ``seqlens[b] + i``
(:func:`libai_b200.ops.functional.kv_cache_append`) and the decode attention reads the buffers directly, so a decoding
step copies nothing but the new rows.  ``seqlens`` and ``kv_start`` (the left padding of each sample) are int32 device
tensors read inside the kernels; ``length`` is their host-side mirror (every sample holds the same number of rows, the
left padding included), which sizes the windows and decides when the buffers must grow.

With ``kv_dtype=torch.float8_e4m3fn`` the K and V buffers hold E4M3 bytes and each row has an fp32 scale,
``k_scale`` / ``v_scale`` ``[batch, heads, capacity]`` (the format of :func:`OF.kv_cache_quantize_ref`): about half the
bytes of a bf16 cache, at the accuracy of a per-row 8-bit float.  Every attention over such a cache is the attention
over its dequantized rows.  It is a user's choice (``generate(kv_cache_dtype="fp8")``), never made for them.

``PagedKVCache`` holds the same logical rows in pages of 64 (``generate(paged_kv_cache=True)``): the sequences of one
prompt (beams, or ``num_return_sequences`` samples) share its prompt's pages, and a beam reorder rewrites block tables
instead of copying the cache.
"""
from __future__ import annotations

import logging
from typing import Iterable, List, Optional, Tuple

import torch

from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dutil

logger = logging.getLogger(__name__)


def left_padding(attention_mask: torch.Tensor) -> Optional[torch.Tensor]:
    """``kv_start`` (int32 ``[b]``, the number of leading zeros) of a 2-D padding mask whose rows are "zeros, then ones"
    with at least one one; None for any other mask.  One small host sync."""
    m = attention_mask.to(torch.int8)
    if m.shape[1] > 1 and not bool((m[:, 1:] >= m[:, :-1]).all()):
        return None
    if not bool((m[:, -1] == 1).all()):
        return None
    return (m.shape[1] - m.to(torch.int32).sum(dim=1)).to(torch.int32)


def _ones_runs(attention_mask: torch.Tensor):
    """On the device, for a 2-D padding mask: whether it is 0/1, and per row the index of the first one, one past the
    last one, and the number of ones (int32 ``[b]``; a row without a one has ``start = n``, ``end = 0``)."""
    m = attention_mask.to(torch.int32)
    n = m.shape[1]
    j = torch.arange(n, dtype=torch.int32, device=m.device)[None, :]
    ones = m.sum(dim=1, dtype=torch.int32)
    start = torch.where(m > 0, j, n).amin(dim=1)
    end = torch.where(m > 0, j + 1, 0).amax(dim=1)
    return ((m == 0) | (m == 1)).all(), start, end, ones


def padding_window(attention_mask: torch.Tensor) -> Optional[Tuple[torch.Tensor, torch.Tensor]]:
    """``(kv_start, kv_end)`` (int32 ``[b]``) of a 2-D padding mask whose rows are each one run of ones — "ones, then
    zeros" (right padding), "zeros, then ones" (left padding) or all ones: the keys ``kv_start[b] <= j < kv_end[b]``.
    None for any other mask (a row with a hole, or without a one).  One small host sync."""
    binary, start, end, ones = _ones_runs(attention_mask)
    if not bool(binary & (ones > 0).all() & (end - start == ones).all()):
        return None
    return start.to(torch.int32), end.to(torch.int32)


def _padding_sides(attention_mask: torch.Tensor) -> Tuple[bool, bool, torch.Tensor, torch.Tensor]:
    """``(right, left, start, ones)`` of a 2-D 0/1 padding mask, with one small host sync: ``right`` when every row is
    "ones, then zeros" (all zeros included), ``left`` when every row is "zeros, then ones" with at least one one (an
    all-ones mask is both), and per row the index of the first one and the number of ones (int32 ``[b]``)."""
    binary, start, end, ones = _ones_runs(attention_mask)
    run = end - start == ones   # the row's ones are contiguous (never for a row without a one)
    right = binary & ((run & (start == 0)) | (ones == 0)).all()
    left = binary & (run & (end == attention_mask.shape[1])).all()
    right, left = torch.stack((right, left)).tolist()
    return right, left, start, ones


def padding_bounds(attention_mask: torch.Tensor) -> Optional[Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]]:
    """How the flash kernels take a padded 2-D mask without a dense one: ``(kv_lens, None)`` when every row is right
    padded ("ones, then zeros"; an all-zero row gets ``kv_lens = 0``, which the kernels clamp to 1), else
    ``(None, kv_start)`` when every row is left padded ("zeros, then ones"), both int32 ``[b]``; None for any other mask
    (a hole, padding on both sides, or left and right padded rows together).  One small host sync."""
    right, left, start, ones = _padding_sides(attention_mask)
    if right:
        return ones, None
    if left:
        return None, start
    return None


class PrefixIndex:
    """The prefix index of a paged cache: full pages of 64 rows kept after the sequences that wrote them, so that a later
    prompt starting with the same tokens maps them instead of computing their rows again.

    A full page is immutable once written, so rows with the same key hold the same K/V for the same weights and cache
    format, whatever the call.  A page's key is its parent page (-1 for the first) and the (token id, mask) of its 64
    rows.  The index holds one reference per page: the cache that owns the pool counts it, and takes it back for the
    pages :meth:`evict` and :meth:`clear` return.  Eviction takes the least-recently-used leaf (a page no cached page
    continues), so a cached chain is always a prefix of what was inserted."""

    def __init__(self):
        self.pages = {}      # (parent page or -1, ((token, mask), ... 64)) -> page
        self.keys = {}       # cached page -> its key
        self.children = {}   # cached page -> the number of cached pages that continue it
        self.used = {}       # cached page -> the tick it was last looked up or inserted at
        self.tick = 0

    def __len__(self) -> int:
        return len(self.keys)

    def __contains__(self, page: int) -> bool:
        return page in self.keys

    @staticmethod
    def page_keys(ids: List[int], mask: List[int], pages: int):
        P = OF.PAGE_ROWS
        return [tuple(zip(ids[j * P : (j + 1) * P], mask[j * P : (j + 1) * P])) for j in range(pages)]

    def chain(self, keys) -> List[int]:
        """The cached pages of the longest run of ``keys`` (from the first page on) the index holds."""
        parent, chain = -1, []
        for key in keys:
            page = self.pages.get((parent, key))
            if page is None:
                break
            chain.append(page)
            parent = page
        return chain

    def touch(self, pages: Iterable[int]) -> None:
        """Mark ``pages`` used now (one tick for all of them)."""
        self.tick += 1
        for page in pages:
            self.used[page] = self.tick

    def insert(self, rows) -> List[int]:
        """Index the pages of ``rows``, pairs ``(keys, table_row)``: page ``j`` of a row, under ``keys[j]``, is
        ``table_row[j]`` unless the index holds that key already.  One tick for all rows.  Returns the pages added,
        each of which the index now holds a reference to."""
        self.tick += 1
        added = []
        for keys, table_row in rows:
            parent = -1
            for j, key in enumerate(keys):
                page = self.pages.get((parent, key))
                if page is None:
                    page = table_row[j]
                    if page in self.keys:   # cached under another key: cannot happen for an immutable page
                        break
                    self.pages[(parent, key)], self.keys[page] = page, (parent, key)
                    self.children[page] = 0
                    if parent >= 0:
                        self.children[parent] += 1
                    added.append(page)
                self.used[page] = self.tick
                parent = page
        return added

    def pop_leaf(self, evictable=None) -> Optional[int]:
        """Drop the least-recently-used leaf (among those ``evictable(page)`` accepts) and return it, or None."""
        leaves = [p for p, n in self.children.items() if n == 0 and (evictable is None or evictable(p))]
        if not leaves:
            return None
        leaf = min(leaves, key=lambda p: self.used[p])
        parent, key = self.keys.pop(leaf)
        del self.pages[(parent, key)]
        del self.children[leaf]
        if parent >= 0:
            self.children[parent] -= 1
        return leaf

    def evict(self, budget: int) -> List[int]:
        """Drop least-recently-used leaves down to ``budget`` pages; returns them."""
        out = []
        while len(self.keys) > budget:
            out.append(self.pop_leaf())
        return out

    def clear(self) -> List[int]:
        """Drop every page; returns them."""
        out = list(self.keys)
        self.pages, self.keys, self.children = {}, {}, {}
        return out


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
    def k_scale(self) -> Optional[torch.Tensor]:
        return self.cache.k_scale[self.idx]

    @property
    def v_scale(self) -> Optional[torch.Tensor]:
        return self.cache.v_scale[self.idx]

    @property
    def seqlens(self) -> torch.Tensor:
        return self.cache.seqlens

    @property
    def kv_start(self) -> torch.Tensor:
        return self.cache.kv_start

    @property
    def length(self) -> int:
        return self.cache.length

    @property
    def pages(self) -> dict:
        """The block table of a paged cache's kernels ({} for contiguous buffers)."""
        return {}

    def append(self, qkv: torch.Tensor, cos=None, sin=None) -> torch.Tensor:
        """Write k, v of the packed projection ``qkv`` (per-head ``[b, s, a, 3d]`` or grouped ``[b, s, g, r + 2, d]``) at
        rows ``seqlens[b] + i`` (:func:`OF.kv_cache_append`, rotated by ``cos/sin`` when given); returns q ``[b, s, a,
        d]``.  A per-head projection without rotary hands q back as its strided view: nothing needs writing."""
        scales = {} if self.k_scale is None else {"k_scale": self.k_scale, "v_scale": self.v_scale}
        if cos is None and qkv.dim() == 4:
            OF.kv_cache_append(qkv, self.k, self.v, self.seqlens, return_q=False, **scales, **self.pages)
            return qkv[..., : qkv.shape[-1] // 3]
        return OF.kv_cache_append(qkv, self.k, self.v, self.seqlens, cos, sin, **scales, **self.pages)

    def window(self, L: int, dtype) -> Tuple[torch.Tensor, torch.Tensor]:
        """K and V rows ``[:L]``: views of the buffers, or of an FP8 cache its rows dequantized to ``dtype``."""
        if self.k_scale is None:
            return self.k[:, :, :L], self.v[:, :, :L]
        return (OF.kv_cache_dequant(self.k[:, :, :L], self.k_scale[:, :, :L], dtype),
                OF.kv_cache_dequant(self.v[:, :, :L], self.v_scale[:, :, :L], dtype))

    def attend(self, q: torch.Tensor, *, scale: float, causal: bool = True, mask=None, bias=None, alibi_slopes=None,
               rel_bias=None, dropout_p: float = 0.0, training: bool = False, prefix_lens=None) -> torch.Tensor:
        """Attention of the new tokens' ``q`` ``[b, s, a, d]`` over the cache → ``[b, s, a, d]``, contiguous.
        ``causal``: the new tokens were appended this step (self-attention); ``causal=False``: the cache is a fixed
        window the queries all see (cross-attention).  The rows held before this step (``length``) are the same for
        every layer: the model advances the cache after its last layer.

        - a dense 0/1 ``mask`` or additive ``bias`` (the model folded its padding into it): :func:`OF.attention` over
          the window ``[:length + s]`` (causal) or ``[:length]``, non-causal;
        - the causal prefill of an empty cache without ``rel_bias``: the flash kernel over ``[:s]``, the prompt's left
          padding in ``kv_start``; ``prefix_lens`` (int32 ``[b]``, a prefix LM's context width) makes the first
          ``prefix_lens[b]`` rows visible to every new token.  Only this branch takes a prefix: every cached row is
          visible to a later token, so later steps need none, and any other call with ``prefix_lens`` raises
          ``ValueError``;
        - anything else: :func:`OF.decode_attention` (the split-KV kernel up to 16 new tokens, the flash kernel over
          the cache window beyond).

        The first two read an FP8 cache's window dequantized to q's dtype; the decode kernel reads its bytes."""
        past = self.length
        if prefix_lens is not None and (past > 0 or not causal or mask is not None or bias is not None
                                        or alibi_slopes is not None or rel_bias is not None):
            raise ValueError("prefix_lens: only the causal prefill of an empty cache, without mask, bias, ALiBi or "
                             "rel_bias, takes a prefix")
        if mask is not None or bias is not None:
            L = past + q.shape[1] if causal else past
            k, v = self.window(L, q.dtype)
            ctx = OF.attention(q.transpose(1, 2), k, v, causal=False, scale=scale, mask=mask, bias=bias,
                               dropout_p=dropout_p, training=training)
            return ctx.transpose(1, 2).contiguous()   # the reference math's [b, a, s, d] output is not
        if causal and past == 0 and rel_bias is None:
            query, (key, value) = q.transpose(1, 2), self.window(q.shape[1], q.dtype)
            kv_start = self.kv_start if prefix_lens is not None or OF.attention_supported(query, key) else None
            ctx = OF.attention(query, key, value, causal=True, scale=scale, alibi_slopes=alibi_slopes,
                               kv_start=kv_start, dropout_p=dropout_p, training=training, prefix_lens=prefix_lens)
            return ctx.transpose(1, 2)
        scales = {} if self.k_scale is None else {"k_scale": self.k_scale, "v_scale": self.v_scale}
        return OF.decode_attention(q, self.k, self.v, self.seqlens, self.kv_start, scale=scale, past=past,
                                   alibi_slopes=alibi_slopes, rel_bias=rel_bias, causal=causal, **scales, **self.pages)


class StaticKVCache:
    """``dtype``: the dtype of the projections the cache serves; ``kv_dtype``: what the buffers hold (default
    ``dtype``; ``torch.float8_e4m3fn``: E4M3 rows with fp32 row scales, the capacity then a multiple of 4)."""

    def __init__(self, num_layers: int, batch: int, heads: int, head_dim: int, capacity: int,
                 dtype=torch.bfloat16, device=None, layers: Optional[Iterable[int]] = None, kv_dtype=None):
        self.num_layers, self.batch, self.heads, self.head_dim = num_layers, batch, heads, head_dim
        self.dtype, self.device = dtype, torch.device(device) if device is not None else torch.device("cpu")
        self.kv_dtype = dtype if kv_dtype is None else kv_dtype
        if self.kv_dtype not in (dtype, torch.float8_e4m3fn):
            raise ValueError(f"kv_dtype must be the projections' {dtype} or torch.float8_e4m3fn, got {kv_dtype}")
        self.fp8 = self.kv_dtype == torch.float8_e4m3fn
        self.owned = sorted(range(num_layers) if layers is None else layers)
        self.capacity = self._rounded(max(int(capacity), 1))
        self.k: List[Optional[torch.Tensor]] = [None] * num_layers
        self.v: List[Optional[torch.Tensor]] = [None] * num_layers
        self.k_scale: List[Optional[torch.Tensor]] = [None] * num_layers   # FP8: the row scales
        self.v_scale: List[Optional[torch.Tensor]] = [None] * num_layers
        for i in self.owned:
            self.k[i], self.v[i] = self._buffer(self.capacity), self._buffer(self.capacity)
            if self.fp8:
                self.k_scale[i], self.v_scale[i] = self._scales(self.capacity), self._scales(self.capacity)
        self.seqlens = torch.zeros(batch, dtype=torch.int32, device=self.device)
        self.kv_start = torch.zeros(batch, dtype=torch.int32, device=self.device)
        self.length = 0
        self.dense_mask = False   # the cached prompt's padding is not "zeros, then ones": kv_start cannot carry it

    def _buffer(self, capacity):
        # uninitialised: the attention reads rows below the current length only (the decode kernel repeats the last
        # row of the window to fill its last tile; over an FP8 cache it zeroes them), and every such row has been
        # written by an append
        return torch.empty(self.batch, self.heads, capacity, self.head_dim, dtype=self.kv_dtype, device=self.device)

    def _scales(self, capacity):
        return torch.empty(self.batch, self.heads, capacity, dtype=torch.float32, device=self.device)

    def _rounded(self, capacity: int) -> int:
        # the decode kernel loads the scales of a tile from a 16-byte boundary of their row
        return -(-capacity // 4) * 4 if self.fp8 else capacity

    def layer(self, i: int) -> KVCacheLayer:
        return KVCacheLayer(self, i)

    def matches(self, batch: int, dtype, device, kv_dtype=None) -> bool:
        """Whether this cache serves ``batch`` sequences of ``dtype`` projections on ``device`` and holds ``kv_dtype``
        rows (default ``dtype``)."""
        return (self.batch == batch and self.dtype == dtype and self.device == torch.device(device)
                and self.kv_dtype == (dtype if kv_dtype is None else kv_dtype))

    def flash_attention(self) -> bool:
        """True when :func:`OF.attention` over the buffers (an FP8 cache's dequantized to ``dtype``) runs the flash
        kernels, which take a left-padded prompt's padding from ``kv_start``; the reference math needs a dense mask for
        it."""
        k = self.k[self.owned[0]]
        if self.fp8:
            k = torch.empty((self.batch, self.heads, 1, self.head_dim), dtype=self.dtype, device=self.device)
        return OF.attention_supported(k, k)

    def write_rows(self, i: int, k: torch.Tensor, v: torch.Tensor, row0: int = 0) -> None:
        """Write ``k``, ``v`` ``[batch, heads, n, head_dim]`` at rows ``row0 .. row0 + n`` of layer ``i`` (an FP8 cache
        quantizes them by :func:`OF.kv_cache_quantize_ref`).  The lengths are the caller's to advance."""
        n = k.shape[2]
        for buf, scale, x in ((self.k, self.k_scale, k), (self.v, self.v_scale, v)):
            if self.fp8:
                buf[i][:, :, row0 : row0 + n], scale[i][:, :, row0 : row0 + n] = OF.kv_cache_quantize_ref(x)
            else:
                buf[i][:, :, row0 : row0 + n] = x

    def step_needs_dense_mask(self, attention_mask: Optional[torch.Tensor], *, flash: bool,
                              kv_start_ok: bool = True) -> bool:
        """The padding policy of a decoder-only model's step, called once before its layers: True when the layers must
        take ``attention_mask`` (``[b, length + s]``, 1 = token) as a dense mask.  The prefill of an empty cache
        classifies the prompt's padding: a left-padded 2-D mask goes to ``kv_start`` (unless ``kv_start_ok`` is False,
        e.g. when rows precede the prompt), any other padding sets ``dense_mask`` for every later step; the prefill
        itself needs the dense mask for such padding, and for any padding when the attention is not ``flash``.  Later
        steps need it when ``dense_mask`` is set, without a host sync."""
        if self.length > 0:
            return attention_mask is not None and self.dense_mask
        if attention_mask is None:
            return False
        if attention_mask.dim() == 2:
            right, left, start, _ = _padding_sides(attention_mask)
            padded, in_kv_start = not (right and left), left and kv_start_ok
            if in_kv_start:
                self.kv_start.copy_(start)
        else:
            padded, in_kv_start = not bool(attention_mask.all()), False
        self.dense_mask = padded and not in_kv_start
        return padded and (self.dense_mask or not flash)

    def fill(self, kv: Iterable[Tuple[torch.Tensor, torch.Tensor]], S: int,
             window: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> None:
        """Hold a fixed window of ``S`` rows (e.g. the encoder projection a decoder cross-attends to): ``kv`` yields
        ``(k, v)`` ``[b, heads, S, d]`` of every layer, and each sample sees the rows ``kv_start[b] <= j < end[b]`` of
        ``window = (kv_start, end)`` (int32 ``[b]``), or all ``S``.  Read with ``attend(causal=False)``."""
        self.reset()
        if window is None:
            self.seqlens.fill_(S)
        else:
            self.kv_start.copy_(window[0])
            self.seqlens.copy_(window[1])
        self.length = S
        for i, (k, v) in enumerate(kv):
            self.write_rows(i, k, v)

    def reserve(self, n: int) -> None:
        """Make room for ``n`` more rows: the buffers are reallocated at twice their capacity (or more, when needed) and
        the held rows copied over."""
        need = self.length + n
        if need <= self.capacity:
            return
        cap = self._rounded(max(2 * self.capacity, need))
        for i in self.owned:
            for bufs, alloc in ((self.k, self._buffer), (self.v, self._buffer), (self.k_scale, self._scales),
                                (self.v_scale, self._scales)):
                if bufs[i] is None:
                    continue
                new = alloc(cap)
                new[:, :, : self.length] = bufs[i][:, :, : self.length]
                bufs[i] = new
        self.capacity = cap

    def advance(self, n: int) -> None:
        """Count ``n`` appended rows (on the device in place, and in the host mirror)."""
        self.seqlens.add_(n)
        self.length += n

    def rollback(self, n: int) -> None:
        """Drop the last ``n`` rows of every sample (on the device in place, and in the host mirror): a speculative
        verify step's rows past the accepted tokens.  Rows at or past ``seqlens`` are never read (an FP8 cache's
        included), so nothing is cleared; the next append overwrites them."""
        if not 0 <= n <= self.length:
            raise ValueError(f"rollback: 0 <= n <= length ({self.length}), got {n}")
        if n:
            self.seqlens.sub_(n)
            self.length -= n

    def reorder_(self, beam_idx: torch.Tensor) -> None:
        """Gather the samples along the batch dimension in place (beam search)."""
        idx = beam_idx.to(device=self.device, dtype=torch.long)
        L = self.length
        for i in self.owned:
            for buf in (self.k[i], self.v[i], self.k_scale[i], self.v_scale[i]):
                if buf is not None:
                    buf[:, :, :L] = buf[:, :, :L].index_select(0, idx)
        self.seqlens.copy_(self.seqlens.index_select(0, idx))
        self.kv_start.copy_(self.kv_start.index_select(0, idx))

    def reset(self) -> None:
        self.seqlens.zero_()
        self.kv_start.zero_()
        self.length = 0
        self.dense_mask = False


class PagedKVCacheLayer(KVCacheLayer):
    """A layer of a :class:`PagedKVCache`: the kernels take the block table; ``window`` gathers the logical rows."""

    __slots__ = ()

    @property
    def pages(self) -> dict:
        return {"block_table": self.cache.block_table}

    def attend(self, q: torch.Tensor, *, scale: float, causal: bool = True, mask=None, bias=None, alibi_slopes=None,
               rel_bias=None, dropout_p: float = 0.0, training: bool = False, prefix_lens=None) -> torch.Tensor:
        """As :meth:`KVCacheLayer.attend`; the causal prefill of an empty bf16 cache (no mask, bias, ``rel_bias``,
        prefix or dropout) runs the paged flash kernel (:func:`OF.attention_paged`), which reads the pages in place
        and computes what the flash kernel computes over the gathered window."""
        if (causal and self.length == 0 and mask is None and bias is None and rel_bias is None and prefix_lens is None
                and not (training and dropout_p > 0) and OF.attention_paged_supported(q, self.k)):
            return OF.attention_paged(q, self.k, self.v, self.cache.block_table, 0, self.kv_start, scale=scale,
                                      alibi_slopes=alibi_slopes)
        return super().attend(q, scale=scale, causal=causal, mask=mask, bias=bias, alibi_slopes=alibi_slopes,
                              rel_bias=rel_bias, dropout_p=dropout_p, training=training, prefix_lens=prefix_lens)

    def window(self, L: int, dtype) -> Tuple[torch.Tensor, torch.Tensor]:
        t = self.cache.block_table
        k, v = OF.kv_pages_gather(self.k, t, L), OF.kv_pages_gather(self.v, t, L)
        if self.k_scale is None:
            return k, v
        return (OF.kv_cache_dequant(k, OF.kv_pages_gather(self.k_scale, t, L), dtype),
                OF.kv_cache_dequant(v, OF.kv_pages_gather(self.v_scale, t, L), dtype))


class PagedKVCache(StaticKVCache):
    """The logical rows of a :class:`StaticKVCache` in pages of ``PAGE_ROWS`` = 64 rows (one key tile of the decode
    kernel), for generation that runs several sequences per prompt.

    Each owned layer has a K and a V pool ``[num_pages, heads, 64, head_dim]`` (an FP8 cache: E4M3 bytes, with fp32
    row scales ``[num_pages, heads, 64]`` per pool, quantized as in a contiguous cache), and one block table, int32
    ``[batch, max_pages]`` on the device, serves every layer: logical row ``j`` of sequence ``b`` is row ``j % 64`` of
    page ``block_table[b, j // 64]``.  Its host mirror, a reference count per page and a free list live on the host.
    ``seqlens``, ``kv_start`` and ``length`` are logical rows, as in a contiguous cache; ``capacity`` is
    ``max_pages * 64``.

    - ``batch`` prompts are prefilled once, then :meth:`fork` makes each of them ``fork`` sequences that share its
      pages.  A page two sequences share is never written: :meth:`reserve` maps the pages of the rows a step will
      write and gives a sequence whose page there is shared its own copy first (copy on write).  Only the last, partly
      filled page of a sequence can be written while shared, so a full page is never copied.
    - :meth:`reorder_` (beam search) builds the new table rows from the parents' on the host, returns the pages nobody
      references to the free list and writes the table to the device in one copy.
    - The pool is sized once, for the whole call: with ``S = prompt_len // 64`` full prompt pages,
      ``num_pages = batch * S + batch * fork * (max_pages - S)`` — the shared prompt pages once per prompt, and every
      other page once per sequence.  That bounds the distinct pages referenced at any time, copies on write included
      (a copy replaces a reference to a shared page), so generating up to ``capacity`` rows allocates nothing after the
      fork.  With ``fork >= 2`` the pool is smaller than a contiguous cache for the same call whenever
      ``(fork - 1) * S * 64 > fork * (max_pages * 64 - capacity)``.
    """

    def __init__(self, num_layers: int, batch: int, heads: int, head_dim: int, capacity: int,
                 dtype=torch.bfloat16, device=None, layers: Optional[Iterable[int]] = None, kv_dtype=None, *,
                 fork: int = 1, prompt_len: int = 0, prefix_tokens: int = 0):
        self.num_layers, self.heads, self.head_dim = num_layers, heads, head_dim
        self.dtype, self.device = dtype, torch.device(device) if device is not None else torch.device("cpu")
        self.kv_dtype = dtype if kv_dtype is None else kv_dtype
        if self.kv_dtype not in (dtype, torch.float8_e4m3fn):
            raise ValueError(f"kv_dtype must be the projections' {dtype} or torch.float8_e4m3fn, got {kv_dtype}")
        if fork < 1:
            raise ValueError(f"fork must be >= 1, got {fork}")
        self.fp8 = self.kv_dtype == torch.float8_e4m3fn
        self.owned = sorted(range(num_layers) if layers is None else layers)
        self.prompts, self.fork_n, self.rows = batch, fork, batch * fork
        P = OF.PAGE_ROWS
        self.max_pages = -(-max(int(capacity), 1) // P)
        self.capacity = self.max_pages * P
        shared = min(max(int(prompt_len), 0) // P, self.max_pages)
        # the prefix index's budget: extra pages, so the start of a call never evicts
        self.prefix_pages = -(-max(int(prefix_tokens), 0) // P)
        self.num_pages = batch * shared + self.rows * (self.max_pages - shared) + self.prefix_pages
        self._prefix = PrefixIndex()
        self.reused_rows = 0  # the rows the last prefill took from the index
        self.prefix_ok = False   # the call's prompt may be looked up and inserted
        self.index_owner = None  # what the index is valid for (the weights), set by KVCacheOwner
        self.k: List[Optional[torch.Tensor]] = [None] * num_layers
        self.v: List[Optional[torch.Tensor]] = [None] * num_layers
        self.k_scale: List[Optional[torch.Tensor]] = [None] * num_layers
        self.v_scale: List[Optional[torch.Tensor]] = [None] * num_layers
        for i in self.owned:
            # uninitialised, as a contiguous cache's buffers: the kernels read the rows of a sequence's window only
            self.k[i], self.v[i] = (torch.empty(self.num_pages, heads, P, head_dim, dtype=self.kv_dtype,
                                                device=self.device) for _ in range(2))
            if self.fp8:
                self.k_scale[i], self.v_scale[i] = (torch.empty(self.num_pages, heads, P, dtype=torch.float32,
                                                                device=self.device) for _ in range(2))
        self._seqlens = torch.zeros(self.rows, dtype=torch.int32, device=self.device)
        self._kv_start = torch.zeros(self.rows, dtype=torch.int32, device=self.device)
        self._table = torch.full((self.rows, self.max_pages), -1, dtype=torch.int32, device=self.device)
        self.reset()

    def layer(self, i: int) -> KVCacheLayer:
        return PagedKVCacheLayer(self, i)

    def _views(self, batch: int) -> None:
        # views of the full-size tensors: their addresses (which a decode graph reads) do not change at the fork
        self.batch = batch
        self.seqlens, self.kv_start = self._seqlens[:batch], self._kv_start[:batch]
        self.block_table = self._table[:batch]

    def arrays(self) -> List[torch.Tensor]:
        """Every pool (K, V and the FP8 scales of every owned layer): what a page copy copies."""
        return [t for i in self.owned for t in (self.k[i], self.v[i], self.k_scale[i], self.v_scale[i])
                if t is not None]

    def _write_table(self) -> None:
        self._table.copy_(torch.tensor(self.host_table, dtype=torch.int32))

    def _alloc(self) -> int:
        if not self.free:
            raise RuntimeError("PagedKVCache: out of pages (the pool is sized for the call it was allocated for)")
        p = self.free.pop()
        self.refs[p] = 1
        return p

    def _release(self, p: int) -> None:
        self.refs[p] -= 1
        if self.refs[p] == 0:
            self.free.append(p)

    def flash_attention(self) -> bool:
        k = torch.empty((self.batch, self.heads, 1, self.head_dim), dtype=self.dtype, device=self.device)
        return OF.attention_supported(k, k)

    def write_rows(self, i: int, k: torch.Tensor, v: torch.Tensor, row0: int = 0) -> None:
        """As :meth:`StaticKVCache.write_rows`, into the pages of the rows (mapped by :meth:`reserve` first)."""
        n = k.shape[2]
        rows = torch.arange(row0, row0 + n, device=self.device)[None].expand(self.batch, n)
        ids = OF._page_ids(self.block_table, rows, self.num_pages)
        off = rows % OF.PAGE_ROWS
        for pool, scale, x in ((self.k, self.k_scale, k), (self.v, self.v_scale, v)):
            x = x.transpose(1, 2)   # [batch, n, heads, d]
            if self.fp8:
                pool[i][ids, :, off], scale[i][ids, :, off] = OF.kv_cache_quantize_ref(x)
            else:
                pool[i][ids, :, off] = x

    def fill(self, kv, S: int, window=None) -> None:
        raise NotImplementedError("PagedKVCache holds self-attention rows only (no fixed cross-attention window)")

    def reserve(self, n: int) -> None:
        """Map the pages of rows ``length .. length + n`` of every sequence and make each of them the sequence's own: a
        shared page is copied first (one page copy launch for every layer).  The pool is never reallocated."""
        need = self.length + n
        if need > self.capacity:
            raise ValueError(f"PagedKVCache holds up to {self.capacity} rows per sequence, {need} needed")
        P = OF.PAGE_ROWS
        copies, changed = [], False
        for slot in range(self.length // P, -(-need // P)):
            for row in self.host_table[: self.batch]:
                if slot >= self.mapped:
                    row[slot], changed = self._alloc(), True
                elif self.refs[row[slot]] > 1:
                    new = self._alloc()
                    copies.append((row[slot], new))
                    self.refs[row[slot]] -= 1
                    row[slot], changed = new, True
        self.mapped = max(self.mapped, -(-need // P))
        if copies:
            OF.kv_page_copy(self.arrays(), copies)
        if changed:
            self._write_table()

    def _unmap_from(self, slot: int) -> None:
        # every sequence's pages from `slot` on go back (the rows there are no longer held)
        for row in self.host_table[: self.batch]:
            for s in range(slot, self.mapped):
                self._release(row[s])
                row[s] = -1
        self.mapped = min(self.mapped, slot)

    def rollback(self, n: int) -> None:
        super().rollback(n)
        slot = -(-self.length // OF.PAGE_ROWS)
        if slot < self.mapped:
            self._unmap_from(slot)
            self._write_table()

    def fork(self, n: int) -> None:
        """After the prefill of the ``batch`` prompts: each prompt becomes ``n`` sequences (prompt ``p``'s are rows
        ``p * n .. p * n + n - 1``, the order of ``generate``'s expanded inputs) sharing its pages; ``seqlens``,
        ``kv_start`` and the dense-mask flag carry over."""
        if n < 1 or self.batch * n > self.rows:
            raise ValueError(f"fork: {self.batch} prompts x {n} exceed the {self.rows} sequences this cache holds")
        if n == 1:
            return
        b = self.batch
        self.host_table = [list(self.host_table[p]) for p in range(b) for _ in range(n)] + \
            self.host_table[b * n:]
        for row in self.host_table[: b * n : n]:
            for page in row[: self.mapped]:
                self.refs[page] += n - 1
        seqlens, kv_start = self.seqlens.repeat_interleave(n), self.kv_start.repeat_interleave(n)
        self._views(b * n)
        self.seqlens.copy_(seqlens)
        self.kv_start.copy_(kv_start)
        self._write_table()

    def reorder_(self, beam_idx: torch.Tensor) -> None:
        """Sequence ``i`` continues sequence ``beam_idx[i]``: its table row becomes the parent's (one host sync); pages
        no sequence references any more return to the free list.  No page is copied here: a shared last page is copied
        when a sequence next writes to it (:meth:`reserve`)."""
        idx = [int(i) for i in beam_idx.tolist()]
        old = self.host_table
        self.host_table = [list(old[i]) for i in idx] + old[self.batch:]
        refs = self._index_refs()
        for row in self.host_table[: self.batch]:
            for page in row[: self.mapped]:
                refs[page] += 1
        self.free += [p for p in range(self.num_pages) if self.refs[p] > 0 and refs[p] == 0]
        self.refs = refs
        self._write_table()
        dev = beam_idx.to(device=self.device, dtype=torch.long)
        self.seqlens.copy_(self.seqlens.index_select(0, dev))
        self.kv_start.copy_(self.kv_start.index_select(0, dev))

    def reset(self) -> None:
        self._views(self.prompts)
        self._seqlens.zero_()
        self._kv_start.zero_()
        self.length = 0
        self.dense_mask = False
        self.host_table = [[-1] * self.max_pages for _ in range(self.rows)]
        self.refs = self._index_refs()   # the prefix index keeps its pages
        # pages are taken from the end: 0, 1, 2, ...
        self.free = [p for p in range(self.num_pages - 1, -1, -1) if self.refs[p] == 0]
        self.mapped = 0   # the page slots mapped in every sequence's row
        self._write_table()

    # ---- prefix index (PrefixIndex) -------------------------------------------------------------------------------
    # Only a sequence's last, partly filled page is ever written, and a shared one is copied first, so a full page is
    # immutable and a later call can map it.

    _page_keys = staticmethod(PrefixIndex.page_keys)

    @property
    def _index(self) -> dict:
        return self._prefix.pages

    @property
    def _entry(self) -> dict:
        return self._prefix.keys

    def _index_refs(self) -> List[int]:
        refs = [0] * self.num_pages
        for page in self._entry:
            refs[page] = 1
        return refs

    @staticmethod
    def _rows(input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor]):
        ids = input_ids.tolist()
        mask = [[1] * len(r) for r in ids] if attention_mask is None else attention_mask.to(torch.int64).tolist()
        return ids, mask

    def cached_pages(self) -> int:
        return len(self._entry)

    def fits(self, batch: int, fork: int, prompt_len: int, capacity: int, prefix_tokens: int, dtype, device,
             kv_dtype) -> bool:
        """Whether a call of ``batch`` prompts forked ``fork`` times, with ``prompt_len``-token prompts and up to
        ``capacity`` rows, runs on this pool with a prefix budget of ``prefix_tokens``: the pool, and its index, are
        then kept."""
        P = OF.PAGE_ROWS
        shared = min(max(int(prompt_len), 0) // P, self.max_pages)
        need = batch * shared + batch * fork * (self.max_pages - shared) + self.prefix_pages
        return (self.prompts == batch and self.fork_n == fork and self.max_pages * P >= capacity
                and self.prefix_pages == -(-int(prefix_tokens) // P) and need <= self.num_pages
                and self.dtype == dtype and self.device == torch.device(device)
                and self.kv_dtype == (dtype if kv_dtype is None else kv_dtype))

    def clear_prefix_index(self) -> None:
        """Drop every cached page (a page a sequence still maps keeps that sequence's reference)."""
        for page in self._prefix.clear():
            self._release(page)

    def lookup(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor]) -> int:
        """Before the prefill of the ``batch`` prompts ``input_ids`` ``[batch, s]`` on the empty cache: map the longest
        run of cached pages every prompt starts with, at most ``(s - 1) // 64`` (at least one token is prefilled, for the
        first logits), into every row, and set the lengths and ``kv_start`` (the prompt's left padding) as if those rows
        had been prefilled.  Returns the pages taken; ``reused_rows`` counts their rows.  A prompt whose padding needs a
        dense mask is neither looked up nor inserted (``prefix_ok``)."""
        if self.length != 0 or input_ids.shape[0] != self.batch:
            raise ValueError("lookup: the prompts of an empty cache, one per row")
        self.reused_rows = 0
        start = None
        if attention_mask is not None:
            start = left_padding(attention_mask)
        self.prefix_ok = self.prefix_pages > 0 and (attention_mask is None or start is not None)
        if not self.prefix_ok:
            return 0
        s = input_ids.shape[1]
        ids, mask = self._rows(input_ids, attention_mask)
        chains = [self._prefix.chain(self._page_keys(ids[b], mask[b], (s - 1) // OF.PAGE_ROWS))
                  for b in range(self.batch)]
        hit = min(len(c) for c in chains)
        if hit == 0:
            return 0
        self._prefix.touch(page for chain in chains for page in chain[:hit])
        for b, chain in enumerate(chains):
            for j, page in enumerate(chain[:hit]):
                self.host_table[b][j] = page
                self.refs[page] += 1
        rows = hit * OF.PAGE_ROWS
        self.mapped, self.length, self.reused_rows = hit, rows, rows
        self.seqlens.fill_(rows)
        if start is not None:
            self.kv_start.copy_(start)
        self._write_table()
        return hit

    def insert(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor]) -> None:
        """Index the full pages of every sequence's rows ``[:L]`` (``L = input_ids.shape[1] <= length``: the tokens
        fed, with their mask), then evict least-recently-used leaves (pages no cached page continues) down to the
        budget.  Nothing for a call whose prompt is not ``prefix_ok``."""
        if not self.prefix_ok:
            return
        L = min(input_ids.shape[1], self.length)
        ids, mask = self._rows(input_ids[:, :L], None if attention_mask is None else attention_mask[:, :L])
        for page in self._prefix.insert((self._page_keys(ids[b], mask[b], L // OF.PAGE_ROWS), self.host_table[b])
                                        for b in range(self.batch)):
            self.refs[page] += 1
        for page in self._prefix.evict(self.prefix_pages):
            self._release(page)


class RaggedPagedKVCacheLayer(KVCacheLayer):
    """A layer of a :class:`RaggedPagedKVCache`: the ragged append, then the decode rows through the split-KV decode
    kernel and the prompt chunks through the ragged paged flash prefill."""

    __slots__ = ()

    def append(self, qkv: torch.Tensor, cos=None, sin=None) -> torch.Tensor:
        c = self.cache
        return OF.kv_cache_append_paged_varlen(qkv, self.k, self.v, c.table, c.cu_q, c.past, cos, sin, self.k_scale,
                                               self.v_scale)

    def attend(self, q: torch.Tensor, *, scale: float, causal: bool = True, mask=None, bias=None, alibi_slopes=None,
               rel_bias=None, dropout_p: float = 0.0, training: bool = False, prefix_lens=None) -> torch.Tensor:
        """The attention of the step's ``q`` ``[1, T, a, d]``, each token over its own sequence's rows → ``[1, T, a, d]``.
        Causal self-attention only (with or without ALiBi)."""
        if (not causal or mask is not None or bias is not None or rel_bias is not None or prefix_lens is not None
                or (training and dropout_p > 0)):
            raise ValueError("RaggedPagedKVCache: causal self-attention without mask, bias, rel_bias, prefix or "
                             "dropout only")
        c = self.cache
        scales = {"k_scale": self.k_scale, "v_scale": self.v_scale}
        if not c.flash_attention():   # the reference math, every sequence alike
            return OF.attention_paged_varlen(q[0], self.k, self.v, c.table, c.cu_q, c.past, scale=scale,
                                             alibi_slopes=alibi_slopes, **scales)[None]
        mb = c.max_batch
        out = OF.decode_attention(q[0, :mb, None], self.k, self.v, c.past[:mb], c.kv_start, scale=scale,
                                  alibi_slopes=alibi_slopes, block_table=c.table[:mb], **scales)
        out = out.view(1, mb, *q.shape[2:])
        if c.chunks == 0:
            return out
        pre = OF.attention_paged_varlen(q[0, mb:], self.k, self.v, c.table[mb:], c.cu_c, c.past[mb:], c.tiles,
                                        scale=scale, alibi_slopes=alibi_slopes, **scales)
        return torch.cat((out, pre[None]), dim=1)


class RaggedPagedKVCache(StaticKVCache):
    """The KV cache of continuous batching (:class:`~libai_b200.inference.engine.GenerationEngine`): up to
    ``max_batch`` sequences (slots) of their own lengths, whose tokens of one step are packed into one forward over
    ``[1, T]``.  A model's cached step runs on it unchanged: ``layer(i).append`` / ``attend`` and ``advance`` are those
    of a :class:`StaticKVCache` of batch 1.

    - Each owned layer has a K and a V pool ``[num_pages + 1, heads, 64, head_dim]`` in the format of a
      :class:`PagedKVCache`; the last page is the **sink**, which idle decode rows write and read (their outputs are
      discarded).  With ``kv_dtype=torch.float8_e4m3fn`` the pools hold E4M3 bytes and each layer has fp32 row scales
      ``k_scale`` / ``v_scale`` ``[num_pages + 1, heads, 64]`` (``fp8`` is set): the ragged FP8 append writes them, and
      the decode rows and prompt chunks attend over the dequantized rows.  Every other page is the scheduler's:
      :meth:`alloc` and :meth:`release` keep a reference count per page and a free list, and the prefix index
      (:class:`PrefixIndex`) holds one reference per cached page.
    - A step's tokens are the ``max_batch`` decode rows, one per slot in slot order, then the prompt chunks.  Its
      descriptor (:meth:`write_step`), written to the device in one copy, holds the token ids, ``cu_q`` (the
      sequences' token offsets: the decode rows are sequences of one token), ``past`` (the rows each holds), one
      block-table row per sequence (a decode row of a slot that is not decoding maps the sink, with ``past`` 0), the
      chunks' own offsets ``cu_c`` and the prefill's tile list.  The buffers have fixed addresses, so a decode graph
      replays a step of decode rows after its descriptor is rewritten.
    - ``length`` counts the tokens of the current step once :meth:`advance` ran (what a decode graph checks); the
      per-sequence lengths are the scheduler's, written into each step's descriptor.  :meth:`reserve` does nothing:
      the pages are mapped at admission.
    """

    def __init__(self, num_layers: int, max_batch: int, heads: int, head_dim: int, num_pages: int, max_pages: int,
                 max_tokens: int, dtype=torch.bfloat16, device=None, layers: Optional[Iterable[int]] = None,
                 kv_dtype=None):
        self.num_layers, self.heads, self.head_dim = num_layers, heads, head_dim
        self.dtype = dtype
        self.kv_dtype = dtype if kv_dtype is None else kv_dtype
        if self.kv_dtype not in (dtype, torch.float8_e4m3fn):
            raise ValueError(f"kv_dtype must be the projections' {dtype} or torch.float8_e4m3fn, got {kv_dtype}")
        self.device = torch.device(device) if device is not None else torch.device("cpu")
        self.fp8 = self.kv_dtype == torch.float8_e4m3fn
        self.owned = sorted(range(num_layers) if layers is None else layers)
        self.max_batch, self.max_pages, self.max_tokens = max_batch, max_pages, max_tokens
        self.num_pages, self.sink = num_pages, num_pages
        self.batch, self.capacity, self.length, self.dense_mask = 1, max_pages * OF.PAGE_ROWS, 0, False
        P = OF.PAGE_ROWS
        self.k: List[Optional[torch.Tensor]] = [None] * num_layers
        self.v: List[Optional[torch.Tensor]] = [None] * num_layers
        self.k_scale: List[Optional[torch.Tensor]] = [None] * num_layers
        self.v_scale: List[Optional[torch.Tensor]] = [None] * num_layers
        for i in self.owned:
            # uninitialised: the kernels read the rows of each sequence's window only
            self.k[i], self.v[i] = (torch.empty(num_pages + 1, heads, P, head_dim, dtype=self.kv_dtype,
                                                device=self.device) for _ in range(2))
            if self.fp8:
                self.k_scale[i], self.v_scale[i] = (torch.empty(num_pages + 1, heads, P, dtype=torch.float32,
                                                                device=self.device) for _ in range(2))
        self.refs = [0] * num_pages
        self.free = list(range(num_pages - 1, -1, -1))   # pages are taken from the end: 0, 1, 2, ...
        self.prefix = PrefixIndex()
        self.index_owner = None
        # the descriptor: offsets (int32 elements) of its parts in one buffer
        nseq, self.max_tiles = 2 * max_batch, max_tokens // 128 + max_batch
        sizes = (("ids", max_tokens), ("cu_q", nseq + 1), ("past", nseq), ("table", nseq * max_pages),
                 ("cu_c", max_batch + 1), ("tiles", 2 * self.max_tiles), ("rows", 2 * max_batch))
        self._off, n = {}, 0
        for name, size in sizes:
            n += n % 2   # the tiles are read as int2
            self._off[name] = (n, size)
            n += size
        pin = self.device.type == "cuda"
        self._host = torch.zeros(n, dtype=torch.int32, pin_memory=pin)
        self._desc = torch.zeros(n, dtype=torch.int32, device=self.device)
        # the host buffer is rewritten only once the previous step's copy out of it has run: a step that samples no
        # token (prompt chunks that end no prompt) has no host sync of its own
        self._copied = torch.cuda.Event() if pin else None
        self.kv_start = torch.zeros(max_batch, dtype=torch.int32, device=self.device)
        self.seqlens = self._part(self._desc, "past")[:max_batch]
        self._views(max_batch, 0, 0, 0)

    def _part(self, buf: torch.Tensor, name: str) -> torch.Tensor:
        o, n = self._off[name]
        return buf[o : o + n]

    def _views(self, T: int, nseq: int, chunks: int, tiles: int) -> None:
        d = self._desc
        self.T, self.chunks = T, chunks
        nseq = max(nseq, self.max_batch)
        self.ids = self._part(d, "ids")[:T]
        self.cu_q = self._part(d, "cu_q")[: nseq + 1]
        self.past = self._part(d, "past")[:nseq]
        self.table = self._part(d, "table")[: nseq * self.max_pages].view(nseq, self.max_pages)
        self.cu_c = self._part(d, "cu_c")[: chunks + 1]
        self.tiles = self._part(d, "tiles")[: 2 * tiles].view(tiles, 2)

    def layer(self, i: int) -> KVCacheLayer:
        return RaggedPagedKVCacheLayer(self, i)

    def write_step(self, decode, chunks, rows=()) -> Tuple[torch.Tensor, torch.Tensor]:
        """Write the descriptor of a step to the device (one copy) and return its token ids ``[1, T]`` (int64) and
        ``rows`` (the token rows whose logits are sampled; int32), both on the device.  ``decode``: per slot ``None``
        (not decoding) or ``(token, past, pages)``; ``chunks``: the prompt chunks ``(tokens, past, pages)``.  ``pages``
        lists a sequence's table row (its pages in order)."""
        mb, mp = self.max_batch, self.max_pages
        if self._copied is not None:
            self._copied.synchronize()
        h = self._host.numpy()   # the pinned buffer, written in place
        ids, cu, past, cu_c, tiles, sample = (self._part(h, n) for n in ("ids", "cu_q", "past", "cu_c", "tiles",
                                                                          "rows"))
        table = self._part(h, "table").reshape(-1, mp)
        lens = [len(c[0]) for c in chunks]
        nseq, T = mb + len(chunks), mb + sum(lens)
        if len(decode) != mb or len(chunks) > mb or T > self.max_tokens:
            raise ValueError(f"a step holds {mb} decode rows, at most {mb} chunks and {self.max_tokens} tokens")
        table[:nseq] = -1
        for n, d in enumerate(decode):
            if d is None:
                ids[n], past[n], table[n, 0] = 0, 0, self.sink
            else:
                ids[n], past[n] = d[0], d[1]
                table[n, : len(d[2])] = d[2]
        t = mb
        for k, (tok, pst, pages) in enumerate(chunks):
            ids[t : t + len(tok)] = tok
            past[mb + k] = pst
            table[mb + k, : len(pages)] = pages
            t += len(tok)
        cu[: mb + 1] = range(mb + 1)
        cu_c[0] = 0
        cu_c[1 : len(chunks) + 1] = _cumsum(lens)
        cu[mb + 1 : nseq + 1] = [mb + x for x in _cumsum(lens)]
        tl = OF.varlen_tiles(lens, [c[1] for c in chunks]).numpy()
        tiles[: tl.size] = tl.reshape(-1)
        sample[: len(rows)] = rows
        self._desc.copy_(self._host, non_blocking=True)
        if self._copied is not None:
            self._copied.record()
        self._views(T, nseq, len(chunks), tl.shape[0])
        self.length = 0
        return self.ids.long()[None], self._part(self._desc, "rows")[: len(rows)]

    # ---- pages ----------------------------------------------------------------------------------------------------
    def index_only(self, exclude=()) -> int:
        """The pages only the prefix index holds (free on demand), not counting ``exclude``."""
        return sum(1 for p in self.prefix.keys if self.refs[p] == 1 and p not in exclude)

    def available(self, exclude=()) -> int:
        return len(self.free) + self.index_only(exclude)

    def alloc(self, n: int) -> List[int]:
        """``n`` pages of the free list, evicting least-recently-used index-only pages as needed."""
        out = []
        for _ in range(n):
            if not self.free:
                page = self.prefix.pop_leaf(lambda p: self.refs[p] == 1)
                if page is None:
                    raise RuntimeError("RaggedPagedKVCache: out of pages")
                self.release([page])
            page = self.free.pop()
            self.refs[page] = 1
            out.append(page)
        return out

    def retain(self, pages: Iterable[int]) -> None:
        for p in pages:
            self.refs[p] += 1

    def release(self, pages: Iterable[int]) -> None:
        for p in pages:
            self.refs[p] -= 1
            if self.refs[p] == 0:
                self.free.append(p)

    def lookup(self, tokens: List[int]) -> List[int]:
        """The cached pages a prompt of ``tokens`` starts with, at most ``(len - 1) // 64``, mapped by reference (and
        marked used)."""
        keys = PrefixIndex.page_keys(tokens, [1] * len(tokens), (len(tokens) - 1) // OF.PAGE_ROWS)
        chain = self.prefix.chain(keys)
        if chain:
            self.prefix.touch(chain)
            self.retain(chain)
        return chain

    def peek(self, tokens: List[int]) -> List[int]:
        """:meth:`lookup` without taking the pages."""
        keys = PrefixIndex.page_keys(tokens, [1] * len(tokens), (len(tokens) - 1) // OF.PAGE_ROWS)
        return self.prefix.chain(keys)

    def insert(self, tokens: List[int], pages: List[int]) -> None:
        """Index the full pages of a sequence's fed ``tokens`` (its rows), held in ``pages``."""
        full = len(tokens) // OF.PAGE_ROWS
        self.retain(self.prefix.insert([(PrefixIndex.page_keys(tokens, [1] * len(tokens), full), pages)]))

    def clear_prefix_index(self) -> None:
        self.release(self.prefix.clear())

    # ---- the StaticKVCache protocol of a model's cached step --------------------------------------------------------
    def flash_attention(self) -> bool:
        """Whether the native kernels run: the decode rows through the paged decode kernel, the prompt chunks through
        the ragged paged flash prefill (bf16 or FP8 pools)."""
        return OF._decode_native(torch.empty(1, dtype=self.dtype, device=self.device), self.k[self.owned[0]])

    def advance(self, n: int) -> None:
        self.length += n

    def reserve(self, n: int) -> None:
        return None

    def reset(self) -> None:
        self.length = 0

    def write_rows(self, i, k, v, row0=0):
        raise NotImplementedError("RaggedPagedKVCache: rows are written by the ragged append")

    def fill(self, kv, S: int, window=None) -> None:
        raise NotImplementedError("RaggedPagedKVCache holds self-attention rows only")

    def rollback(self, n: int) -> None:
        raise NotImplementedError("RaggedPagedKVCache: no rollback")

    def reorder_(self, beam_idx) -> None:
        raise NotImplementedError("RaggedPagedKVCache: no reorder")


def _cumsum(xs) -> List[int]:
    out, t = [], 0
    for x in xs:
        t += x
        out.append(t)
    return out


class KVCacheOwner:
    """The model side of a :class:`StaticKVCache` for decoder-only models: ``generate`` sizes it through
    ``allocate_kv_cache``, ``set_cache`` / ``past_key_values`` / ``past_length`` keep the generator's cache protocol.
    The model lists its self-attention modules (``query_key_value``, ``head_size``, and ``local_kv_heads`` — the rank's
    key/value heads — or, for modules without grouped-query attention, ``local_heads``)."""

    kv_cache: Optional[StaticKVCache] = None
    past_length = 0
    kv_cache_dtype = None   # what the cache holds: None = the weights' dtype; torch.float8_e4m3fn = FP8 rows
    # a paged cache for the next allocate_kv_cache: (sequences per prompt, prompt length, prefix index budget in
    # tokens), set by generate(); None = a contiguous StaticKVCache
    kv_cache_paging: Optional[Tuple[int, int, int]] = None
    # the rows a step may reach (the last _prepare_cache's max_positions): a replayed decode graph checks it instead
    max_cache_positions: Optional[int] = None

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
        qkv = mods[0].query_key_value
        w = qkv.weight
        # the activations' dtype: a Linear1D with FP8 weights keeps it apart (LoRA wrappers have no compute_dtype)
        dtype = getattr(qkv, "compute_dtype", None) or w.dtype
        c = self.kv_cache
        heads = getattr(mods[0], "local_kv_heads", mods[0].local_heads)
        if self.kv_cache_paging is not None:
            fork, prompt_len, prefix_tokens = self.kv_cache_paging
            if not (prefix_tokens > 0 and isinstance(c, PagedKVCache)
                    and c.fits(batch, fork, prompt_len, max_length, prefix_tokens, dtype, w.device, self.kv_cache_dtype)):
                if prefix_tokens > 0 and isinstance(c, PagedKVCache) and c.cached_pages():
                    logger.info("prefix cache: this call does not fit the paged pool; a new pool starts empty")
                # sized for this call: the old cache (and a graph on it) go first
                self.kv_cache = self._decode_graph = c = None
                c = PagedKVCache(len(mods), batch, heads, mods[0].head_size, max_length, dtype, w.device, owned,
                                 self.kv_cache_dtype, fork=fork, prompt_len=prompt_len, prefix_tokens=prefix_tokens)
            weights = self._prefix_cache_weights()
            if c.index_owner != weights:   # the index holds K/V of other weights
                c.clear_prefix_index()
                c.index_owner = weights
        elif (c is None or isinstance(c, PagedKVCache) or not c.matches(batch, dtype, w.device, self.kv_cache_dtype)
              or c.capacity < max_length):
            c = StaticKVCache(len(mods), batch, heads, mods[0].head_size, max_length, dtype, w.device, owned,
                              self.kv_cache_dtype)
            self._decode_graph = None   # a decode graph of the old cache (and its memory pool) goes with it
        c.reset()
        self.kv_cache, self.past_length = c, 0
        return c

    def _prefix_cache_weights(self) -> tuple:
        # every parameter's storage and version: load_state_dict, in-place updates and weight quantization change them
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

    # rows a step writes before the prompt's (ChatGLM's P-tuning prefix): such a cache takes no prefix index
    cache_rows_before_prompt = 0

    def clear_prefix_cache(self) -> None:
        """Empty the prefix index of the model's paged cache (``generate(prefix_cache_tokens=...)``)."""
        if isinstance(self.kv_cache, PagedKVCache):
            self.kv_cache.clear_prefix_index()

    def _prepare_cache(self, input_ids, max_positions: Optional[int] = None) -> StaticKVCache:
        """The cache for this step's ``input_ids`` ``[b, s]``: allocated for a new batch, grown to fit ``s`` more rows."""
        bsz, s_len = input_ids.shape
        c = self.kv_cache
        if c is None or (c.length == 0 and c.batch != bsz):
            c = self.allocate_kv_cache(bsz, s_len)
        self.max_cache_positions = max_positions
        if max_positions is not None and c.length + s_len > max_positions:
            raise ValueError(f"The maximum supported length is {max_positions}, "
                             f"and the current length is {c.length + s_len}.")
        c.reserve(s_len)
        return c

    def prepare_inputs_for_generation(self, input_ids, past=None, attention_mask=None, use_cache=None, **kwargs):
        """With a warm cache only the newest token is fed; the padding mask always covers cache + new tokens."""
        if past is not None and use_cache:
            input_ids = input_ids[:, -1:]
        out = {"input_ids": input_ids, "use_cache": bool(use_cache)}
        if attention_mask is not None and not bool(attention_mask.all()):
            out["attention_mask"] = attention_mask
        return out

    def set_cache(self, past_key_values):
        """``None`` empties the cache (its buffers are kept); a :class:`StaticKVCache` becomes the model's cache."""
        if past_key_values is None:
            if self.kv_cache is not None:
                self.kv_cache.reset()
        else:
            assert isinstance(past_key_values, StaticKVCache), "set_cache expects a StaticKVCache"
            self.kv_cache = past_key_values
        self.past_length = 0 if self.kv_cache is None else self.kv_cache.length
