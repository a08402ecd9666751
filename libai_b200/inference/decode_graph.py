"""Replay ``generate()``'s cached decode steps from a CUDA graph (``generate(decode_graphs=True)``).

A decode step of a :class:`~libai_b200.inference.kv_cache.KVCacheOwner` launches every kernel of every layer from
Python, and at batch 1 the host's enqueue time, not the GPU, sets the decoding rate.  Every kernel on that path reads
what changes from step to step on the device (the cache lengths ``seqlens``, the left padding ``kv_start``; the
positions of GPT-2, ChatGLM and GLM), so one capture of a step replays every later one: one graph launch per step.

Capture protocol (:class:`DecodeGraph`): a step is first run eagerly (a real step, which also performs every lazy
one-time setup: extension load, ``cudaFuncSetAttribute``, driver entry points); the next one is captured, which runs
its Python once but no kernel, so every host-side effect of the captured Python (``cache.length``, the model's
``past_length``) is rolled back; that step and every later one are then replayed, and after each replay the host
mirrors advance by the step's rows: one, or ``tokens`` for a step that opts in to more (a speculative verify step,
``step(..., tokens=k + 1)``).  The device-side ``seqlens.add_`` of ``StaticKVCache.advance`` is inside the graph, so after
every step the cache rows, ``seqlens``, ``kv_start`` and the host mirror are what eager decoding leaves, bit for bit.

A graph is kept per model and keyed by the batch, the caches' buffer addresses, capacity and KV dtype, the weights'
addresses and the step's input signature; a new key captures again and frees the old graph's memory pool.  A model
that allocates a new cache drops its graph at once, so a replaced cache's buffers are not kept alive by it.  Beam
search's in-place ``StaticKVCache.reorder_`` keeps the key, and so does a :class:`PagedKVCache`'s reorder, which
rewrites its block table in place; such a cache maps the pages of a step's rows before the capture and before every
replay.  A step the graph cannot reproduce runs eagerly, with the
same tokens and one log line per reason (:func:`fallback_reason`), and so does every step of a key whose capture
failed.
"""
from __future__ import annotations

import logging
import time
from typing import Dict, Optional

import torch

from libai_b200 import ops
from libai_b200.ops import use_native
from libai_b200.utils import distributed as dutil

from .kv_cache import PagedKVCache, StaticKVCache

logger = logging.getLogger(__name__)

# step inputs the model reads on the device: each is copied into a static buffer of the graph before a replay
STATIC_INPUTS = ("input_ids", "decoder_input_ids", "position_ids")
# inputs a cached step provably ignores while no cache needs a dense mask: padding masks (kv_start holds a left-padded
# prompt's padding) and an encoder-decoder model's encoder inputs (its cross cache holds their projection)
IGNORED_INPUTS = ("attention_mask", "encoder_input_ids", "encoder_attn_mask", "encoder_decoder_attn_mask")
# the most new tokens a replayed step takes: the split-KV decode kernel's limit (OF.decode_attention)
MAX_TOKENS = 16


class DecodeCall:
    """One ``generate()`` call's use of decode graphs: the reasons already logged, and the weights' addresses (taken at
    the first decode step, after the prefill has placed every lazily built buffer)."""

    def __init__(self):
        self.logged = set()
        self.weights = None


def _caches(model):
    """The model's self-attention cache and, for T5/mT5, the cross cache."""
    cross = getattr(model, "cross_cache", None)
    return [model.kv_cache] + ([cross] if isinstance(cross, StaticKVCache) else [])


def _cache_key(c: StaticKVCache):
    # addresses, not the object: the graph reads and writes these buffers and nothing else of the cache, and a key
    # that held the cache would keep a replaced one's buffers alive (a paged cache: its pools and block table, which
    # a reorder rewrites in place)
    buffers = [t for bufs in (c.k, c.v, c.k_scale, c.v_scale) for t in bufs if t is not None]
    if isinstance(c, PagedKVCache):
        buffers.append(c.block_table)
    return (c.batch, c.capacity, c.kv_dtype, tuple(t.data_ptr() for t in buffers), c.seqlens.data_ptr(),
            c.kv_start.data_ptr())


def _signature(inputs: Dict):
    sig = []
    for k in sorted(inputs):
        v = inputs[k]
        if k in STATIC_INPUTS and torch.is_tensor(v):
            sig.append((k, tuple(v.shape), v.dtype, v.device))
        elif torch.is_tensor(v):
            sig.append((k, "tensor"))   # ignored by the step; whether it is given still picks the model's branch
        else:
            sig.append((k, v))
    return tuple(sig)


def fallback_reason(model, inputs: Dict, tokens: int = 1) -> Optional[str]:
    """Why this decode step (the cache is not empty) of ``tokens`` new tokens cannot replay a graph, or None when it
    can."""
    cache = model.kv_cache
    if cache.device.type != "cuda":
        return "the cache is not on a CUDA device"
    topo = dutil.get_dist_util()
    if topo.tensor_parallel_size > 1 or topo.pipeline_parallel_size > 1:
        return "tensor- or pipeline-parallel inference"
    if not (use_native(cache.seqlens) and cache.dtype == torch.bfloat16 and cache.head_dim in (64, 128)):
        return "the step does not run the native bf16 kernels"
    ids = inputs.get("decoder_input_ids", inputs.get("input_ids"))
    if not torch.is_tensor(ids) or ids.dim() != 2 or ids.shape[1] != tokens:
        return "more than one new token" if tokens == 1 else f"not {tokens} new tokens"
    if any(c.dense_mask for c in _caches(model)):
        return "the prompt's padding needs a dense mask"
    if cache.length + tokens > cache.capacity:
        return "the cache must grow"
    limit = model.max_cache_positions
    if limit is not None and cache.length + tokens > limit:
        return "the step passes the model's maximum length"
    for k, v in inputs.items():
        if torch.is_tensor(v) and k not in STATIC_INPUTS and k not in IGNORED_INPUTS:
            return f"input {k!r} is not a static buffer"
    return None


class DecodeGraph:
    """The CUDA graph of one decode step of ``model`` on its current cache(s): static input buffers, the captured graph
    and its outputs.  :meth:`step` runs the eager warm-up step, captures, and replays."""

    def __init__(self, key, inputs: Dict, tokens: int = 1):
        self.key = key
        self.tokens = tokens       # the new tokens (cache rows) of one step
        self.static = {k: v.clone() for k, v in inputs.items() if k in STATIC_INPUTS and torch.is_tensor(v)}
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.outputs = None
        self.warm = False          # an eager decode step has run since this graph was created
        self.launches = 0          # the kernels of one eager step (ops.launch_count)
        self.capture_ms = 0.0      # the capture alone (the eager step before it not included)
        self.failed: Optional[str] = None   # why the capture failed: every step on this key then runs eagerly

    def step(self, model, inputs: Dict, call: DecodeCall):
        if self.graph is None:
            if self.failed is None and not self.warm:
                self.warm = True
                return model(**inputs)
            if self.failed is None:
                try:
                    self._capture(model, inputs)
                except Exception as e:   # the graph is an optimisation: the step runs eagerly, as it would without
                    self.failed = f"the capture failed: {type(e).__name__}: {str(e)[:200]}"
            if self.failed is not None:
                return _eager(model, inputs, call, self.failed, logging.WARNING)
        return self.replay(model, inputs)

    def _capture(self, model, inputs: Dict):
        # a paged cache maps (and copies on write) the pages of the step's rows now: the captured step must not
        model.kv_cache.reserve(self.tokens)
        caches = _caches(model)
        lengths, past = [c.length for c in caches], model.past_length
        call = {**inputs, **self.static}
        stream = torch.cuda.current_stream()
        t0 = time.perf_counter()
        n0 = ops.launch_count()
        graph = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(graph):
                outputs = model(**call)
        finally:
            # the captured Python ran once and no kernel did: undo what it did on the host (and, after a failed
            # capture, the switch to the capture stream)
            torch.cuda.set_stream(stream)
            self.launches = ops.launch_count() - n0
            ops.count_launch(-self.launches)
            advanced = caches[0].length - lengths[0]
            for c, n in zip(caches, lengths):
                c.length = n
            model.past_length = past
        if advanced != self.tokens:
            raise RuntimeError(f"the captured step advanced the cache by {advanced} rows, not {self.tokens}")
        self.graph, self.outputs = graph, outputs
        self.capture_ms = (time.perf_counter() - t0) * 1e3

    def replay(self, model, inputs: Dict):
        for k, v in self.static.items():
            v.copy_(inputs[k])
        # a replayed step runs no Python: the pages of its rows are mapped first (a contiguous cache has its rows)
        model.kv_cache.reserve(self.tokens)
        self.graph.replay()
        ops.count_launch(self.launches)
        cache = model.kv_cache
        cache.length += self.tokens
        model.past_length = cache.length
        # the graph's outputs are overwritten by the next replay: hand out copies
        return {k: v.clone() if torch.is_tensor(v) else v for k, v in self.outputs.items()}


def _eager(model, inputs: Dict, call: DecodeCall, reason: str, level=logging.INFO):
    """The eager step, with one log line per reason and call."""
    if reason not in call.logged:
        call.logged.add(reason)
        logger.log(level, "decode graphs: eager decode steps for %s (%s)", type(model).__name__, reason)
    return model(**inputs)


def step(model, inputs: Dict, call: DecodeCall, tokens: int = 1):
    """One cached step of ``model`` (``model(**inputs)``): replayed from the model's :class:`DecodeGraph` when the step
    is eligible, else eager (the prefill, and each :func:`fallback_reason` or failed capture, logged once per call).
    ``tokens``: the new tokens of the step the graph captures and replays, 1 to 16 (a speculative verify step takes
    k + 1); a step with another number of new tokens runs eagerly."""
    if not 1 <= tokens <= MAX_TOKENS:
        raise ValueError(f"tokens: a decode graph replays steps of 1 to {MAX_TOKENS} new tokens, got {tokens}")
    cache = getattr(model, "kv_cache", None)
    if not isinstance(cache, StaticKVCache) or cache.length == 0 or not inputs.get("use_cache"):
        return model(**inputs)
    reason = fallback_reason(model, inputs) if tokens == 1 else fallback_reason(model, inputs, tokens)
    if reason is not None:
        return _eager(model, inputs, call, reason)
    if call.weights is None:
        call.weights = tuple(t.data_ptr() for t in (*model.parameters(), *model.buffers()))
    key = (call.weights, _signature(inputs), tuple(_cache_key(c) for c in _caches(model)))
    graph = current_graph(model)
    if graph is None or graph.key != key:
        model._decode_graph = None   # the old graph and its memory pool go first
        graph = model._decode_graph = DecodeGraph(key, inputs, tokens)
    return graph.step(model, inputs, call)


def current_graph(model) -> Optional[DecodeGraph]:
    """The model's decode graph (None before its first eligible step)."""
    return getattr(model, "_decode_graph", None)
