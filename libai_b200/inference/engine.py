"""Continuous batching: a request-level generation engine on a paged KV cache.

``generate()`` batches statically: a batch is padded to its longest prompt and runs until its slowest sequence ends.
:class:`GenerationEngine` instead lets requests join and leave a running batch at every step.  Each step is one forward
over ``[1, T]`` tokens of a :class:`~libai_b200.inference.kv_cache.RaggedPagedKVCache`: one decode row per slot
(``max_batch`` of them, in slot order; idle ones write and read the cache's sink page), then prompt chunks that fill
the rest of ``max_tokens_per_step``.  The decode rows run the paged split-KV decode kernel and the chunks the ragged
paged flash prefill, each sequence at its own length.

Scheduling rules:

- First come, first served.  A request is admitted when a slot is free and the pool has room for
  ``ceil((prompt + max_new_tokens) / 64)`` pages (capped at the model's maximum length), minus the pages of its prefix
  hit; pages only the prefix index holds count as free and are evicted on demand.  Its pages are reserved at
  admission and there is no preemption, so a running request never runs out of pages.
- Prompt chunks take the step's remaining token budget in admission order; a prompt longer than what is left
  continues in the next step from where it stopped (chunked prefill).
- A token is sampled for every decoding slot and for every prompt whose last chunk ran; one host sync per step reads
  them.  A request finishes on its ``eos_token_id``, after ``max_new_tokens``, or at the model's maximum length; its
  slot and pages are freed in the same step (with ``prefix_caching``, the full pages of the tokens it fed are indexed
  first).
- ``prefix_caching``: at admission the longest cached chain of the prompt's full pages, at most
  ``(len - 1) // 64``, is mapped by reference and only the rest is fed.  The index is cleared when the weights change
  (a parameter's ``data_ptr()`` or ``_version``), as ``generate()``'s is.
- ``decode_graphs``: a step without prompt chunks replays one CUDA graph (:class:`~.decode_graph.DecodeGraph`) of
  ``max_batch`` decode rows, whose inputs are the cache's descriptor buffers; steps with chunks run eagerly.
- ``kv_cache_dtype="fp8"``: the pools hold E4M3 rows with fp32 row scales (the format of ``generate(kv_cache_dtype=
  "fp8")``), about half the bytes of bf16 pages, so the same memory admits about twice the requests.  The ragged FP8
  append writes the rows; the decode rows run the paged FP8 decode kernel and the chunks the FP8 ragged prefill, both
  over the dequantized rows.  Chunked prefill, prefix caching and decode graphs work as on bf16 pools.

Supported models are those whose class sets ``continuous_batching = True`` (their cached step takes positions only
from the cache's per-sequence lengths): the Llama family and BLOOM.  The model's own ``kv_cache`` and decode graph are
left as they are, so ``generate()`` before and after an engine run gives the same outputs.
"""
from __future__ import annotations

import time
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import torch

from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dutil

from .decode_graph import DecodeCall, DecodeGraph
from .generator.generation_logits_processor import (
    LogitsProcessorList,
    TemperatureLogitsWarper,
    TopKLogitsWarper,
    TopPLogitsWarper,
)
from .generator.generation_utils import _kv_cache_dtype
from .kv_cache import RaggedPagedKVCache


@dataclass
class RequestOutput:
    request_id: int
    new_tokens: List[int]
    finished: bool
    finish_reason: Optional[str] = None   # "eos", "length" (max_new_tokens) or "max_length" (the model's)


@dataclass
class _Request:
    id: int
    tokens: List[int]            # the prompt, then the generated tokens
    prompt_len: int
    max_new: int
    eos: Optional[int]
    t_arrival: float
    slot: int = -1
    pages: List[int] = field(default_factory=list)
    fed: int = 0                 # the rows in the cache (prefix hit included)
    t_first: Optional[float] = None
    t_done: Optional[float] = None
    finish_reason: Optional[str] = None

    @property
    def generated(self) -> List[int]:
        return self.tokens[self.prompt_len :]


class _Forward:
    """The engine's cached step in the form :class:`DecodeGraph` drives: ``kv_cache``, ``past_length`` and a call on
    ``{"input_ids", "use_cache"}`` returning the logits."""

    def __init__(self, model, cache: RaggedPagedKVCache):
        self.model, self.kv_cache, self.past_length = model, cache, 0

    def __call__(self, input_ids, use_cache=True):
        return {"logits": self.model.continuous_batching_logits(input_ids, self.kv_cache)}


class GenerationEngine:
    """Continuous batching for a model with ``continuous_batching = True`` (see the module docstring).

    ``num_pages``: the pool's pages of 64 rows per layer (default: room for ``max_batch`` sequences of the model's
    maximum length, or of 2,048 tokens for a model without one).  ``kv_cache_dtype``: None (the weights' dtype), or
    ``"fp8"`` / ``torch.float8_e4m3fn`` for FP8 (E4M3) pools.  Sampling is engine-wide: greedy, or with
    ``do_sample`` temperature / top-k / top-p through ``generate()``'s logits warpers."""

    def __init__(self, model, max_batch: int = 32, max_tokens_per_step: int = 2048, num_pages: Optional[int] = None,
                 prefix_caching: bool = False, decode_graphs: bool = False, do_sample: bool = False,
                 temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0, kv_cache_dtype=None):
        if not getattr(type(model), "continuous_batching", False):
            raise ValueError(f"{type(model).__name__} does not support continuous batching (its cached step does not "
                             "take positions from the cache's per-sequence lengths)")
        if getattr(model, "kv_cache_dtype", None) is not None:
            raise ValueError("the engine's KV dtype is its own kv_cache_dtype argument (e.g. 'fp8' for an FP8 cache), "
                             "not the model's kv_cache_dtype attribute, which generate() sets")
        kv_dtype = _kv_cache_dtype(kv_cache_dtype)
        topo = dutil.get_dist_util()
        if topo.tensor_parallel_size > 1 or topo.pipeline_parallel_size > 1:
            raise ValueError("continuous batching does not run under tensor or pipeline parallelism")
        if max_batch < 1 or max_tokens_per_step <= max_batch:
            raise ValueError(f"need max_batch >= 1 and max_tokens_per_step > max_batch, got {max_batch}, "
                             f"{max_tokens_per_step}")
        P = OF.PAGE_ROWS
        mods = model._cache_attention_modules()
        qkv = mods[0].query_key_value
        w = qkv.weight
        dtype = getattr(qkv, "compute_dtype", None) or w.dtype
        heads = getattr(mods[0], "local_kv_heads", mods[0].local_heads)
        self.max_length = model.continuous_batching_max_length()
        if num_pages is None:
            num_pages = max_batch * -(-(self.max_length or 2048) // P)
        if num_pages < 1:
            raise ValueError(f"num_pages must be >= 1, got {num_pages}")
        max_pages = num_pages if self.max_length is None else min(num_pages, -(-self.max_length // P))
        self.model, self.max_batch, self.max_tokens = model, max_batch, max_tokens_per_step
        self.prefix_caching, self.decode_graphs = prefix_caching, decode_graphs
        self.cache = RaggedPagedKVCache(len(mods), max_batch, heads, mods[0].head_size, num_pages, max_pages,
                                        max_tokens_per_step, dtype, w.device, kv_dtype=kv_dtype)
        self._forward = _Forward(model, self.cache)
        self.do_sample = do_sample
        self.warpers = LogitsProcessorList()
        if do_sample:
            if temperature != 1.0:
                self.warpers.append(TemperatureLogitsWarper(float(temperature)))
            if top_k:
                self.warpers.append(TopKLogitsWarper(top_k=int(top_k)))
            if top_p < 1.0:
                self.warpers.append(TopPLogitsWarper(top_p=top_p))
        self.slots: List[Optional[_Request]] = [None] * max_batch
        self.waiting: List[_Request] = []
        self.requests: Dict[int, _Request] = {}
        self._next_id = 0
        self._graph: Optional[DecodeGraph] = None
        self._graph_call = DecodeCall()
        self.graph_captures = 0     # CUDA graph captures of the decode step
        self.reused_pages = 0       # pages mapped from the prefix index at admission
        self.steps = 0

    # ---- requests -----------------------------------------------------------------------------------------------
    def add_request(self, prompt_ids, max_new_tokens: int = 128, eos_token_id: Optional[int] = None) -> int:
        """Queue a request (``prompt_ids``: a list of ints or a 1-D LongTensor); returns its id.  Raises ``ValueError``
        for one that could never run: an empty prompt, ``max_new_tokens < 1``, a prompt past the model's maximum
        length, or more pages than the pool holds."""
        tokens = [int(t) for t in (prompt_ids.tolist() if torch.is_tensor(prompt_ids) else prompt_ids)]
        if not tokens or max_new_tokens < 1:
            raise ValueError("a request needs at least one prompt token and max_new_tokens >= 1")
        if self.max_length is not None and len(tokens) > self.max_length:
            raise ValueError(f"the prompt's {len(tokens)} tokens run past the model's maximum length "
                             f"{self.max_length}")
        need = self._pages_needed(len(tokens), max_new_tokens)
        if need > self.cache.num_pages or need > self.cache.max_pages:
            raise ValueError(f"the request needs {need} pages of 64 rows; the pool holds {self.cache.num_pages}, "
                             f"a sequence at most {self.cache.max_pages}")
        rid = self._next_id
        self._next_id += 1
        req = _Request(rid, tokens, len(tokens), int(max_new_tokens), eos_token_id, time.perf_counter())
        self.requests[rid] = req
        self.waiting.append(req)
        return rid

    def _pages_needed(self, prompt_len: int, max_new: int) -> int:
        rows = prompt_len + max_new
        if self.max_length is not None:
            rows = min(rows, self.max_length)
        return -(-rows // OF.PAGE_ROWS)

    def has_unfinished(self) -> bool:
        return bool(self.waiting) or any(r is not None for r in self.slots)

    def _admit(self) -> None:
        c = self.cache
        if self.prefix_caching:
            weights = self.model._prefix_cache_weights()
            if c.index_owner != weights:   # the index holds K/V of other weights
                c.clear_prefix_index()
                c.index_owner = weights
        while self.waiting and None in self.slots:
            req = self.waiting[0]
            hit = c.peek(req.tokens) if self.prefix_caching else []
            need = self._pages_needed(req.prompt_len, req.max_new) - len(hit)
            if need > c.available(exclude=set(hit)):
                break   # first come, first served: later requests wait too
            self.waiting.pop(0)
            if hit:
                hit = c.lookup(req.tokens)
                self.reused_pages += len(hit)
            req.pages = hit + c.alloc(need)
            req.fed = len(hit) * OF.PAGE_ROWS
            req.slot = self.slots.index(None)
            self.slots[req.slot] = req

    # ---- a step -------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def step(self) -> List[RequestOutput]:
        """Admit what fits, run one forward over the decode rows and prompt chunks, and sample; returns the tokens
        emitted this step, one :class:`RequestOutput` per request that got one."""
        self._admit()
        if all(r is None for r in self.slots):
            return []
        decode, chunks, samplers = [None] * self.max_batch, [], []
        budget = self.max_tokens - self.max_batch
        for slot, req in enumerate(self.slots):
            if req is not None and req.fed == len(req.tokens) - 1 and len(req.tokens) > req.prompt_len:
                decode[slot] = (req.tokens[-1], req.fed, req.pages)
                samplers.append((slot, req, 1))
        row = self.max_batch
        for req in sorted((r for r in self.slots if r is not None and r.fed < r.prompt_len), key=lambda r: r.id):
            n = min(req.prompt_len - req.fed, budget)
            if n == 0:
                break
            chunks.append((req.tokens[req.fed : req.fed + n], req.fed, req.pages))
            budget -= n
            row += n
            if req.fed + n == req.prompt_len:
                samplers.append((row - 1, req, n))
            else:
                req.fed += n   # the rest of the prompt continues in a later step
        ids, rows = self.cache.write_step(decode, chunks, [s[0] for s in samplers])
        inputs = {"input_ids": ids, "use_cache": True}
        if self.decode_graphs and not chunks and self.cache.device.type == "cuda":
            # keyed by the addresses the capture reads: weights moved to new storage are captured again
            key = tuple(t.data_ptr() for t in (*self.model.parameters(), *self.model.buffers()))
            if self._graph is None or self._graph.key != key:
                self._graph = None   # the old graph and its memory pool go first
                self._graph = DecodeGraph(key, inputs, tokens=self.max_batch)
            captured = self._graph.graph is not None
            logits = self._graph.step(self._forward, inputs, self._graph_call)["logits"]
            self.graph_captures += int(not captured and self._graph.graph is not None)
        else:
            logits = self._forward(**inputs)["logits"]
        self.steps += 1
        outputs = []
        if samplers:
            toks = self._sample(logits[0].index_select(0, rows)).tolist()   # the step's one host sync
            now = time.perf_counter()
            for (_, req, n), tok in zip(samplers, toks):
                req.fed += n
                req.tokens.append(int(tok))
                if req.t_first is None:
                    req.t_first = now
                reason = None
                if req.eos is not None and tok == req.eos:
                    reason = "eos"
                elif len(req.tokens) - req.prompt_len >= req.max_new:
                    reason = "length"
                elif self.max_length is not None and len(req.tokens) >= self.max_length:
                    reason = "max_length"   # the next token has no position left
                if reason is not None:
                    self._finish(req, reason, now)
                outputs.append(RequestOutput(req.id, [int(tok)], reason is not None, reason))
        return outputs

    def _sample(self, logits: torch.Tensor) -> torch.Tensor:
        scores = logits.float()
        if not self.do_sample:
            return scores.argmax(dim=-1)
        scores = self.warpers(None, scores)
        return torch.multinomial(torch.softmax(scores, dim=-1), num_samples=1).squeeze(1)

    def _finish(self, req: _Request, reason: str, now: float) -> None:
        if self.prefix_caching:
            self.cache.insert(req.tokens[: req.fed], req.pages)
        self.cache.release(req.pages)
        req.pages, req.finish_reason, req.t_done = [], reason, now
        self.slots[req.slot] = None

    def generate(self, prompts, max_new_tokens: int = 128, eos_token_id: Optional[int] = None) -> List[List[int]]:
        """Run ``prompts`` (lists of ints or 1-D LongTensors) to completion; returns their new tokens, in input order."""
        ids = [self.add_request(p, max_new_tokens, eos_token_id) for p in prompts]
        while self.has_unfinished():
            self.step()
        return [self.requests[i].generated for i in ids]
