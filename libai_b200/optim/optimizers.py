"""Flat-buffer optimizers with built-in data-parallel gradient sync, ZeRO partitioning, global-norm
clipping and mixed precision (bf16 params + fp32 master).

What the reference gets from OneFlow (``flow.optim.AdamW`` + nn.Graph switches: ZeRO
``graph_base.py:69-70``, fused model update ``:75``, fused cast+scale ``:76``, grad clipping stored
in the param groups ``optim/build.py:86-88`` and applied by ``optimizer.clip_grad()``
``engine/trainer.py:284``) is provided explicitly here, designed around H100:

* every param group lives in ONE contiguous buffer: low-precision params (``param_flat``), fp32
  gradients (``grad_flat`` – the wgmma wgrad kernels accumulate into it directly through
  ``param.main_grad``), fp32 master weights and Adam moments.  One fused kernel launch updates a
  whole group (K18), the gradient norm is one reduction over the flat buffer (K19).
* ``zero_stage >= 1`` partitions master/moments (and the update) over the DP group: the gradient
  all-reduce becomes reduce-scatter → update owned slice → all-gather of the low-precision params
  (K3/K4).  With the native backend the three steps run as one NVLink peer-memory kernel
  (``libai_b200/ops/zero_kernels.py``); the NCCL sequence is the oracle/baseline.

``state_dict()`` returns *logical* tensors keyed by parameter name (ZeRO shards merged, TP shards
gathered) so optimizer checkpoints are layout independent like the reference's.
"""
from __future__ import annotations

import os

import math
from collections import OrderedDict
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from libai_b200 import ops
from libai_b200.ops import count_launch, load_ext, use_native
from libai_b200.ops import impl as ops_impl
from libai_b200.parallel import state as pstate
from libai_b200.utils import distributed as dutil

_ALIGN = 256  # elements; keeps every shard 1 KiB aligned for 128-bit vector access


class _Group:
    """Flat storage of one param group."""

    def __init__(self, params: List[torch.nn.Parameter], dp_size: int, dp_rank: int, sharded: bool,
                 symm_ws=None, index: int = 0):
        self.params = params
        self.symm = None
        self.dtype = params[0].dtype
        self.device = params[0].device
        assert all(p.dtype == self.dtype for p in params), "mixed dtypes inside one param group"
        self.offsets = []
        n = 0
        for p in params:
            self.offsets.append(n)
            n += p.numel()
            n = (n + 7) // 8 * 8  # keep every parameter 16B/32B aligned inside the flat buffer
        chunk = _ALIGN * dp_size
        self.numel = (n + chunk - 1) // chunk * chunk
        if symm_ws is not None:
            # NVLink peer-mapped buffers: the fused ZeRO kernels read peers' gradients and write peers'
            # parameters directly (K3/K4)
            # LIBAI_B200_NVLS=1 (opt-in): bind the buffers to an NVSwitch multicast object — the reduce-scatter then reads
            # in-switch sums (multimem.ld_reduce), the parameter all-gather is one multimem.st per vector.  Off by default:
            # a reduce-SCATTER through the switch still has every GPU send its whole buffer (only the inbound side
            # shrinks), so it cannot beat the unicast pull on full-duplex links; results are bit-identical.
            nvls = os.environ.get("LIBAI_B200_NVLS", "0") == "1" and self.dtype == torch.bfloat16
            pbuf = symm_ws.buffer(("zero_param", index, self.numel, nvls), self.numel * params[0].element_size(), multicast=nvls)
            gbuf = symm_ws.buffer(("zero_grad", index, self.numel, nvls), self.numel * 4, multicast=nvls)
            self.param_flat = pbuf.view(self.dtype, (self.numel,))
            self.grad_flat = gbuf.view(torch.float32, (self.numel,))
            self.symm = dict(ws=symm_ws, param=pbuf, grad=gbuf)
        else:
            self.param_flat = torch.zeros(self.numel, dtype=self.dtype, device=self.device)
            self.grad_flat = torch.zeros(self.numel, dtype=torch.float32, device=self.device)
        for p, off in zip(params, self.offsets):
            self.param_flat[off : off + p.numel()].copy_(p.data.reshape(-1))
            attrs = {k: getattr(p, k) for k in ("tp_dim", "tp_stride", "sequence_parallel", "init_index", "shared_from") if hasattr(p, k)}
            p.data = self.param_flat[off : off + p.numel()].view(p.shape)
            for k, v in attrs.items():
                setattr(p, k, v)
            p.main_grad = self.grad_flat[off : off + p.numel()].view(p.shape)
            p.grad_added_to_main_grad = False
        self.sharded = sharded
        per = self.numel // dp_size if sharded else self.numel
        self.lo = dp_rank * per if sharded else 0
        self.hi = self.lo + per
        self.master = None
        if self.dtype != torch.float32:
            self.master = self.param_flat[self.lo : self.hi].float()
        self.state: Dict[str, torch.Tensor] = {}

    def master_view(self) -> torch.Tensor:
        return self.master if self.master is not None else self.param_flat[self.lo : self.hi]

    def grad_shard(self) -> torch.Tensor:
        return self.grad_flat[self.lo : self.hi]

    def lp_shard(self) -> torch.Tensor:
        """Low-precision parameters of the owned range (what the update writes)."""
        return self.param_flat[self.lo : self.hi]

    def reduced_view(self, lo: int, hi: int) -> torch.Tensor:
        """Reduced gradients of the flat range ``[lo, hi)`` (inside the owned range)."""
        return self.grad_flat[lo:hi]


class FlatOptimizer(torch.optim.Optimizer):
    """Base class: flat buffers + DP sync + ZeRO + clipping; subclasses implement ``_update``."""

    state_names: tuple = ()

    def __init__(self, params, defaults):
        super().__init__(params, defaults)
        self._groups: Optional[List[_Group]] = None
        self.zero_stage = 0
        self.dp_grad_reduce = "mean"
        self._param_names: Dict[int, str] = {}
        self._step_count = 0
        self.grad_scale = 1.0  # multiply grads by this before use (1/loss_scale for fp16)
        self.last_grad_norm: Optional[torch.Tensor] = None
        self.skipped_steps = 0
        self.overlap_grad_sync = False
        self._synced = False
        # ZeRO over NVLink peer memory: reduce-scatter / Adam / all-gather as fused kernels instead of NCCL
        self.fused_zero_comm = True

    # ------------------------------------------------------------------ configuration
    def configure(self, *, zero_stage: int = 0, param_names: Optional[Dict[int, str]] = None,
                  dp_grad_reduce: str = "mean", model=None):
        """Called by the trainer before the first step.  ``model`` (a ``PipelineStageMixin``) lets ZeRO stage 2 / 3 bucket
        the parameters per transformer block (``zero_buckets.py``)."""
        self.zero_stage = int(zero_stage)
        self.dp_grad_reduce = dp_grad_reduce
        self._model = model
        if param_names:
            self._param_names = dict(param_names)
        return self

    @property
    def bucket_hooks(self):
        """Hooks ``forward_stage`` has to call around every block (ZeRO stage 2 / 3), else ``None``."""
        return getattr(self, "_bucket_hooks", None)

    def setup(self):
        """Materialise the flat buffers (idempotent). Must run before the first forward so that
        ``param.main_grad`` exists for the wgrad kernels."""
        if self._groups is not None:
            return self
        topo = dutil.get_dist_util()
        sharded = self.zero_stage >= 1 and topo.data_parallel_size > 1
        self._groups = []
        self._hp_index: List[int] = []          # param_groups index of every entry of _groups
        if sharded and self.zero_stage >= 2:
            # gradients (stage 2) / parameters too (stage 3) partitioned: per-block buckets, see zero_buckets.py
            from .zero_buckets import ZeroBucketHooks, build_buckets

            per_group, by_layer = build_buckets(self.param_groups, getattr(self, "_model", None),
                                                topo.data_parallel_size, topo.dp_rank, self.zero_stage)
            for gi, buckets in enumerate(per_group):
                for b in buckets:
                    for name in self.state_names:
                        b.state[name] = torch.zeros(b.per, dtype=torch.float32, device=b.device)
                    self._groups.append(b)
                    self._hp_index.append(gi)
            self._bucket_hooks = ZeroBucketHooks(by_layer, self.dp_grad_reduce, self.zero_stage) if by_layer else None
            if not by_layer:
                import logging

                logging.getLogger(__name__).warning(
                    "ZeRO stage %d: the model exposes no `stage_layers()` blocks — all parameters form one resident "
                    "bucket (memory profile of stage 1)", self.zero_stage)
            return self
        for gi, g in enumerate(self.param_groups):
            params = [p for p in g["params"] if p.device.type != "meta" and p.requires_grad]
            self._hp_index.append(gi)
            if not params:
                self._groups.append(None)
                continue
            ws = None
            if (sharded and self.fused_zero_comm and params[0].is_cuda and params[0].dtype == torch.bfloat16
                    and ops_impl() == "native" and topo.data_parallel_size <= 8 and self.zero_stage == 1):
                from libai_b200.parallel.symm_mem import get_workspace

                ws = get_workspace(topo.dp_group)
            fg = _Group(params, topo.data_parallel_size, topo.dp_rank, sharded, symm_ws=ws, index=gi)
            for name in self.state_names:
                fg.state[name] = torch.zeros(fg.hi - fg.lo, dtype=torch.float32, device=fg.device)
            self._groups.append(fg)
        return self

    # ------------------------------------------------------------------ gradients
    def zero_grad(self, set_to_none: bool = True):
        self.setup()
        for fg in self._groups:
            if fg is None:
                continue
            if hasattr(fg, "red"):           # ZeRO-2/3 bucket: the persistent piece is the reduced-gradient shard
                fg.red.zero_()
                if fg.grad_flat is not None:
                    fg.grad_flat.zero_()
                for p in fg.params:
                    p.grad = None
                    p.grad_added_to_main_grad = False
                continue
            fg.grad_flat.zero_()
            fg.reduced_from = fg.hi          # nothing of the owned slice has been reduced yet
            if getattr(fg, "sq_partial", None) is not None:
                fg.sq_partial.zero_()
            for p in fg.params:
                p.grad = None
                p.grad_added_to_main_grad = False
        self._synced = False
        self._early_launched = False

    # ---- early (overlapped) data-parallel reduction ------------------------------------------------
    _LAYER_RE = None

    def plan_overlap(self, num_triggers: int = 4):
        """Decide at which block boundaries of the backward pass the gradient reduce-scatter of the already-final tail
        of each flat buffer is started.  Parameters are laid out in registration order (embeddings, block 0 … block
        L-1, final norm), backward finishes them in reverse, so after the backward of block ``i`` everything from the
        first parameter of block ``i`` to the end of the buffer is final.  Returns the trigger layer indices (empty
        when the layout does not allow it: model-parallel fix-ups pending, no fused NVLink path, unknown names)."""
        import re

        self.setup()
        topo = dutil.get_dist_util()
        self._overlap_plan = {}
        if (topo.dp_group is None or topo.pipeline_parallel_size > 1
                or (topo.sequence_parallel and topo.tensor_parallel_size > 1)):
            return ()
        pat = re.compile(r"\.layers\.(\d+)\.")
        layers_seen = set()
        per_group = []
        for fg in self._groups:
            if fg is None or fg.symm is None:
                per_group.append(None)
                continue
            idx = []
            for p in fg.params:
                m = pat.search(self._param_names.get(id(p), ""))
                idx.append(int(m.group(1)) if m else None)
            known = [i for i in idx if i is not None]
            if not known:
                per_group.append(None)
                continue
            first, last = idx.index(known[0]), len(idx) - 1 - idx[::-1].index(known[-1])
            # registration order must be monotone in the block index between the first and last block parameter
            body = [i for i in idx[first:last + 1] if i is not None]
            if body != sorted(body):
                per_group.append(None)
                continue
            start = {}
            for k in range(first, last + 1):
                if idx[k] is not None and idx[k] not in start:
                    start[idx[k]] = (k, fg.offsets[k])
            per_group.append(dict(idx=idx, start=start, first=first))
            layers_seen.update(start)
        if not layers_seen or all(g is None for g in per_group):
            return ()
        n_layers = max(layers_seen) + 1
        step = max(1, n_layers // (num_triggers + 1))
        triggers = tuple(sorted({l for l in range(step, n_layers, step)} & layers_seen))
        self._overlap_plan = dict(groups=per_group, triggers=triggers)
        return triggers

    def on_grads_ready(self, layer_idx: int):
        """Called from the backward pass (``_GradBoundary``) of the last micro-batch: gradients of block ``layer_idx``
        and everything registered after it are final.  Every rank launches the reduce-scatter of the part of ITS slice
        that lies in that tail on a side stream; the kernel's own flag exchange makes sure the peers got there too."""
        plan = getattr(self, "_overlap_plan", None)
        if not plan or layer_idx not in plan["triggers"]:
            return
        topo = dutil.get_dist_util()
        ext = load_ext()
        if getattr(self, "_side_stream", None) is None:
            self._side_stream = torch.cuda.Stream()
        work = []
        for fg, gp in zip(self._groups, plan["groups"]):
            if fg is None or gp is None or layer_idx not in gp["start"]:
                continue
            k0, off = gp["start"][layer_idx]
            # everything in the tail must already sit in main_grad (the native backward accumulates there directly;
            # a parameter still waiting for autograd's AccumulateGrad cannot be reduced early)
            if not all(p.grad_added_to_main_grad and p.grad is None for p in fg.params[k0:]):
                return
            # parameter offsets are multiples of 8 elements and slice bounds multiples of 256: float4-aligned
            a = min(max(off, fg.lo), fg.reduced_from)
            work.append((fg, a))
        if not work:
            return
        ev = torch.cuda.Event()
        ev.record()
        self._side_stream.wait_event(ev)
        scale = 1.0 / topo.data_parallel_size if self.dp_grad_reduce == "mean" else 1.0
        with torch.cuda.stream(self._side_stream):
            for fg, a in work:
                ws = fg.symm["ws"]
                b = fg.reduced_from
                if getattr(fg, "sq_partial", None) is None:
                    fg.sq_partial = torch.zeros(1, dtype=torch.float32, device=fg.device)
                # (an empty range still takes part in the flag exchange: all ranks issue the same launch sequence)
                ext.zero_reduce_scatter(fg.symm["grad"].peer_ptrs(0), ws.flags.peer_ptrs(0), fg.grad_flat[a:b],
                                        fg.sq_partial, a, b - a, scale, ws.world, ws.rank, ws.next_epoch(),
                                        fg.symm["grad"].mc_ptr)
                count_launch()
                fg.reduced_from = a
        self._early_launched = True

    def _collect_autograd_grads(self):
        """Fold ``p.grad`` (produced by the PyTorch reference path) into ``main_grad``."""
        for fg in self._groups:
            if fg is None or hasattr(fg, "red"):
                continue
            for p in fg.params:
                if p.grad is not None:
                    p.main_grad.add_(p.grad.to(torch.float32))
                    p.grad = None

    def sync_gradients(self):
        """Model-parallel fix-ups + data-parallel reduction of the flat gradient buffers."""
        self.setup()
        if self._synced:
            return
        self._collect_autograd_grads()
        topo = dutil.get_dist_util()
        if self.bucket_hooks is not None:
            self.bucket_hooks.flush()           # the last block's reduce-scatter may still be in flight
        for fg in self._groups:
            if fg is None:
                continue
            if hasattr(fg, "red"):
                # ZeRO-2/3: block buckets were reduce-scattered from the backward hooks; what is still open here are
                # the persistent buckets (embeddings / heads / final norm) and blocks that ran outside forward_stage
                scale = 1.0 / topo.data_parallel_size if self.dp_grad_reduce == "mean" else 1.0
                if fg.grad_flat is None and any(p.grad is not None for p in fg.params):
                    fg.open_grads()
                fg.reduce_grads(topo, scale)
                continue
            # (1) parameters replicated over TP whose grads were computed on token shards (LayerNorm γ/β, row-parallel
            # biases): ONE all-reduce over a packed buffer instead of one tiny NCCL call per parameter (≈150 per step
            # for the 24-layer model — host launch latency, not bandwidth, was the cost)
            if topo.sequence_parallel and topo.tp_group is not None:
                sp_grads = [p.main_grad.view(-1) for p in fg.params if getattr(p, "sequence_parallel", False)]
                if len(sp_grads) == 1:
                    dist.all_reduce(sp_grads[0], group=topo.tp_group)
                elif sp_grads:
                    packed = torch.cat(sp_grads)
                    dist.all_reduce(packed, group=topo.tp_group)
                    torch._foreach_copy_(sp_grads, list(packed.split([g.numel() for g in sp_grads])))
            # (2) tied embeddings living on first and last pipeline stage
            if topo.embedding_group is not None:
                for p in fg.params:
                    if getattr(p, "shared_from", None) is not None or getattr(p, "is_tied_source", False):
                        dist.all_reduce(p.main_grad, group=topo.embedding_group)
            # (3) data parallel
            if topo.dp_group is not None and fg.symm is not None:
                ext = load_ext()
                ws = fg.symm["ws"]
                scale = 1.0 / topo.data_parallel_size if self.dp_grad_reduce == "mean" else 1.0
                if getattr(fg, "sq_partial", None) is None:
                    fg.sq_partial = torch.zeros(1, dtype=torch.float32, device=fg.device)
                if getattr(self, "_early_launched", False):
                    # the tail [reduced_from, hi) was reduced during the backward pass on the side stream
                    torch.cuda.current_stream().wait_stream(self._side_stream)
                b = getattr(fg, "reduced_from", fg.hi)
                if b == fg.hi:
                    fg.sq_partial.zero_()
                ext.zero_reduce_scatter(fg.symm["grad"].peer_ptrs(0), ws.flags.peer_ptrs(0), fg.grad_flat[fg.lo:b],
                                        fg.sq_partial, fg.lo, b - fg.lo, scale, ws.world, ws.rank, ws.next_epoch(),
                                        fg.symm["grad"].mc_ptr)
                count_launch()
                fg.reduced_from = fg.lo
            elif topo.dp_group is not None:
                if self.dp_grad_reduce == "mean":
                    fg.grad_flat.div_(topo.data_parallel_size)
                if fg.sharded and fg.device.type == "cuda":
                    dist.reduce_scatter_tensor(fg.grad_shard(), fg.grad_flat, group=topo.dp_group)
                else:
                    dist.all_reduce(fg.grad_flat, group=topo.dp_group)
        self._synced = True

    # ------------------------------------------------------------------ clipping
    def _global_grad_norm(self, norm_type: float) -> torch.Tensor:
        """Norm over *all* parameters of the model-parallel group (each logical element once)."""
        topo = dutil.get_dist_util()
        dev = None
        total = None
        def _acc(seg):
            if math.isinf(norm_type):
                return seg.abs().max() if seg.numel() else torch.zeros((), device=seg.device)
            if norm_type == 2.0:
                if (seg.numel() and seg.dtype == torch.float32 and seg.is_contiguous() and seg.data_ptr() % 16 == 0
                        and use_native(seg)):
                    # one pass over the flat fp32 gradient buffer (K19); `pow(2).sum()` would write and re-read a
                    # temporary as large as the buffer (1.4 GB for the 345M-parameter benchmark model)
                    count_launch()
                    return load_ext().sqnorm(seg).reshape(())
                return torch.dot(seg.reshape(-1), seg.reshape(-1)) if seg.numel() else torch.zeros((), device=seg.device)
            return seg.abs().pow(norm_type).sum()

        for fg in self._groups:
            if fg is None:
                continue
            dev = fg.device
            # every logical element once: skip TP-replicated parameters on tp_rank != 0 and the
            # last-stage copy of tied weights (their gradients are identical duplicates)
            skip = []
            for p, off in zip(fg.params, fg.offsets):
                dup_tp = topo.tensor_parallel_size > 1 and getattr(p, "tp_dim", None) is None and topo.tp_rank != 0
                dup_tied = getattr(p, "shared_from", None) is not None
                if dup_tp or dup_tied:
                    lo, hi = max(off, fg.lo), min(off + p.numel(), fg.hi)
                    if lo < hi:
                        skip.append((lo, hi))
            view = fg.reduced_view
            if math.isinf(norm_type) and skip:
                acc = torch.zeros((), dtype=torch.float32, device=dev)
                cur = fg.lo
                for lo, hi in skip + [(fg.hi, fg.hi)]:
                    if cur < lo:
                        acc = torch.maximum(acc, _acc(view(cur, lo)))
                    cur = max(cur, hi)
            else:
                acc = _acc(fg.grad_shard())
                if skip:
                    # ONE reduction over the packed duplicates (≈150 LayerNorm / bias segments under tensor parallelism:
                    # one kernel per segment made the step host-bound on tp_rank != 0)
                    merged = []
                    for lo, hi in skip:
                        if merged and merged[-1][1] + 8 >= lo:       # neighbours (≤ alignment padding apart, zeros)
                            merged[-1] = (merged[-1][0], hi)
                        else:
                            merged.append((lo, hi))
                    dup = torch.cat([view(lo, hi) for lo, hi in merged]) if len(merged) > 1 else view(merged[0][0], merged[0][1])
                    acc = acc - (torch.dot(dup, dup) if norm_type == 2.0 else dup.abs().pow(norm_type).sum())
            total = acc if total is None else (torch.maximum(total, acc) if math.isinf(norm_type) else total + acc)
        if total is None:
            total = torch.zeros((), dtype=torch.float32, device=dutil.get_device())
        op = dist.ReduceOp.MAX if math.isinf(norm_type) else dist.ReduceOp.SUM
        if dist.is_initialized() and topo.world_size > 1:
            sharded = any(fg is not None and fg.sharded for fg in self._groups)
            if sharded and topo.dp_group is not None:
                dist.all_reduce(total, op=op, group=topo.dp_group)
            if topo.tp_group is not None:
                dist.all_reduce(total, op=op, group=topo.tp_group)
            if topo.pp_group is not None:
                dist.all_reduce(total, op=op, group=topo.pp_group)
        if not math.isinf(norm_type):
            total = total.pow(1.0 / norm_type)
        return total * self.grad_scale

    def clip_grad(self):
        """Reference-API entry point (``optimizer.clip_grad()``): computes the clip coefficient
        that ``step`` folds into the update.  Calling it is optional – ``step`` does it."""
        self.sync_gradients()
        g0 = next((g for g in self.param_groups if "clip_grad_max_norm" in g), None)
        if g0 is None:
            self._clip_coef = None
            return None
        max_norm = float(g0["clip_grad_max_norm"])
        norm = self._global_grad_norm(float(g0["clip_grad_norm_type"]))
        self.last_grad_norm = norm
        self._clip_coef = torch.clamp(max_norm / (norm + 1e-6), max=1.0)
        return norm

    # ------------------------------------------------------------------ step
    @torch.no_grad()
    def step(self, closure=None):
        self.setup()
        self.sync_gradients()
        if not hasattr(self, "_clip_coef") or self._clip_coef is None:
            self.clip_grad()
        coef = self._clip_coef
        self._clip_coef = None
        # fp16 dynamic loss scaling: skip the update on overflow (decided by the scaler)
        if getattr(self, "found_inf", False):
            self.skipped_steps += 1
            self.found_inf = False
            # The fused ZeRO update ends with a cross-rank barrier that keeps a fast rank from zeroing / refilling its
            # gradient buffer while a slow peer still pulls from it in the reduce-scatter.  A skipped step skips that
            # kernel, so it must keep the barrier.
            for fg in self._groups:
                if fg is not None and fg.symm is not None:
                    ws = fg.symm["ws"]
                    load_ext().device_barrier(ws.flags.peer_ptrs(0), ws.world, ws.rank, 3, ws.next_epoch())
                    count_launch()
                    break
            return None
        self._step_count += 1
        ops.bump_fp8_weight_epoch()     # parameters are rewritten in place: cached E4M3 weight copies are stale
        topo = dutil.get_dist_util()
        for gi, fg in zip(self._hp_index, self._groups):
            if fg is None:
                continue
            g = self.param_groups[gi]
            scale = coef * self.grad_scale if coef is not None else None
            if fg.symm is not None and hasattr(self, "_fused_zero_update"):
                self._fused_zero_update(g, fg, self._step_count, scale)
                continue
            self._update(g, fg, self._step_count, scale)
            if hasattr(fg, "red"):
                fg.publish_params(topo.dp_group)      # ZeRO-2 (and resident buckets of ZeRO-3): refresh the full copy
                continue
            if fg.sharded:
                shard = fg.param_flat[fg.lo : fg.hi]
                if fg.device.type == "cuda":
                    dist.all_gather_into_tensor(fg.param_flat, shard, group=topo.dp_group)
                else:
                    parts = [torch.empty_like(shard) for _ in range(topo.data_parallel_size)]
                    dist.all_gather(parts, shard.clone(), group=topo.dp_group)
                    fg.param_flat.copy_(torch.cat(parts))
        return None

    def _update(self, group: dict, fg: _Group, step: int, scale: Optional[torch.Tensor]):
        raise NotImplementedError

    # ------------------------------------------------------------------ (de)serialisation
    def _names(self, fg: _Group) -> List[str]:
        if not hasattr(self, "_positional_names"):
            # fallback when no names were configured: position in the optimizer's param groups (stable across runs)
            self._positional_names = {}
            k = 0
            for g in self.param_groups:
                for p in g["params"]:
                    self._positional_names[id(p)] = f"param_{k}"
                    k += 1
        return [self._param_names.get(id(p), self._positional_names.get(id(p), f"param_{id(p)}")) for p in fg.params]

    def _gather_shard(self, fg: _Group, shard: torch.Tensor) -> torch.Tensor:
        topo = dutil.get_dist_util()
        if not fg.sharded:
            return shard
        parts = [torch.empty_like(shard) for _ in range(topo.data_parallel_size)]
        dist.all_gather(parts, shard.contiguous(), group=topo.dp_group)
        return torch.cat(parts)

    def state_dict(self):
        """Logical state: ``{"state": {param_name: {state_name: full tensor}}, "param_groups", "step"}``.
        Collective (all ranks call); complete on rank 0."""
        self.setup()
        topo = dutil.get_dist_util()
        local = OrderedDict()
        for fg in self._groups:
            if fg is None:
                continue
            fulls = {k: self._gather_shard(fg, v) for k, v in fg.state.items()}
            if fg.master is not None:
                fulls["master"] = self._gather_shard(fg, fg.master)
            for p, off, name in zip(fg.params, fg.offsets, self._names(fg)):
                entry = {}
                for k, flat in fulls.items():
                    t = flat[off : off + p.numel()].view(p.shape)
                    t = pstate.gather_tp(t, getattr(p, "tp_dim", None))
                    if topo.dp_rank == 0 and topo.tp_rank == 0:
                        entry[k] = t.cpu()
                if entry:
                    local[name] = entry
        if topo.pipeline_parallel_size > 1 and dist.is_initialized():
            parts = dutil.all_gather_py_object(local if (topo.dp_rank == 0 and topo.tp_rank == 0) else None)
            if dutil.get_rank() == 0:
                local = OrderedDict()
                for part in parts:
                    if part:
                        local.update(part)
        groups = [{k: v for k, v in g.items() if k != "params"} for g in self.param_groups]
        return {"state": local, "param_groups": groups, "step": self._step_count}

    def refresh_master(self):
        """Re-derive the fp32 master weights from the (low-precision) parameters.  Must run after model weights were
        written behind the optimizer's back (``train.load_weight``, a checkpoint without ``master`` entries): the
        master copy is what ``step`` updates and writes back, so a stale one silently discards the loaded weights."""
        if self._groups is None:
            return self
        with torch.no_grad():
            for fg in self._groups:
                if fg is None:
                    continue
                if hasattr(fg, "red"):
                    if fg.param_flat is not None:       # (non-resident ZeRO-3 buckets: see params_materialized)
                        fg.adopt_param_values()
                elif fg.master is not None:
                    fg.master.copy_(fg.param_flat[fg.lo : fg.hi])
        ops.bump_fp8_weight_epoch()
        return self

    def params_materialized(self, writeback: bool = False):
        """Context manager: every parameter holds its full, current value while inside (ZeRO stage 3 keeps block
        parameters as 1/dp shards between uses) — checkpoint save / load, weight loaders and anything else that reads or
        writes ``model.parameters()`` directly must run inside.  ``writeback``: the values were modified (a checkpoint
        was loaded): every rank takes its slice back as shard + fp32 master on exit."""
        from contextlib import contextmanager

        @contextmanager
        def ctx():
            self.setup()
            topo = dutil.get_dist_util()
            opened = []
            for fg in self._groups:
                if fg is not None and hasattr(fg, "red") and fg.param_flat is None:
                    fg.gather_params(topo.dp_group)
                    opened.append(fg)
            try:
                yield self
            finally:
                for fg in self._groups:
                    if fg is not None and hasattr(fg, "red") and writeback and fg.param_flat is not None:
                        fg.adopt_param_values()
                for fg in opened:
                    fg.release_params()

        return ctx()

    def load_state_dict(self, sd):
        self.setup()
        ops.bump_fp8_weight_epoch()
        self._step_count = int(sd.get("step", 0))
        for g, saved in zip(self.param_groups, sd.get("param_groups", [])):
            for k, v in saved.items():
                if k != "params":
                    g[k] = v
        state = sd.get("state", {})
        for fg in self._groups:
            if fg is None:
                continue
            for p, off, name in zip(fg.params, fg.offsets, self._names(fg)):
                entry = state.get(name)
                if entry is None and getattr(p, "shared_from", None) is not None:
                    # tied-weight copy on the last pipeline stage: take the source parameter's state
                    prefix = name.rsplit(".", 1)[0] + "." if "." in name else ""
                    entry = state.get(prefix + p.shared_from)
                if entry is None:
                    continue
                lo, hi = max(off, fg.lo), min(off + p.numel(), fg.hi)
                if lo >= hi:
                    continue
                for k, full in entry.items():
                    local = pstate.shard_tp(full, getattr(p, "tp_dim", None)).reshape(-1)
                    seg = local[lo - off : hi - off].to(fg.device, torch.float32)
                    if k == "master":
                        if fg.master is not None:
                            fg.master[lo - fg.lo : hi - fg.lo].copy_(seg)
                    elif k in fg.state:
                        fg.state[k][lo - fg.lo : hi - fg.lo].copy_(seg)


class AdamW(FlatOptimizer):
    """AdamW with decoupled weight decay: ``p ← p − lr·(m̂/(√v̂+ε) + wd·p)`` (reference defaults:
    configs/common/optim.py:6-20 – lr 1e-4, wd 0.01, betas (0.9, 0.999), bias correction on)."""

    state_names = ("exp_avg", "exp_avg_sq")
    decoupled = True

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=False,
                 do_bias_correction=True, **unused):
        if amsgrad:
            raise NotImplementedError("amsgrad is not supported")
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay,
                        do_bias_correction=do_bias_correction)
        super().__init__(params, defaults)

    def _update(self, group, fg, step, scale):
        lr, (b1, b2), eps, wd = group["lr"], group["betas"], group["eps"], group["weight_decay"]
        if group.get("do_bias_correction", True):
            bc1, bc2 = 1.0 - b1 ** step, 1.0 - b2 ** step
        else:
            bc1 = bc2 = 1.0
        g = fg.grad_shard()
        m, v = fg.state["exp_avg"], fg.state["exp_avg_sq"]
        master = fg.master_view()
        if use_native(g):
            ext = load_ext()
            scale_t = scale if scale is not None else torch.ones((), dtype=torch.float32, device=g.device)
            out_lp = fg.lp_shard() if fg.master is not None else None
            ext.fused_adamw(master, g, m, v, out_lp, scale_t.reshape(1).float(), float(lr), float(b1), float(b2),
                            float(eps), float(wd), float(bc1), float(bc2), bool(self.decoupled))
            count_launch()
            return
        if scale is not None:
            g = g * scale
        if not self.decoupled and wd != 0.0:
            g = g + wd * master
        m.mul_(b1).add_(g, alpha=1.0 - b1)
        v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
        denom = (v / bc2).sqrt_().add_(eps)
        upd = (m / bc1) / denom
        if self.decoupled and wd != 0.0:
            upd = upd + wd * master
        master.add_(upd, alpha=-lr)
        if fg.master is not None:
            fg.lp_shard().copy_(master)


    def _fused_zero_update(self, group, fg, step, scale):
        """AdamW on the owned slice + all-gather of the bf16 parameters by P2P stores, one kernel."""
        ext = load_ext()
        ws = fg.symm["ws"]
        lr, (b1, b2), eps, wd = group["lr"], group["betas"], group["eps"], group["weight_decay"]
        bc1, bc2 = (1.0 - b1 ** step, 1.0 - b2 ** step) if group.get("do_bias_correction", True) else (1.0, 1.0)
        clip = scale if scale is not None else torch.ones((), dtype=torch.float32, device=fg.device)
        ext.zero_adam_allgather(
            fg.master, fg.grad_shard(), fg.state["exp_avg"], fg.state["exp_avg_sq"], fg.symm["param"].peer_ptrs(0),
            ws.flags.peer_ptrs(0), ws.done_counter[0:1], clip.reshape(1).float(), fg.lo, fg.hi - fg.lo, float(lr),
            float(b1), float(b2), float(eps), float(wd), float(bc1), float(bc2), bool(self.decoupled), ws.world, ws.rank,
            ws.next_epoch(), fg.symm["param"].mc_ptr,
        )
        count_launch()


class Adam(AdamW):
    """Adam with L2 (coupled) weight decay."""

    decoupled = False


class SGD(FlatOptimizer):
    state_names = ("momentum_buffer",)

    def __init__(self, params, lr=1e-3, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False, **unused):
        defaults = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay, nesterov=nesterov)
        super().__init__(params, defaults)

    def _update(self, group, fg, step, scale):
        lr, mom, damp, wd, nest = (group[k] for k in ("lr", "momentum", "dampening", "weight_decay", "nesterov"))
        g = fg.grad_shard()
        if scale is not None:
            g = g * scale
        master = fg.master_view()
        if wd != 0.0:
            g = g + wd * master
        if mom != 0.0:
            buf = fg.state["momentum_buffer"]
            if step == 1:
                buf.copy_(g)
            else:
                buf.mul_(mom).add_(g, alpha=1.0 - damp)
            g = g + mom * buf if nest else buf
        master.add_(g, alpha=-lr)
        if fg.master is not None:
            fg.lp_shard().copy_(master)


class LAMB(FlatOptimizer):
    """Layer-wise adaptive moments (You et al. 2019) on the flat buffers: Adam direction per element, then one trust
    ratio ``‖w‖ / ‖update‖`` per *parameter tensor*.  Used by the ResMLP recipe (reference configs/resmlp_imagenet.py:52
    selects ``flow.optim.LAMB``).  Under ZeRO the per-tensor norms are completed with one all-reduce over the
    data-parallel group (a shard may cut through a tensor)."""

    state_names = ("exp_avg", "exp_avg_sq")

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.0, adam_w_mode=True,
                 do_bias_correction=True, **unused):
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, adam_w_mode=adam_w_mode,
                        do_bias_correction=do_bias_correction)
        super().__init__(params, defaults)

    def _update(self, group, fg, step, scale):
        lr, (b1, b2), eps, wd = group["lr"], group["betas"], group["eps"], group["weight_decay"]
        bc1, bc2 = (1.0 - b1 ** step, 1.0 - b2 ** step) if group.get("do_bias_correction", True) else (1.0, 1.0)
        g = fg.grad_shard()
        if scale is not None:
            g = g * scale
        master = fg.master_view()
        m, v = fg.state["exp_avg"], fg.state["exp_avg_sq"]
        if not group.get("adam_w_mode", True) and wd != 0.0:
            g = g + wd * master
        m.mul_(b1).add_(g, alpha=1.0 - b1)
        v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
        upd = (m / bc1) / ((v / bc2).sqrt_().add_(eps))
        if group.get("adam_w_mode", True) and wd != 0.0:
            upd.add_(master, alpha=wd)
        # per-tensor squared norms over the part of each tensor that lives in [lo, hi)
        n = len(fg.params)
        sq = torch.zeros(2, n, dtype=torch.float32, device=master.device)
        spans = []
        for i, (p, off) in enumerate(zip(fg.params, fg.offsets)):
            a, b = max(off, fg.lo) - fg.lo, min(off + p.numel(), fg.hi) - fg.lo
            spans.append((a, b))
            if b > a:
                sq[0, i] = master[a:b].pow(2).sum()
                sq[1, i] = upd[a:b].pow(2).sum()
        if fg.sharded:
            topo = dutil.get_dist_util()
            if topo.data_parallel_size > 1:
                dist.all_reduce(sq, group=topo.dp_group)
        w_norm, u_norm = sq[0].sqrt(), sq[1].sqrt()
        trust = torch.where((w_norm > 0) & (u_norm > 0), w_norm / u_norm, torch.ones_like(w_norm))
        for i, (a, b) in enumerate(spans):
            if b > a:
                master[a:b].add_(upd[a:b] * trust[i], alpha=-lr)
        if fg.master is not None:
            fg.lp_shard().copy_(master)
