"""CUDA-graph capture of the transformer blocks.

A training step of the 24-layer benchmark model issues ≈820 kernels, so the time the host needs to enqueue them is
comparable to the device time of a small step (``bench.py`` reports ``host_enqueue_ms_per_step``).  The blocks are where the launches are (≈14 forward + ≈20 backward kernels each), they
have static shapes and no host synchronisation, so each block's forward and backward are captured once into CUDA graphs
(``torch.cuda.make_graphed_callables``) and replayed: 48 graph launches replace ≈800 kernel launches per step.

Why this works with the native backward: the wgrad / bias-grad / LayerNorm-grad kernels accumulate straight into the
optimizer's persistent fp32 ``main_grad`` buffer and return ``None`` to autograd — those kernels (and the TMA
descriptors they were launched with, which are by-value kernel parameters) are part of the captured backward graph and
replay against the same addresses.  Parameters live in the optimizer's flat buffer, i.e. at fixed addresses as well.

Tensor-parallel blocks are captured too when the collectives are the fused ones (``train.dist.fused_tp_comm``): the
AG→GEMM / GEMM→RS kernels keep their call counters, arrival targets and write credits in device memory and advance them
themselves, so a replay is indistinguishable from a fresh launch.

Not captured: embedding, LM head + loss, optimizer, NCCL collectives.  Restrictions (checked): besides the hidden state a
block may take model buffers as keyword tensors (RoPE tables — Llama) and a right-padded ``KeyPaddingMask`` (BERT,
RoBERTa: its key lengths become a second graph input); no activation checkpointing.  Dropout inside captured blocks draws its Philox offset
from a device counter that the dropout kernels advance (``ops/functional.py``), so replays produce fresh masks.
"""
from __future__ import annotations

import logging
from typing import List, Optional, Sequence

import torch
from torch import nn

from libai_b200 import ops

logger = logging.getLogger(__name__)


def _with_launch_count(block: nn.Module, fwd_kernels: int, bwd_kernels: int) -> nn.Module:
    """The kernels inside a replayed graph are still launches of our kernels: keep ``ops.launch_count()`` honest.
    (``make_graphed_callables`` patches ``block.forward`` in place, so module names / state-dict keys are unchanged.)"""
    graphed_forward = block.forward

    def forward(hidden):
        ops.count_launch(fwd_kernels + (bwd_kernels if torch.is_grad_enabled() and block.training else 0))
        return graphed_forward(hidden)

    block.forward = forward
    return block


def graph_transformer_blocks(blocks: Sequence[nn.Module], sample_hidden: torch.Tensor, warmup_iters: int = 3
                             ) -> Optional[List[nn.Module]]:
    """Capture ``blocks`` (called as ``block(hidden)``) for inputs shaped like ``sample_hidden``.  Returns the graphed
    replacements, or ``None`` (with a log line) when a precondition does not hold."""
    if not sample_hidden.is_cuda:
        return None
    # (dropout inside the blocks is fine: the native kernels take their Philox (seed, offset) from PyTorch's CUDA
    # generator, which hands out graph-safe state during capture and refreshes the offset before every replay)
    # Per-block kernel counts for the launch bookkeeping.  The forward count comes from a no-grad eager call (it also
    # makes sure every lazy one-time setup has happened: cudaFuncSetAttribute, extension load, driver entry points);
    # the backward count from the warm-up + capture passes below.  No eager *backward* here: it would leave
    # AccumulateGrad nodes bound to the current stream, and the capture stream would then depend on uncaptured work
    # (cudaErrorStreamCaptureIsolation).
    with torch.no_grad():
        n0 = ops.launch_count()
        blocks[0](sample_hidden.detach())
        fwd_kernels = ops.launch_count() - n0
    torch.cuda.synchronize()
    samples = tuple((sample_hidden.detach().clone().requires_grad_(True),) for _ in blocks)
    n0 = ops.launch_count()
    graphed = torch.cuda.make_graphed_callables(tuple(blocks), samples, num_warmup_iters=warmup_iters,
                                                allow_unused_input=True)
    per_block = (ops.launch_count() - n0) // ((warmup_iters + 1) * len(blocks))
    ops.count_launch(-(ops.launch_count() - n0))          # warm-up / capture launches are not training launches
    graphed = graphed if isinstance(graphed, (tuple, list)) else (graphed,)
    counts = [(fwd_kernels, max(per_block - fwd_kernels, 0))] * len(blocks)
    return [_with_launch_count(g, f, b) for g, (f, b) in zip(graphed, counts)]


# --------------------------------------------------------------------------------------------------------------------
# pipeline parallelism: several micro-batches of one block are in flight (1F1B), so every block gets `n_slots` captured
# copies — micro-batch i runs (forward, and later backward) on copy i % n_slots, whose saved activations nobody else
# touches in between (stage s of p keeps at most p - s micro-batches in flight, FIFO).
# --------------------------------------------------------------------------------------------------------------------
_CURRENT_SLOT = 0


def set_micro_batch_slot(i: int) -> None:
    """Called by the pipeline schedule before the forward of micro-batch ``i``."""
    global _CURRENT_SLOT
    _CURRENT_SLOT = int(i)


class BlockCallSpec:
    """How a model calls its blocks besides the hidden state (discovered from one eager call):

    * ``const_kwargs`` – keyword tensors that are buffers of the model (RoPE cos/sin tables): the same storage on every
      call, so the captured kernels simply keep reading it;
    * ``key_lengths`` – the block takes a ``KeyPaddingMask`` as second positional argument (BERT / RoBERTa): its
      per-sample key lengths (int32 ``[b]``) become a second *graph input*, copied into the static buffer on replay.
    """

    def __init__(self, const_kwargs=None, key_lengths: Optional[torch.Tensor] = None):
        self.const_kwargs = dict(const_kwargs or {})
        self.key_lengths = key_lengths

    @property
    def trivial(self) -> bool:
        return not self.const_kwargs and self.key_lengths is None

    def matches(self, args, kwargs) -> bool:
        """Can this call be served by the captured graph?  (Otherwise the caller runs the eager block.)"""
        live = {k: v for k, v in kwargs.items() if v is not None}
        if set(live) != set(self.const_kwargs) or any(live[k] is not self.const_kwargs[k] for k in live):
            return False
        if self.key_lengths is None:
            return len(args) == 0
        if len(args) != 1:
            return False
        from libai_b200.layers.attention import KeyPaddingMask

        m = args[0]
        return (isinstance(m, KeyPaddingMask) and m.lengths.shape == self.key_lengths.shape and m.is_prefix())

    def graph_inputs(self, args):
        return (args[0].lengths,) if self.key_lengths is not None else ()


def classify_block_call(model: nn.Module, args, kwargs) -> Optional[BlockCallSpec]:
    """``args`` / ``kwargs``: what the first block received after the hidden state.  ``None`` = not capturable."""
    from libai_b200.layers.attention import KeyPaddingMask

    buffers = {id(b) for b in model.buffers()}
    const = {}
    for k, v in kwargs.items():
        if v is None:
            continue
        if not (torch.is_tensor(v) and id(v) in buffers):
            return None
        const[k] = v
    args = [a for a in args]
    while args and args[-1] is None:
        args.pop()
    if not args:
        return BlockCallSpec(const)
    if len(args) == 1 and isinstance(args[0], KeyPaddingMask) and args[0].is_prefix():
        return BlockCallSpec(const, args[0].lengths)
    return None


class _EagerBlock:
    """Plain callable around a block's original forward: ``make_graphed_callables`` then treats the parameters as
    captured constants (they live at fixed addresses in the optimizer's flat buffer and their gradients are
    accumulated into ``main_grad`` by the captured backward kernels themselves)."""

    def __init__(self, block, spec: Optional[BlockCallSpec] = None):
        self.fn = block.forward
        self.spec = spec or BlockCallSpec()

    def __call__(self, hidden, lengths=None):
        if lengths is None:
            return self.fn(hidden, **self.spec.const_kwargs)
        from libai_b200.layers.attention import KeyPaddingMask

        return self.fn(hidden, KeyPaddingMask.from_lengths(lengths), **self.spec.const_kwargs)


def graph_blocks_multi_slot(blocks: Sequence[nn.Module], sample_hidden: torch.Tensor, n_slots: int, warmup_iters: int = 3,
                            spec: Optional[BlockCallSpec] = None) -> bool:
    spec = spec or BlockCallSpec()
    extra = (spec.key_lengths.detach().clone(),) if spec.key_lengths is not None else ()
    with torch.no_grad():
        n0 = ops.launch_count()
        _EagerBlock(blocks[0], spec)(sample_hidden.detach(), *extra)
        fwd_kernels = ops.launch_count() - n0
    torch.cuda.synchronize()
    fns = tuple(_EagerBlock(b, spec) for _ in range(n_slots) for b in blocks)
    samples = tuple((sample_hidden.detach().clone().requires_grad_(True),) + tuple(e.clone() for e in extra) for _ in fns)
    n0 = ops.launch_count()
    graphed = torch.cuda.make_graphed_callables(fns, samples, num_warmup_iters=warmup_iters, allow_unused_input=True)
    per_block = (ops.launch_count() - n0) // ((warmup_iters + 1) * len(fns))
    ops.count_launch(-(ops.launch_count() - n0))
    bwd_kernels = max(per_block - fwd_kernels, 0)
    # every parameter gradient of the blocks must have gone into main_grad (captured side effect): a parameter that
    # still relies on autograd's AccumulateGrad would silently get no gradient from a function-style graphed callable
    for b in blocks:
        for p in b.parameters():
            if p.requires_grad and (p.grad is not None or not getattr(p, "grad_added_to_main_grad", False)):
                raise RuntimeError("a block parameter gets its gradient through autograd (not main_grad): cannot capture")
    nb = len(blocks)
    for k, block in enumerate(blocks):
        eager = fns[k].fn
        slots = [graphed[s * nb + k] for s in range(n_slots)]

        def forward(hidden, *args, _eager=eager, _slots=slots, _block=block, **kwargs):
            if not (torch.is_grad_enabled() and _block.training and hidden.requires_grad
                    and hidden.shape == sample_hidden.shape and spec.matches(args, kwargs)):
                return _eager(hidden, *args, **kwargs)
            ops.count_launch(fwd_kernels + bwd_kernels)
            return _slots[_CURRENT_SLOT % len(_slots)](hidden, *spec.graph_inputs(args))

        block.forward = forward
    return True


def enable_for_model(model: nn.Module, example_batch: dict) -> bool:
    """Replace the blocks of a ``PipelineStageMixin`` model by graphed versions.  ``example_batch``: one training batch
    (device tensors) used to discover the hidden-state shape.  The gradient buffers must be zeroed afterwards (the
    capture runs backward passes)."""
    from libai_b200.utils import distributed as dutil

    topo = dutil.get_dist_util()
    zero_hooks = getattr(model, "zero_hooks", None)
    if zero_hooks is not None and not getattr(zero_hooks, "graph_capturable", False):
        logger.warning("cuda graphs: ZeRO stage 3 (the blocks' parameter storage comes and goes) — not captured")
        return False
    if zero_hooks is not None:
        # stage 2: the blocks' gradient buckets live in pooled buffers at fixed addresses; bind them for the capture
        # (the hooks that open / reduce them sit outside the blocks, in forward_stage)
        zero_hooks.open_all()
        try:
            return _enable_for_model(model, example_batch, topo)
        finally:
            zero_hooks.close_all()
    return _enable_for_model(model, example_batch, topo)


def _enable_for_model(model: nn.Module, example_batch: dict, topo) -> bool:
    if (getattr(model, "activation_checkpoint", False)
            or (topo.tensor_parallel_size > 1 and not topo.fused_tp_comm)):
        # (checkpointing re-runs the forward inside backward; tensor parallelism is captured only in its fused form —
        # AG→GEMM / GEMM→RS kernels whose handshake state lives in device memory (ops/comm_gemm.py) — the NCCL form
        # keeps eager launches)
        logger.warning("cuda graphs: NCCL-form tensor parallelism / activation checkpointing — not captured")
        return False
    if topo.pipeline_parallel_size > 1:
        return _enable_for_pipeline_stage(model, example_batch, topo)
    layers = model.stage_layers() if hasattr(model, "stage_layers") else None
    if not isinstance(layers, (nn.ModuleList, nn.Sequential)) or len(layers) == 0:
        return False
    shapes = {}

    def grab(mod, args, kwargs):
        shapes["hidden"] = args[0]
        shapes["args"], shapes["kwargs"] = tuple(args[1:]), dict(kwargs)

    h = layers[0].register_forward_pre_hook(grab, with_kwargs=True)
    was_training = model.training
    model.train()
    with torch.no_grad():
        model(**example_batch)
    h.remove()
    spec = classify_block_call(model, shapes.get("args", ()), shapes.get("kwargs", {})) if torch.is_tensor(shapes.get("hidden")) else None
    if spec is None:
        logger.warning("cuda graphs: blocks take arguments that are neither model buffers nor a right-padded key mask — not captured")
        return False
    try:
        if spec.trivial:
            new = graph_transformer_blocks(list(layers), shapes["hidden"])
        else:
            # extra inputs: function-style capture (parameters are constants of the graph, their gradients go to main_grad)
            new = list(layers) if graph_blocks_multi_slot(list(layers), shapes["hidden"], 1, spec=spec) else None
    except Exception as e:   # capture is an optimisation: never take the run down with it
        logger.warning("cuda graphs: capture failed (%s: %s) — staying with eager launches", type(e).__name__, str(e)[:200])
        try:
            torch.cuda.synchronize()
        except Exception:
            pass
        model.train(was_training)
        return False
    if new is None:
        model.train(was_training)
        return False
    assert all(a is b for a, b in zip(new, layers)), "make_graphed_callables is expected to patch the modules in place"
    model.train(was_training)
    logger.info("cuda graphs: captured forward+backward of %d blocks (hidden %s)", len(new), tuple(shapes["hidden"].shape))
    return True


def _enable_for_pipeline_stage(model: nn.Module, example_batch: dict, topo) -> bool:
    """Pipeline stage: capture the blocks this stage owns, ``pp - stage`` copies each (see ``graph_blocks_multi_slot``).
    The hidden-state shape is the stage's p2p payload; it is derived from the batch (token-sharded under sequence
    parallelism) instead of running the model, because only the first stage can run without a received activation."""
    layers = model.stage_layers() if hasattr(model, "stage_layers") else None
    if not isinstance(layers, (nn.ModuleList, nn.Sequential)) or len(layers) == 0:
        return False
    own = [l for l in layers if topo.owns_layer(getattr(l, "layer_idx", 0))]
    if not own:
        return False
    ids = example_batch.get("input_ids")
    if ids is None or ids.dim() != 2:
        logger.warning("cuda graphs: pipeline stage without `input_ids` [b, s] in the batch — not captured")
        return False
    p0 = next(own[0].parameters())
    hidden_size = getattr(own[0], "hidden_size", None)
    if hidden_size is None:
        return False
    b, sq = ids.shape
    if topo.sequence_parallel:
        from libai_b200.layers.embedding import set_sp_shape

        set_sp_shape(b, sq)
        shape = (b * sq // topo.tensor_parallel_size, hidden_size)
    else:
        shape = (b, sq, hidden_size)
    sample = torch.randn(shape, device=p0.device, dtype=p0.dtype) * 0.02
    n_slots = topo.pipeline_parallel_size - topo.pp_rank
    was_training = model.training
    model.train()
    try:
        ok = graph_blocks_multi_slot(own, sample, n_slots)
    except Exception as e:   # capture is an optimisation: never take the run down with it
        logger.warning("cuda graphs: pipeline-stage capture failed (%s: %s) — staying with eager launches", type(e).__name__, str(e)[:200])
        try:
            torch.cuda.synchronize()
        except Exception:
            pass
        ok = False
    model.train(was_training)
    if ok:
        logger.info("cuda graphs: stage %d captured forward+backward of %d blocks x %d micro-batch slots (hidden %s)",
                    topo.pp_rank, len(own), n_slots, tuple(shape))
    # all stages must agree (the fused tensor-parallel kernels inside the graphs are collectives)
    import torch.distributed as dist

    flag = torch.tensor([1 if ok else 0], device=p0.device)
    if dist.is_initialized():
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if int(flag.item()) == 0 and ok:
        logger.warning("cuda graphs: another rank failed to capture — this run cannot mix graphed and eager stages safely")
    return bool(flag.item())
