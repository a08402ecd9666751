"""Tensor-parallel linears whose collective runs INSIDE the GEMM kernel (NVLink peer memory).

    column parallel (sequence-parallel input):   y        = all_gather(x_shard) · Wᵀ      → AG→GEMM
    row parallel    (sequence-parallel output):  y_shard  = reduce_scatter(x · Wᵀ)        → GEMM→RS
    column wgrad:                                dW       = dyᵀ · all_gather(x_shard)     → AG→GEMM (gathered B, TN)

One kernel does both the math and the transfer (``csrc/gemm_sm90.cu`` COMM_AG / COMM_RS): copy CTAs push the local
shard to the peers with TMA bulk copies while wgmma tiles that only need local rows are already running; the RS
epilogue stores partial tiles straight into the owner's staging slot over NVLink and the owners reduce as arrivals are
counted.  The whole handshake state (call counters, arrival targets, "done reading" credits) lives in device memory and
is advanced by the kernels themselves: a call site always launches with the same parameters, so transformer blocks
containing these ops are captured into CUDA graphs (``engine/cuda_graphs.py``) and replayed.

The NCCL versions in ``libai_b200/parallel/mappings.py`` are the oracle and the baseline (reference:
libai/layers/linear.py:123-149 does GEMM→all-reduce / identity→all-reduce on replicated activations).
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch

from libai_b200.ops import count_launch, load_ext
from libai_b200.ops import functional as OF
from libai_b200.ops.functional import _ACT_IDS, reject_quantized_weight
from libai_b200.parallel.symm_mem import CommWorkspace, get_workspace

_BM = 128


def _n_comm_ctas(world: int) -> int:
    """Copy CTAs of the AG kernels: each streams ~200 KB in flight through its TMA ring; more destinations → more CTAs.
    A fixed share of the SMs (a sixth up to 4 ranks, two ninths beyond: 22 / 29 of an H100's 132); not yet tuned on
    H100 (``tests/gpu_comm_bench.py`` sweeps it on two or more GPUs)."""
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return sms // 6 if world <= 4 else (2 * sms) // 9


class _TPState:
    """Shape-keyed symmetric buffers + device-side handshake words of one TP group."""

    def __init__(self, group):
        self.ws: CommWorkspace = get_workspace(group)
        self.world, self.rank = self.ws.world, self.ws.rank
        self.ag: Dict[Tuple[int, int], dict] = {}
        self.rs: Dict[Tuple[int, int], dict] = {}

    def _handshake(self, n_flag_words: int):
        """Per buffer parity: arrival counters and a ``done`` row in the symmetric flag buffer + local state words
        (``[completed calls, CTA exit counter]``)."""
        flags = [self.ws.alloc_flags(n_flag_words), self.ws.alloc_flags(n_flag_words)]
        done = [self.ws.alloc_flags(self.world), self.ws.alloc_flags(self.world)]
        state = [torch.zeros(4, dtype=torch.int32, device=self.ws.device) for _ in range(2)]
        return dict(flag_offs=flags, done_offs=done, state=state, calls=0)

    # gathered operand buffers [2 parities][M, K]; arrival counter per 128-row block
    def ag_state(self, M: int, K: int) -> dict:
        key = (M, K)
        if key not in self.ag:
            s = self._handshake(M // _BM)
            s["buf"] = self.ws.buffer(("ag", M, K), 2 * M * K * 2)
            self.ag[key] = s
        return self.ag[key]

    # staging [2 parities][world][M/world, N]; arrival counter per 128-row block of the owned rows
    def rs_state(self, M: int, N: int) -> dict:
        key = (M, N)
        if key not in self.rs:
            s = self._handshake(M // self.world // _BM)
            s["buf"] = self.ws.buffer(("rs", M, N), 2 * M * N * 2)
            self.rs[key] = s
        return self.rs[key]


_STATES: Dict[int, _TPState] = {}


def _state(group) -> _TPState:
    if id(group) not in _STATES:
        _STATES[id(group)] = _TPState(group)
    return _STATES[id(group)]


def reset_states() -> None:
    """Drop all symmetric buffers (tests / re-initialised process groups)."""
    _STATES.clear()


def fused_supported(M: int, N: int, K: int, world: int) -> bool:
    return M % (_BM * world) == 0 and N % 8 == 0 and K % 8 == 0 and 2 <= world <= 8


# Keep all_gather(x) of the forward for the weight gradient (one device copy of [tokens, h] per column-parallel linear
# and layer) instead of gathering x a second time inside the wgrad kernel: trades b·s·h·2 bytes of activation memory per
# column-parallel linear for the exposed NVLink synchronisation of a gathering wgrad.  ``LIBAI_B200_SP_SAVE_GATHERED=0``
# restores the re-gather
# (Megatron's sequence-parallel memory profile).
import os as _os

_SAVE_GATHERED = _os.environ.get("LIBAI_B200_SP_SAVE_GATHERED", "1") == "1"


def set_save_gathered(enabled: bool) -> None:
    global _SAVE_GATHERED
    _SAVE_GATHERED = bool(enabled)


def _snapshot_gathered(gathered: torch.Tensor, x_shard: torch.Tensor, rank: int) -> torch.Tensor:
    """Private copy of the gathered operand (the symmetric buffer is reused by the next AG call); the local rows were
    never written into the buffer (the kernel reads them from ``x_shard``)."""
    rows = x_shard.shape[0]
    full = gathered.clone()
    full[rank * rows : (rank + 1) * rows].copy_(x_shard)
    count_launch(2)
    return full


def _next(s: dict) -> int:
    """Buffer parity of this call.  Static per call site once captured in a CUDA graph; correctness does not depend on
    strict alternation (the kernels hand out write credits), it only avoids waiting for them."""
    par = s["calls"] & 1
    s["calls"] += 1
    return par


# --------------------------------------------------------------------------------------------------
# raw fused ops
# --------------------------------------------------------------------------------------------------
def ag_gemm(x_shard: torch.Tensor, w: torch.Tensor, bias, act, group, layout: int = 0, need_pre: bool = False,
            pre_in=None, colsum=None, fill_local: bool = False):
    """``epilogue(all_gather(x_shard) @ op(w))`` → ``(y [M, N], pre, x_full)``.

    ``layout`` 0: w is ``[N, K]``; 1: w is ``[K, N]``.  Epilogue: ``+ bias`` then ``act`` (``pre`` = the pre-activation
    when ``need_pre``), or with ``pre_in``: ``· act'(pre_in)`` (dgrad fused with the activation backward) and optional
    fp32 column sums into ``colsum``.  ``x_full`` (the local gathered buffer) is complete only with ``fill_local``."""
    reject_quantized_weight("comm_gemm.ag_gemm", w)
    ext = load_ext()
    st = _state(group)
    rows, K = x_shard.shape
    M = rows * st.world
    s = st.ag_state(M, K)
    par = _next(s)
    gathered = s["buf"].view(torch.bfloat16, (2, M, K))[par]
    if fill_local:
        # the local rows of the gathered buffer are only needed by LATER kernels of this stream (the wgrad that reuses
        # all_gather(dy)): a plain device copy at HBM speed instead of a second job for the copy
        # CTAs, whose throughput is what the kernel waits for
        gathered[st.rank * rows : (st.rank + 1) * rows].copy_(x_shard)
        count_launch()
    y, pre = ext.ag_gemm(
        gathered, x_shard, w, layout, bias, _ACT_IDS[act], need_pre, pre_in, colsum, False, st.world, st.rank,
        s["buf"].peer_ptrs(par * M * K * 2), st.ws.flags.peer_ptrs(s["flag_offs"][par]),
        st.ws.flags.peer_ptrs(s["done_offs"][par]), s["state"][par], _n_comm_ctas(st.world),
    )
    count_launch()
    return y, (pre if need_pre else None), gathered


def ag_wgrad(gy: torch.Tensor, x_shard: torch.Tensor, out: torch.Tensor, accumulate: bool, group) -> None:
    """``out [N_local, K] (+)= gyᵀ @ all_gather(x_shard)`` (fp32) with the all-gather inside the wgrad kernel."""
    ext = load_ext()
    st = _state(group)
    rows, K = x_shard.shape
    M = rows * st.world
    s = st.ag_state(M, K)
    par = _next(s)
    gathered = s["buf"].view(torch.bfloat16, (2, M, K))[par]
    ext.ag_wgrad(
        gy, gathered, x_shard, out, accumulate, st.world, st.rank, s["buf"].peer_ptrs(par * M * K * 2),
        st.ws.flags.peer_ptrs(s["flag_offs"][par]), st.ws.flags.peer_ptrs(s["done_offs"][par]), s["state"][par],
        _n_comm_ctas(st.world),
    )
    count_launch()


def gemm_rs(x: torch.Tensor, w: torch.Tensor, bias, residual, group, layout: int = 0):
    """``reduce_scatter(x @ op(w)) (+ bias) (+ residual)`` → ``[M / world, N]``."""
    reject_quantized_weight("comm_gemm.gemm_rs", w)
    ext = load_ext()
    st = _state(group)
    M = x.shape[0]
    N = w.shape[0] if layout == 0 else w.shape[1]
    s = st.rs_state(M, N)
    par = _next(s)
    y = ext.gemm_rs(
        x, w, layout, bias, residual, st.world, st.rank, s["buf"].peer_ptrs(0),
        st.ws.flags.peer_ptrs(s["flag_offs"][par]), st.ws.flags.peer_ptrs(s["done_offs"][par]), s["state"][par],
        par * M * N,
    )
    count_launch()
    return y


def _wgrad_ag(gy, x_shard, w, group):
    """dW of a column-parallel weight with the all-gather of ``x_shard`` inside the wgrad kernel; the destination
    follows :func:`functional._weight_grad`'s rule."""
    main_grad = OF._main_grad(w)
    if main_grad is not None:
        ag_wgrad(gy, x_shard, main_grad, True, group)
        w.grad_added_to_main_grad = True
        return None
    out = torch.empty(w.shape, dtype=torch.float32, device=w.device)
    ag_wgrad(gy, x_shard, out, False, group)
    return out.to(w.dtype)


# --------------------------------------------------------------------------------------------------
# autograd wrappers
# --------------------------------------------------------------------------------------------------
class ColumnParallelLinearFused(torch.autograd.Function):
    """fwd AG→GEMM (+bias, +act in the epilogue); bwd dx_shard = GEMM→RS(dy, W), dW = dyᵀ · all_gather(x_shard) as
    one gathered-B wgrad kernel (no separate all-gather)."""

    @staticmethod
    def forward(ctx, x_shard, w, bias, act, group):
        has_act = act not in (None, "none")
        # every gradient, the bias' alone included, goes through the activation backward, which reads the pre-activation
        need_pre = has_act and any(ctx.needs_input_grad[:3])
        y, pre, gathered = ag_gemm(x_shard, w, bias, act if has_act else None, group, need_pre=need_pre)
        x_full = None
        if _SAVE_GATHERED and ctx.needs_input_grad[1]:
            x_full = _snapshot_gathered(gathered, x_shard, _state(group).rank)
        ctx.save_for_backward(x_shard, w, pre, x_full)
        ctx.act, ctx.group, ctx.bias_param = (act if has_act else None), group, bias
        return y

    @staticmethod
    def backward(ctx, gy):
        ext = load_ext()
        x_shard, w, pre, x_full = ctx.saved_tensors
        gy = gy.contiguous()
        if ctx.act is not None:
            gy = ext.act_bwd(gy, pre, _ACT_IDS[ctx.act])
            count_launch()
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            gx = gemm_rs(gy, w, None, None, ctx.group, layout=1)  # dy [M, N_loc] · W [N_loc, K]
        if ctx.needs_input_grad[1]:
            gw = OF._weight_grad(ext, gy, x_full, w) if x_full is not None else _wgrad_ag(gy, x_shard, w, ctx.group)
        if ctx.needs_input_grad[2]:
            gb = OF._bias_grad(ext, gy, ctx.bias_param)
        return gx, gw, gb, None, None


class RowParallelLinearFused(torch.autograd.Function):
    """fwd y_shard = GEMM→RS(x, W) (+bias +residual in the reduce phase);
    bwd dx = AG→GEMM(dy_shard, W) and dW = all_gather(dy_shard)ᵀ · x (the gathered dy comes for free)."""

    @staticmethod
    def forward(ctx, x, w, bias, residual, group):
        y = gemm_rs(x, w, bias, residual, group)
        ctx.save_for_backward(x, w)
        ctx.group, ctx.bias_param, ctx.has_res = group, bias, residual is not None
        return y

    @staticmethod
    def backward(ctx, gy_shard):
        ext = load_ext()
        x, w = ctx.saved_tensors
        gy_shard = gy_shard.contiguous()
        gw = gb = None
        need_w = ctx.needs_input_grad[1]
        gx, _, gy_full = ag_gemm(gy_shard, w, None, None, ctx.group, layout=1, fill_local=need_w)  # dy_full [M, N] · W [N, K_loc]
        if need_w:
            gw = OF._weight_grad(ext, gy_full, x, w)
        if ctx.needs_input_grad[2]:
            gb = OF._bias_grad(ext, gy_shard, ctx.bias_param)  # partial over token shards: summed over TP by sync_gradients
        return (gx if ctx.needs_input_grad[0] else None), gw, gb, (gy_shard if ctx.has_res else None), None


class TPMLPFused(torch.autograd.Function):
    """``x_shard → AG→GEMM(+b1, act) → GEMM→RS(+b2, +residual)`` as one autograd node (4 collectives fused into 4 GEMM
    kernels forward+backward, plus the gathered-B wgrad): the backward's first kernel is the AG→GEMM dgrad of the second
    linear with the activation backward *and* the first bias' gradient in its epilogue."""

    @staticmethod
    def forward(ctx, x_shard, w1, b1, w2, b2, residual, act, group):
        h, pre, gathered = ag_gemm(x_shard, w1, b1, act, group, need_pre=True)
        x_full = None
        if _SAVE_GATHERED and ctx.needs_input_grad[1]:
            x_full = _snapshot_gathered(gathered, x_shard, _state(group).rank)
        y = gemm_rs(h, w2, b2, residual, group)
        ctx.save_for_backward(x_shard, w1, w2, pre, h, x_full)
        ctx.act, ctx.group, ctx.b1, ctx.b2, ctx.has_res = act, group, b1, b2, residual is not None
        return y

    @staticmethod
    def backward(ctx, gy_shard):
        ext = load_ext()
        x_shard, w1, w2, pre, h, x_full = ctx.saved_tensors
        gy_shard = gy_shard.contiguous()
        b1, b2 = ctx.b1, ctx.b2
        fused_gb1 = OF._fused_bias_grad_target(b1) if ctx.needs_input_grad[2] else None
        need_w2 = ctx.needs_input_grad[3]
        # dpre = (all_gather(dy_shard) · W2) ⊙ act'(pre)   [+ column sums → b1.main_grad]
        dpre, _, gy_full = ag_gemm(gy_shard, w2, None, ctx.act, ctx.group, layout=1, pre_in=pre, colsum=fused_gb1,
                                   fill_local=need_w2)
        gw2 = OF._weight_grad(ext, gy_full, h, w2) if need_w2 else None
        gb2 = OF._bias_grad(ext, gy_shard, b2) if ctx.needs_input_grad[4] else None
        gx = gemm_rs(dpre, w1, None, None, ctx.group, layout=1) if ctx.needs_input_grad[0] else None
        gw1 = None
        if ctx.needs_input_grad[1]:
            gw1 = OF._weight_grad(ext, dpre, x_full, w1) if x_full is not None else _wgrad_ag(dpre, x_shard, w1, ctx.group)
        gb1 = None
        if fused_gb1 is not None:
            b1.grad_added_to_main_grad = True
        elif ctx.needs_input_grad[2]:
            gb1 = OF._bias_grad(ext, dpre, b1)
        return gx, gw1, gb1, gw2, gb2, (gy_shard if ctx.has_res else None), None, None


def column_parallel_linear(x_shard, w, bias, act, group):
    reject_quantized_weight("comm_gemm.column_parallel_linear", w)
    return ColumnParallelLinearFused.apply(x_shard, w, bias, act, group)


def row_parallel_linear(x, w, bias, residual, group):
    reject_quantized_weight("comm_gemm.row_parallel_linear", w)
    return RowParallelLinearFused.apply(x, w, bias, residual, group)


def tp_mlp(x_shard, w1, b1, w2, b2, residual, act, group):
    reject_quantized_weight("comm_gemm.tp_mlp", w1, w2)
    return TPMLPFused.apply(x_shard, w1, b1, w2, b2, residual, act, group)
