"""Gated MLP (SwiGLU) with the gate and up projections as ONE GEMM.

Reference: projects/Llama/llama.py:81-113 — ``down(silu(gate(x)) * up(x))`` with two separate column-parallel linears and an
unfused elementwise product ("fuse gate/up as one 2f/t GEMM").  The two weights stay separate
``Parameter``s (checkpoints, HF loaders and the reference's module names are unchanged); once the optimizer has moved the
parameters into its flat buffer they are adjacent in memory, so a ``[2F, K]`` view over both — and over their fp32
``main_grad`` slices — costs nothing:

* forward: one GEMM ``x · [Wg; Wu]ᵀ → [T, 2F] = [gate | up]`` (tensor parallel: ONE all-gather→GEMM instead of two
  all-gathers of the same activations), a packed SwiGLU kernel, the down projection;
* backward: one dgrad GEMM over ``K = 2F`` (TP: one GEMM→reduce-scatter instead of two plus an add), one wgrad into the
  fused ``main_grad`` view (TP: one gathered-B wgrad kernel).
"""
from __future__ import annotations

import os
from typing import Optional, Tuple

import torch

from libai_b200.ops import count_launch, load_ext
from libai_b200.ops import functional as OF
from libai_b200.ops.functional import reject_quantized_weight

_ENABLED = os.environ.get("LIBAI_B200_FUSED_GATE_UP", "1") == "1"


def enabled() -> bool:
    return _ENABLED


def set_enabled(flag: bool) -> None:
    global _ENABLED
    _ENABLED = bool(flag)


def _adjacent(a: torch.Tensor, b: torch.Tensor) -> bool:
    return (a.shape == b.shape and a.dtype == b.dtype and a.is_contiguous() and b.is_contiguous()
            and a.untyped_storage().data_ptr() == b.untyped_storage().data_ptr()
            and b.data_ptr() == a.data_ptr() + a.numel() * a.element_size())


def fused_gate_up_views(wg: torch.Tensor, wu: torch.Tensor) -> Optional[Tuple[torch.Tensor, Optional[torch.Tensor]]]:
    """``([2F, K] weight view, [2F, K] fp32 main_grad view or None)`` when the two weights are adjacent in one buffer."""
    if wg.dim() != 2 or not _adjacent(wg, wu):
        return None
    f, k = wg.shape
    w = torch.as_strided(wg.detach(), (2 * f, k), (k, 1))
    g1, g2 = OF._main_grad(wg), OF._main_grad(wu)
    mg = None
    if g1 is not None and g2 is not None and _adjacent(g1, g2):
        mg = torch.as_strided(g1, (2 * f, k), (k, 1))
    return w, mg


def _gate_up_grads(wg, wu, out):
    """Autograd's gradients of the gate and up weights after the ``[2F, K]`` wgrad: ``None`` for both when it
    accumulated into the fused ``main_grad`` view (``out`` is None), else the halves of its fresh fp32 result."""
    if out is None:
        wg.grad_added_to_main_grad = True
        wu.grad_added_to_main_grad = True
        return None, None
    f = wg.shape[0]
    return out[:f].to(wg.dtype), out[f:].to(wu.dtype)


class GatedMLPFn(torch.autograd.Function):
    """Single-GPU / data-parallel form: ``y = (silu(x Wgᵀ) * (x Wuᵀ)) Wdᵀ`` with ``[Wg; Wu]`` as one GEMM operand."""

    @staticmethod
    def forward(ctx, x, wg, wu, wd):
        ext = load_ext()
        w, _ = fused_gate_up_views(wg, wu)
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        gu = ext.gemm(x2, w, 0, None, None, False, torch.bfloat16)
        h = ext.swiglu_packed_fwd(gu)
        y = ext.gemm(h, wd, 0, None, None, False, torch.bfloat16)
        count_launch(3)
        ctx.save_for_backward(x2, gu, h)
        ctx.params = (wg, wu, wd)
        return y.view(*x.shape[:-1], wd.shape[0])

    @staticmethod
    def backward(ctx, gy):
        ext = load_ext()
        x2, gu, h = ctx.saved_tensors
        wg, wu, wd = ctx.params
        w, mg = fused_gate_up_views(wg, wu)
        g2 = gy.reshape(-1, gy.shape[-1]).contiguous()
        dh = ext.gemm(g2, wd, 1, None, None, False, torch.bfloat16)
        gwd = OF._weight_grad(ext, g2, h, wd) if ctx.needs_input_grad[3] else None
        dgu = ext.swiglu_packed_bwd(dh, gu)
        gx = ext.gemm(dgu, w, 1, None, None, False, torch.bfloat16).view(*gy.shape[:-1], x2.shape[1]) if ctx.needs_input_grad[0] else None
        gwg = gwu = None
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            out = None
            if mg is not None:
                ext.gemm(dgu, x2, 2, None, mg, True, torch.float32)
            else:
                out = ext.gemm(dgu, x2, 2, None, None, False, torch.float32)
            count_launch()
            gwg, gwu = _gate_up_grads(wg, wu, out)
        count_launch(3)
        return gx, gwg, gwu, gwd


class TPGatedMLPFused(torch.autograd.Function):
    """Tensor-parallel form on token-sharded activations: all-gather→GEMM against ``[Wg; Wu]`` (this rank's rows of
    both), packed SwiGLU, GEMM→reduce-scatter through ``Wd`` (+ residual in its reduce phase)."""

    @staticmethod
    def forward(ctx, x_shard, wg, wu, wd, residual, group):
        from libai_b200.ops import comm_gemm

        ext = load_ext()
        w, _ = fused_gate_up_views(wg, wu)
        gu, _, _ = comm_gemm.ag_gemm(x_shard, w, None, None, group)
        h = ext.swiglu_packed_fwd(gu)
        count_launch()
        y = comm_gemm.gemm_rs(h, wd, None, residual, group)
        ctx.save_for_backward(x_shard, gu, h)
        ctx.params, ctx.group, ctx.has_res = (wg, wu, wd), group, residual is not None
        return y

    @staticmethod
    def backward(ctx, gy_shard):
        from libai_b200.ops import comm_gemm

        ext = load_ext()
        x_shard, gu, h = ctx.saved_tensors
        wg, wu, wd = ctx.params
        w, mg = fused_gate_up_views(wg, wu)
        gy_shard = gy_shard.contiguous()
        need_wd = ctx.needs_input_grad[3]
        dh, _, gy_full = comm_gemm.ag_gemm(gy_shard, wd, None, None, ctx.group, layout=1, fill_local=need_wd)
        gwd = OF._weight_grad(ext, gy_full, h, wd) if need_wd else None
        dgu = ext.swiglu_packed_bwd(dh, gu)
        count_launch()
        gx = comm_gemm.gemm_rs(dgu, w, None, None, ctx.group, layout=1) if ctx.needs_input_grad[0] else None
        gwg = gwu = None
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            out = None
            if mg is not None:
                comm_gemm.ag_wgrad(dgu, x_shard, mg, True, ctx.group)
            else:
                out = torch.empty(w.shape, dtype=torch.float32, device=w.device)
                comm_gemm.ag_wgrad(dgu, x_shard, out, False, ctx.group)
            gwg, gwu = _gate_up_grads(wg, wu, out)
        return gx, gwg, gwu, gwd, (gy_shard if ctx.has_res else None), None


def gated_mlp(x, wg, wu, wd):
    reject_quantized_weight("gated_mlp", wg, wu, wd)
    return GatedMLPFn.apply(x, wg, wu, wd)


def tp_gated_mlp(x_shard, wg, wu, wd, residual, group):
    reject_quantized_weight("tp_gated_mlp", wg, wu, wd)
    return TPGatedMLPFused.apply(x_shard, wg, wu, wd, residual, group)
