"""Autograd-aware tensor-parallel communication primitives.

The reference expresses these as SBP changes (``to_global(sbp=..., grad_sbp=...)``, e.g.
libai/layers/linear.py:123-149); here they are explicit collectives on the TP process group:

================  =======================  =======================
function          forward                  backward
================  =======================  =======================
copy_to_tp        identity                 all-reduce
reduce_from_tp    all-reduce               identity
gather_from_sp    all-gather (tokens)      reduce-scatter (tokens)
reduce_scatter_to_sp  reduce-scatter       all-gather
scatter_to_sp     take local token slice   all-gather
gather_from_tp    all-gather (last dim)    take local slice
================  =======================  =======================

"sp" = Megatron-style sequence parallelism: activations outside the TP region are sharded over
the *flattened token* dimension (dim 0).  On H100 the GEMM-adjacent pairs (all-gather→GEMM,
GEMM→reduce-scatter) are replaced by fused kernels (see ``libai_b200/ops/comm_gemm.py``); these
NCCL versions are the oracle and the baseline.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from libai_b200.utils import distributed as dutil


def _tp():
    topo = dutil.get_dist_util()
    return topo.tp_group, topo.tensor_parallel_size, topo.tp_rank


def _all_reduce(x):
    group, size, _ = _tp()
    if size == 1:
        return x
    x = x.contiguous()
    dist.all_reduce(x, group=group)
    return x


def _all_gather_dim0(x):
    group, size, _ = _tp()
    if size == 1:
        return x
    x = x.contiguous()
    out = torch.empty((x.shape[0] * size,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    dist.all_gather_into_tensor(out, x, group=group)
    return out


def _reduce_scatter_dim0(x):
    group, size, _ = _tp()
    if size == 1:
        return x
    x = x.contiguous()
    assert x.shape[0] % size == 0, f"token dim {x.shape[0]} not divisible by tp={size}"
    out = torch.empty((x.shape[0] // size,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    if x.device.type == "cpu":  # gloo has no reduce_scatter_tensor
        tmp = x.clone()
        dist.all_reduce(tmp, group=group)
        _, _, r = _tp()
        out.copy_(tmp.narrow(0, r * out.shape[0], out.shape[0]))
    else:
        dist.reduce_scatter_tensor(out, x, group=group)
    return out


def _split_dim0(x):
    _, size, r = _tp()
    if size == 1:
        return x
    n = x.shape[0] // size
    return x.narrow(0, r * n, n).contiguous()


def _all_gather_last(x):
    group, size, _ = _tp()
    if size == 1:
        return x
    parts = [torch.empty_like(x) for _ in range(size)]
    dist.all_gather(parts, x.contiguous(), group=group)
    return torch.cat(parts, dim=-1)


def _split_last(x):
    _, size, r = _tp()
    if size == 1:
        return x
    n = x.shape[-1] // size
    return x.narrow(-1, r * n, n).contiguous()


class _CopyToTP(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return x

    @staticmethod
    def backward(ctx, g):
        return _all_reduce(g)


class _ReduceFromTP(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return _all_reduce(x)

    @staticmethod
    def backward(ctx, g):
        return g


class _GatherFromSP(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, reduce_scatter_grad):
        ctx.rs = reduce_scatter_grad
        return _all_gather_dim0(x)

    @staticmethod
    def backward(ctx, g):
        return (_reduce_scatter_dim0(g) if ctx.rs else _split_dim0(g)), None


class _ReduceScatterToSP(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return _reduce_scatter_dim0(x)

    @staticmethod
    def backward(ctx, g):
        return _all_gather_dim0(g)


class _ScatterToSP(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return _split_dim0(x)

    @staticmethod
    def backward(ctx, g):
        return _all_gather_dim0(g)


class _GatherFromTP(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return _all_gather_last(x)

    @staticmethod
    def backward(ctx, g):
        return _split_last(g)


def copy_to_tp(x):
    return _CopyToTP.apply(x) if dutil.get_tensor_parallel_size() > 1 else x


def reduce_from_tp(x):
    return _ReduceFromTP.apply(x) if dutil.get_tensor_parallel_size() > 1 else x


def gather_from_sp(x, reduce_scatter_grad: bool = True):
    return _GatherFromSP.apply(x, reduce_scatter_grad) if dutil.get_tensor_parallel_size() > 1 else x


def reduce_scatter_to_sp(x):
    return _ReduceScatterToSP.apply(x) if dutil.get_tensor_parallel_size() > 1 else x


def scatter_to_sp(x):
    return _ScatterToSP.apply(x) if dutil.get_tensor_parallel_size() > 1 else x


def gather_from_tp(x):
    return _GatherFromTP.apply(x) if dutil.get_tensor_parallel_size() > 1 else x
