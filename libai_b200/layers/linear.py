"""Data / column / row parallel linear layers.

Spec: reference libai/layers/linear.py:25-180 — weight is ``[out, in]``; ``parallel="col"``
splits the output features (weight dim 0, bias dim 0), ``parallel="row"`` splits the input
features (weight dim 1, bias replicated), ``skip_bias_add`` returns ``(y, bias)`` so the caller
can fuse the bias into the next op, ``layer_idx`` selects the pipeline stage.

Communication (explicit, instead of SBP boxing):

* col: fwd identity on x / bwd all-reduce(dx) over TP; with sequence parallelism
  fwd all-gather(x) / bwd reduce-scatter(dx).
* row: fwd all-reduce(y) over TP; with sequence parallelism fwd reduce-scatter(y) /
  bwd all-gather(dy).

On H100 the sequence-parallel pairs run as single fused kernels (AG→GEMM, GEMM→RS over NVLink
peer memory, ``libai_b200/ops/comm_gemm.py``) when ``train.dist.fused_tp_comm`` is on.
"""
from __future__ import annotations

import torch
from torch import nn

from libai_b200.ops import functional as OF
from libai_b200.parallel import mappings
from libai_b200.utils import distributed as dutil

from ._param import create_parameter, xavier_normal_, zeros_


class Linear1D(nn.Module):
    def __init__(
        self,
        in_features,
        out_features,
        bias=True,
        parallel="data",
        init_method=xavier_normal_,
        skip_bias_add=False,
        dtype=None,
        *,
        layer_idx=0,
    ):
        super().__init__()
        if parallel not in ("data", "col", "row"):
            raise KeyError(f"{parallel} is not supported! Only support ('data', 'row' and 'col')")
        self.in_features = in_features
        self.out_features = out_features
        self.parallel = parallel
        self.skip_bias_add = skip_bias_add
        self.layer_idx = layer_idx
        w_dim = {"data": None, "col": 0, "row": 1}[parallel]
        b_dim = 0 if parallel == "col" else None
        self.weight = create_parameter(
            (out_features, in_features), init_method, tp_dim=w_dim, layer_idx=layer_idx, dtype=dtype
        )
        self.bias = (
            create_parameter((out_features,), zeros_, tp_dim=b_dim, layer_idx=layer_idx, dtype=dtype)
            if bias
            else None
        )
        if parallel == "row" and self.bias is not None:
            # added after the reduce-scatter, i.e. on token shards: its gradient is partial per TP rank
            self.bias.sequence_parallel = dutil.get_dist_util().sequence_parallel

    def fused_bias_residual(self, x, residual):
        """Row-parallel fast path of the block-output projections under fused tensor parallelism:
        ``reduce_scatter(x @ Wᵀ) + bias + residual`` in ONE kernel (bias and residual are added by the reduce phase of
        the GEMM→RS kernel).  Returns ``None`` when the fused kernel does not apply (caller falls back)."""
        topo = dutil.get_dist_util()
        if not (topo.fused_tp_comm and self.parallel == "row" and x.is_cuda and x.dtype == self.weight.dtype):
            return None
        return self._forward_fused(x, self.bias, None, topo, residual=residual)

    def forward(self, x, act=None):
        """``act`` (optional activation name) is fused into the GEMM epilogue when the bias is
        applied here (i.e. not with ``skip_bias_add``)."""
        topo = dutil.get_dist_util()
        sp = topo.sequence_parallel
        bias_now = None if self.skip_bias_add else self.bias
        if topo.fused_tp_comm and self.parallel in ("col", "row") and x.is_cuda and x.dtype == self.weight.dtype:
            y = self._forward_fused(x, bias_now, act, topo)
            if y is not None:
                return (y, self.bias) if self.skip_bias_add else y
        if self.parallel == "col":
            x = mappings.gather_from_sp(x) if sp else mappings.copy_to_tp(x)
            y = OF.linear(x, self.weight, bias_now, act)
        elif self.parallel == "row":
            y = OF.linear(x, self.weight, None, None)
            y = mappings.reduce_scatter_to_sp(y) if sp else mappings.reduce_from_tp(y)
            if bias_now is not None:
                y = y + bias_now.to(y.dtype)
            if act is not None:
                y = OF._act_ref(y, act)
        else:
            y = OF.linear(x, self.weight, bias_now, act)
        if self.skip_bias_add:
            return y, self.bias
        return y

    def _forward_fused(self, x, bias_now, act, topo, residual=None):
        """AG->GEMM / GEMM->RS with the collective inside the wgmma kernel (None = shape unsupported)."""
        from libai_b200.ops import comm_gemm, use_native

        if not use_native(x) or x.dtype != torch.bfloat16:
            return None
        x2 = x.reshape(-1, x.shape[-1])
        t = topo.tensor_parallel_size
        if self.parallel == "col":
            M, N, K = x2.shape[0] * t, self.weight.shape[0], x2.shape[1]
            if not comm_gemm.fused_supported(M, N, K, t):
                return None
            return comm_gemm.column_parallel_linear(x2.contiguous(), self.weight, bias_now, act, topo.tp_group)
        M, N, K = x2.shape[0], self.weight.shape[0], x2.shape[1]
        if not comm_gemm.fused_supported(M, N, K, t) or act is not None:
            return None
        if residual is not None:
            residual = residual.reshape(-1, N).contiguous()
        return comm_gemm.row_parallel_linear(x2.contiguous(), self.weight, bias_now, residual, topo.tp_group)

    def extra_repr(self) -> str:
        return "in_features={}, out_features={}, bias={}, parallel={}".format(
            self.in_features, self.out_features, self.bias is not None, self.parallel
        )


# reference alias (libai/layers/linear.py:180)
Linear = Linear1D
