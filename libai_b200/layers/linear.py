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

For inference, ``quantize_fp8_`` turns the layer's weight into FP8 (E4M3) bytes with one fp32 scale per output
channel of this rank's shard, and ``quantize_int4_`` into packed 4-bit values with a scale and zero point per row and
group of 128 input columns; the forward then runs ``OF.linear_fp8w`` or ``OF.linear_int4w`` inside the same TP mappings.
"""
from __future__ import annotations

import torch
from torch import nn

from libai_b200.ops import functional as OF
from libai_b200.parallel import mappings
from libai_b200.utils import distributed as dutil

from ._param import create_parameter, xavier_normal_, zeros_


_FP8_SOURCE_DTYPES = (torch.bfloat16, torch.float16, torch.float32)


class Linear1D(nn.Module):
    compute_dtype = None   # FP8 or INT4 weights: the dtype of the inputs, outputs and bias (the weight's dtype before)

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

    @property
    def fp8(self) -> bool:
        """The weight is FP8 (E4M3) bytes with row scales ``weight_scale`` (:meth:`quantize_fp8_`)."""
        return self.weight.dtype == torch.float8_e4m3fn

    @property
    def int4(self) -> bool:
        """The weight is packed INT4 values with group scales ``weight_scale`` and zeros ``weight_zero``
        (:meth:`quantize_int4_`)."""
        return self.weight.dtype == torch.uint8

    @property
    def quantized(self) -> bool:
        """The weight is FP8 or INT4: only ``OF.linear_fp8w`` / ``OF.linear_int4w`` read it, never a bf16 GEMM."""
        return self.fp8 or self.int4

    @torch.no_grad()
    def quantize_fp8_(self):
        """Replace the weight ``[out_local, in_local]`` by its FP8 (E4M3) bytes and the fp32 scales ``weight_scale``
        ``[out_local]``, one per output channel: ``s = amax|w_n| / 448`` (1 for an all-zero row), bytes
        ``e4m3_rn_satfinite(w / s)`` (``OF.kv_cache_quantize_ref``); the weight reads back as ``float(e)·s``.  The bias
        and the activations keep the weight's former dtype (``compute_dtype``).  For inference only; a second call is a
        no-op."""
        if self.fp8:
            return self
        w = self.weight
        if self.int4 or w.dtype not in _FP8_SOURCE_DTYPES:
            raise TypeError(f"quantize_fp8_: a {w.dtype} weight (bf16, fp16 or fp32 expected)")
        e, s = OF.kv_cache_quantize_ref(w)
        self.compute_dtype = w.dtype
        self.weight = nn.Parameter(e, requires_grad=False)
        self.weight_scale = nn.Parameter(s, requires_grad=False)
        return self

    @torch.no_grad()
    def quantize_int4_(self):
        """Replace the weight ``[out_local, in_local]`` (``in_local % 128 == 0``, finite) by its 4-bit values packed two
        per byte (uint8 ``[out_local, in_local / 2]``), with a bf16 scale ``weight_scale`` and a uint8 zero point
        ``weight_zero`` ``[out_local, in_local / 128]`` per row and group of 128 columns (``OF.int4_quantize_ref``); the
        weight reads back as ``bf16_rn((q − z) · s)``.  The bias and the activations keep the weight's former dtype
        (``compute_dtype``).  For inference only; a second call is a no-op."""
        if self.int4:
            return self
        w = self.weight
        if self.fp8 or w.dtype not in _FP8_SOURCE_DTYPES:
            raise TypeError(f"quantize_int4_: a {w.dtype} weight (bf16, fp16 or fp32 expected)")
        q, s, z = OF.int4_quantize_ref(w)
        self.compute_dtype = w.dtype
        self.weight = nn.Parameter(q, requires_grad=False)
        self.weight_scale = nn.Parameter(s, requires_grad=False)
        self.weight_zero = nn.Parameter(z, requires_grad=False)
        return self

    def _apply(self, fn, recurse=True):
        """Dtype casts (``.to(dtype)``, ``.bfloat16()``, ``.half()``, ``.float()``) leave FP8 or INT4 bytes and their
        scales (and zeros) as they are and change ``compute_dtype`` (and the bias) instead; device moves move them."""
        if not self.quantized:
            return super()._apply(fn, recurse)
        probe = fn(torch.empty(0, dtype=self.compute_dtype, device=self.weight.device))
        order = list(self._parameters)
        held = {k: self._parameters.pop(k) for k in ("weight", "weight_scale", "weight_zero") if k in self._parameters}
        try:
            super()._apply(fn, recurse)
        finally:
            rest = dict(self._parameters)
            self._parameters.clear()
            self._parameters.update({k: held[k] if k in held else rest[k] for k in order})
        for k, p in held.items():
            if p.device != probe.device:
                self._parameters[k] = nn.Parameter(p.detach().to(probe.device), requires_grad=False)
        if probe.is_floating_point():
            self.compute_dtype = probe.dtype
        return self

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
            y = self._gemm(x, bias_now, act)
        elif self.parallel == "row":
            y = self._gemm(x, None, None)
            y = mappings.reduce_scatter_to_sp(y) if sp else mappings.reduce_from_tp(y)
            if bias_now is not None:
                y = y + bias_now.to(y.dtype)
            if act is not None:
                y = OF._act_ref(y, act)
        else:
            y = self._gemm(x, bias_now, act)
        if self.skip_bias_add:
            return y, self.bias
        return y

    def _gemm(self, x, bias, act):
        if self.fp8:
            return OF.linear_fp8w(x, self.weight, self.weight_scale, bias, act)
        if self.int4:
            return OF.linear_int4w(x, self.weight, self.weight_scale, self.weight_zero, bias, act)
        return OF.linear(x, self.weight, bias, act)

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
        return "in_features={}, out_features={}, bias={}, parallel={}{}".format(
            self.in_features, self.out_features, self.bias is not None, self.parallel,
            f", weight={'fp8' if self.fp8 else 'int4 (group 128)'} (compute_dtype={self.compute_dtype})"
            if self.quantized else "",
        )


# reference alias (libai/layers/linear.py:180)
Linear = Linear1D
