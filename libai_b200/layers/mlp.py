"""Transformer feed-forward block.

Spec: reference libai/layers/mlp.py:22-114 — ``h→f`` column-parallel linear, bias+GELU, ``f→h``
row-parallel linear, bias+dropout.  The bias+GELU runs in the epilogue of the first GEMM
(``Linear1D.forward(act=...)``) and bias+dropout+residual is one fused op; ``bias_gelu_fusion``
/ ``bias_dropout_fusion`` are accepted for config compatibility (both paths compute the same
function).
"""
import torch
from torch import nn

from libai_b200.ops import functional as OF
from libai_b200.parallel import mappings
from libai_b200.utils import distributed as dutil

from ._param import xavier_normal_
from .linear import Linear


class MLP(nn.Module):
    def __init__(
        self,
        hidden_size,
        ffn_hidden_size,
        output_dropout_prob=0.0,
        init_method=xavier_normal_,
        output_layer_init_method=None,
        bias_gelu_fusion=False,
        bias_dropout_fusion=False,
        *,
        layer_idx=0,
    ):
        super().__init__()
        self.output_dropout_prob = output_dropout_prob
        self.bias_gelu_fusion = bias_gelu_fusion
        self.bias_dropout_fusion = bias_dropout_fusion
        if output_layer_init_method is None:
            output_layer_init_method = init_method
        self.dense_h_to_4h = Linear(
            hidden_size, ffn_hidden_size, bias=True, parallel="col", skip_bias_add=False,
            init_method=init_method, layer_idx=layer_idx,
        )
        self.dense_4h_to_h = Linear(
            ffn_hidden_size, hidden_size, bias=True, parallel="row", skip_bias_add=True,
            init_method=output_layer_init_method, layer_idx=layer_idx,
        )

    def forward(self, hidden_states, residual=None):
        """Returns ``residual + dropout(mlp(x))`` when ``residual`` is given (fused epilogue)."""
        topo = dutil.get_dist_util()
        # FP8 and INT4 weights take the per-Linear path: OF.mlp and the fused TP kernels multiply bf16 weights only
        quantized = getattr(self.dense_h_to_4h, "quantized", False) or getattr(self.dense_4h_to_h, "quantized", False)
        if not topo.sequence_parallel and not topo.fused_tp_comm and not quantized:
            # both GEMMs in one autograd node: GELU' runs in the epilogue of the second layer's dgrad
            x = mappings.copy_to_tp(hidden_states)
            if (residual is not None and topo.tensor_parallel_size == 1
                    and (self.output_dropout_prob == 0.0 or not self.training) and x.dtype == torch.bfloat16):
                # no reduction and no dropout between the second GEMM and the residual add: bias + residual go
                # into that GEMM's epilogue
                return OF.mlp(x, self.dense_h_to_4h.weight, self.dense_h_to_4h.bias, self.dense_4h_to_h.weight, "gelu",
                              self.dense_4h_to_h.bias, residual)
            out = OF.mlp(x, self.dense_h_to_4h.weight, self.dense_h_to_4h.bias, self.dense_4h_to_h.weight, "gelu")
            out, bias = mappings.reduce_from_tp(out), self.dense_4h_to_h.bias
        else:
            if (topo.fused_tp_comm and not quantized and hidden_states.is_cuda and hidden_states.dtype == torch.bfloat16
                    and hidden_states.dim() == 2 and (self.output_dropout_prob == 0.0 or not self.training)):
                # both linears + their collectives + bias/GELU/bias/residual as one autograd node (ops/comm_gemm.py)
                from libai_b200.ops import comm_gemm, use_native

                t = topo.tensor_parallel_size
                M, K = hidden_states.shape[0] * t, hidden_states.shape[1]
                f_loc = self.dense_h_to_4h.weight.shape[0]
                if (use_native(hidden_states) and comm_gemm.fused_supported(M, f_loc, K, t)
                        and comm_gemm.fused_supported(M, K, f_loc, t)):
                    res = residual.reshape(-1, K).contiguous() if residual is not None else None
                    return comm_gemm.tp_mlp(hidden_states.contiguous(), self.dense_h_to_4h.weight, self.dense_h_to_4h.bias,
                                            self.dense_4h_to_h.weight, self.dense_4h_to_h.bias, res, "gelu", topo.tp_group)
            inter = self.dense_h_to_4h(hidden_states, act="gelu")
            out, bias = self.dense_4h_to_h(inter)
        return OF.bias_dropout_add(out, bias, residual, self.output_dropout_prob, self.training)

    def extra_repr(self) -> str:
        return "bias_gelu_fusion={}, bias_dropout_fusion={}, dropout={}".format(
            self.bias_gelu_fusion, self.bias_dropout_fusion, self.output_dropout_prob
        )
