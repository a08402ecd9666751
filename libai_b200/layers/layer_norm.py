"""LayerNorm / RMSLayerNorm backed by the fused sm_90a norm kernels.

Spec: reference libai/layers/layer_norm.py:22-131 — parameters are replicated, normalisation is
over the trailing ``normalized_shape`` dims, ``elementwise_affine`` / ``bias`` switches, ``eps``.
Under sequence parallelism the parameters see only ``1/t`` of the tokens per rank, so their
gradients are summed over the TP group (flag ``sequence_parallel`` on the parameter, consumed by
the gradient-sync engine).
"""
from torch import nn

from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dutil

from ._param import create_parameter, ones_, zeros_


class LayerNorm(nn.Module):
    def __init__(self, normalized_shape, eps=1e-5, elementwise_affine=True, bias=True, *, layer_idx=0, dtype=None):
        super().__init__()
        if isinstance(normalized_shape, int):
            normalized_shape = (normalized_shape,)
        self.normalized_shape = tuple(normalized_shape)
        self.eps = eps
        self.elementwise_affine = elementwise_affine
        self.layer_idx = layer_idx
        if elementwise_affine:
            self.weight = create_parameter(self.normalized_shape, ones_, layer_idx=layer_idx, dtype=dtype)
            self.bias = create_parameter(self.normalized_shape, zeros_, layer_idx=layer_idx, dtype=dtype) if bias else None
            sp = dutil.get_dist_util().sequence_parallel
            for p in (self.weight, self.bias):
                if p is not None:
                    p.sequence_parallel = sp
        else:
            self.register_parameter("weight", None)
            self.register_parameter("bias", None)

    def forward(self, x):
        assert x.shape[-len(self.normalized_shape):] == self.normalized_shape
        if len(self.normalized_shape) != 1:
            lead = x.shape[: x.dim() - len(self.normalized_shape)]
            y = OF.layer_norm(
                x.reshape(*lead, -1),
                None if self.weight is None else self.weight.reshape(-1),
                None if self.bias is None else self.bias.reshape(-1),
                self.eps,
            )
            return y.view(x.shape)
        return OF.layer_norm(x, self.weight, self.bias, self.eps)

    def forward_with_skip(self, x):
        """``(norm(x), x_for_the_residual_path)``: in a pre-LN block the gradient of the skip connection is then added
        inside the LayerNorm backward kernel instead of by a separate autograd add."""
        if len(self.normalized_shape) != 1 or self.weight is None:
            return self.forward(x), x
        return OF.layer_norm_with_skip(x, self.weight, self.bias, self.eps)

    def extra_repr(self) -> str:
        return "{normalized_shape}, eps={eps}, elementwise_affine={elementwise_affine}".format(**self.__dict__)


class RMSLayerNorm(nn.Module):
    """T5 / Llama style RMS norm: ``x * rsqrt(mean(x²) + eps) * weight`` (no mean subtraction, no bias)."""

    def __init__(self, normalized_shape, eps=1e-6, *, layer_idx=0, dtype=None):
        super().__init__()
        if isinstance(normalized_shape, int):
            normalized_shape = (normalized_shape,)
        self.normalized_shape = tuple(normalized_shape)
        self.eps = eps
        self.layer_idx = layer_idx
        self.weight = create_parameter(self.normalized_shape, ones_, layer_idx=layer_idx, dtype=dtype)
        self.weight.sequence_parallel = dutil.get_dist_util().sequence_parallel

    def forward(self, x):
        return OF.rms_norm(x, self.weight, self.eps)

    def extra_repr(self) -> str:
        return f"{self.normalized_shape}, eps={self.eps}"
