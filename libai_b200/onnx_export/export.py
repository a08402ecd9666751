"""Graph export of trained models.

Spec: reference libai/onnx_export/{gpt2_to_onnx.py,t5_to_onnx.py} — wrap the eager model, trace it with example
inputs and write an ONNX file (there through ``oneflow_onnx``).  Here ``torch.onnx.export`` does the conversion of
the PyTorch reference path of the model (``LIBAI_B200_IMPL=ref``: the hand-written sm_90a kernels have no ONNX
symbolics, the exported graph uses the mathematically identical library ops).  When the ``onnx`` package is not
installed the model is exported as a TorchScript trace instead (``.pt``), which serves the same deployment role.
"""
from __future__ import annotations

import logging
import os
from typing import Dict, Sequence, Tuple

import torch
from torch import nn

logger = logging.getLogger(__name__)


class ExportWrapper(nn.Module):
    """Positional-input / tensor-output façade over a dict-returning libai_b200 model."""

    def __init__(self, model: nn.Module, input_names: Sequence[str], output_key: str, **fixed_kwargs):
        super().__init__()
        self.model, self.input_names, self.output_key, self.fixed_kwargs = model, list(input_names), output_key, fixed_kwargs

    def forward(self, *inputs):
        out = self.model(**dict(zip(self.input_names, inputs)), **self.fixed_kwargs)
        return out[self.output_key] if isinstance(out, dict) else out


def onnx_available() -> bool:
    try:
        import onnx  # noqa: F401

        return True
    except ImportError:
        return False


def export_model(model: nn.Module, example_inputs: Dict[str, torch.Tensor], output_key: str, path: str,
                 dynamic_axes: Dict[str, Dict[int, str]] = None, opset: int = 17, **fixed_kwargs) -> Tuple[str, str]:
    """Export ``model`` called as ``model(**example_inputs, **fixed_kwargs)[output_key]``.
    Returns ``(format, file)`` with format ``"onnx"`` or ``"torchscript"``."""
    prev = os.environ.get("LIBAI_B200_IMPL")
    os.environ["LIBAI_B200_IMPL"] = "ref"  # trace the library-op path
    try:
        model = model.eval()
        names = list(example_inputs.keys())
        wrapper = ExportWrapper(model, names, output_key, **fixed_kwargs)
        args = tuple(example_inputs[n] for n in names)
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with torch.no_grad():
            if onnx_available():
                file = path if path.endswith(".onnx") else path + ".onnx"
                torch.onnx.export(wrapper, args, file, input_names=names, output_names=[output_key],
                                  dynamic_axes=dynamic_axes, opset_version=opset, do_constant_folding=True)
                return "onnx", file
            logger.warning("`onnx` is not installed: exporting a TorchScript trace instead of an ONNX file")
            file = (path[:-5] if path.endswith(".onnx") else path) + ".pt"
            traced = torch.jit.trace(wrapper, args, check_trace=False, strict=False)
            traced.save(file)
            return "torchscript", file
    finally:
        if prev is None:
            os.environ.pop("LIBAI_B200_IMPL", None)
        else:
            os.environ["LIBAI_B200_IMPL"] = prev
