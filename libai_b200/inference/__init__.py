import torch

from .engine import GenerationEngine, RequestOutput  # noqa: F401


def quantize_weights_fp8_(model, exclude=("lm_head", "output_layer")):
    """Convert, in place, every ``Linear1D`` of ``model`` whose qualified name does not end with one of ``exclude`` to
    FP8 (E4M3) weights with one fp32 scale per output channel (``Linear1D.quantize_fp8_``), and return the model.

    The weights are quantized one parameter at a time, so memory never holds two copies of the model.  Layers that are
    not a ``Linear1D`` keep their dtype: embeddings, norms, and the output heads tied to the embedding (GPT-2's and
    BLOOM's ``LMLogits``); so do the untied heads named in ``exclude``.  For inference only: a quantized layer raises
    on a forward that would need a gradient, and quantized checkpoints are neither written nor read (quantize after
    loading).  Raises ``TypeError``, converting nothing, when a weight to convert is not bf16, fp16 or fp32; layers
    already converted are left as they are, so a second call is a no-op."""
    from libai_b200.layers.linear import _FP8_SOURCE_DTYPES, Linear1D

    todo = [(n, m) for n, m in model.named_modules()
            if isinstance(m, Linear1D) and not m.fp8 and not any(n.endswith(e) for e in exclude)]
    for n, m in todo:
        if m.weight.dtype not in _FP8_SOURCE_DTYPES:
            raise TypeError(f"quantize_weights_fp8_: {n}.weight is {m.weight.dtype} (bf16, fp16 or fp32 expected)")
    for _, m in todo:
        m.quantize_fp8_()
    return model


def quantize_weights_int4_(model, exclude=("lm_head", "output_layer")):
    """Convert, in place, every ``Linear1D`` of ``model`` whose qualified name does not end with one of ``exclude`` to
    group-wise INT4 weights: 4-bit values packed two per byte, with a bf16 scale and a uint8 zero point per row and group
    of 128 input columns (``Linear1D.quantize_int4_``), and return the model.

    The layers kept as they are, and the memory and inference-only rules, are those of :func:`quantize_weights_fp8_`.
    Every layer to convert is checked before any is converted: a weight that is not bf16, fp16 or fp32 (an FP8 layer
    among them) raises ``TypeError``, and one whose input size is not a multiple of 128 or that holds a non-finite value
    raises ``ValueError``.  Layers already in INT4 are left as they are, so a second call is a no-op."""
    from libai_b200.layers.linear import _FP8_SOURCE_DTYPES, Linear1D
    from libai_b200.ops.functional import INT4_GROUP

    todo = [(n, m) for n, m in model.named_modules()
            if isinstance(m, Linear1D) and not m.int4 and not any(n.endswith(e) for e in exclude)]
    for n, m in todo:
        w = m.weight
        if m.fp8 or w.dtype not in _FP8_SOURCE_DTYPES:
            raise TypeError(f"quantize_weights_int4_: {n}.weight is {w.dtype} (bf16, fp16 or fp32 expected)")
        if w.dim() != 2 or w.shape[1] % INT4_GROUP != 0:
            raise ValueError(f"quantize_weights_int4_: {n}.weight {tuple(w.shape)} needs an input size that is a "
                             f"multiple of {INT4_GROUP}")
        if not bool(torch.isfinite(w).all()):
            raise ValueError(f"quantize_weights_int4_: {n}.weight has a non-finite value")
    for _, m in todo:
        m.quantize_int4_()
    return model
