"""Hot operators.

Every operator has two implementations:

* ``native`` – hand-written sm_90a CUDA kernels in ``libai_b200/csrc`` (wgmma/TMA GEMMs,
  fused norms, flash attention, fused optimizer, vocab-parallel cross entropy, in-kernel
  NVLink collectives).  This is the product and the only path GPU training takes.
* ``ref`` – plain PyTorch (+ ``torch.distributed``).  Test oracle, CPU/gloo plumbing path and the
  honest "NCCL + library GEMM" baseline (select with ``LIBAI_B200_IMPL=ref``).

The extension is built in-tree by ``__graft_entry__.build()`` / ``python -m libai_b200.ops.build``
and loaded from ``libai_b200/_C.so``.  On a CUDA device a missing extension is a hard error, never
a silent fallback.
"""
from __future__ import annotations

import os
import threading

import torch

_LOCK = threading.Lock()
_EXT = None
_EXT_ERR = None
_SO_PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "_C.so")
_LAUNCH_COUNT = 0


def so_path() -> str:
    return _SO_PATH


def impl() -> str:
    """'native' (default) or 'ref' (``LIBAI_B200_IMPL=ref`` forces the PyTorch path on GPU)."""
    return os.environ.get("LIBAI_B200_IMPL", "native")


class _FastOps:
    """``torch.ops.libai_b200`` with every operator resolved once to its ``.default`` overload.  Calling the
    ``OpOverloadPacket`` (what ``torch.ops.ns.name(...)`` is) re-resolves the overload on every call — a few
    microseconds of Python per kernel launch, several hundred times per training step."""

    def __init__(self, namespace):
        self._ns = namespace

    def __getattr__(self, name):
        packet = getattr(self._ns, name)
        op = getattr(packet, "default", packet)
        setattr(self, name, op)
        return op


def load_ext(required: bool = True):
    """Load ``libai_b200/_C.so`` once and return the operator namespace (``torch.ops.libai_b200``)."""
    global _EXT, _EXT_ERR
    if _EXT is not None:
        return _EXT
    with _LOCK:
        if _EXT is not None:
            return _EXT
        try:
            if not os.path.exists(_SO_PATH):
                raise FileNotFoundError(
                    f"{_SO_PATH} not found - build it with `python -m libai_b200.ops.build`"
                )
            torch.ops.load_library(_SO_PATH)
            _EXT = _FastOps(torch.ops.libai_b200)
        except Exception as e:  # noqa
            _EXT_ERR = e
            if required:
                raise RuntimeError(
                    "libai_b200 native extension is required on CUDA devices but could not be "
                    f"loaded: {e}"
                ) from e
            return None
    return _EXT


def use_native(*tensors) -> bool:
    """True when the native sm_90a kernel must be used for these tensors."""
    if impl() != "native":
        return False
    for t in tensors:
        if isinstance(t, torch.Tensor):
            if not t.is_cuda:
                return False
            load_ext(required=True)
            return True
    return False


def count_launch(n: int = 1) -> None:
    global _LAUNCH_COUNT
    _LAUNCH_COUNT += n


def launch_count() -> int:
    """Number of native kernel launches issued through the python wrappers (bench bookkeeping)."""
    return _LAUNCH_COUNT


def reset_launch_count() -> None:
    global _LAUNCH_COUNT
    _LAUNCH_COUNT = 0


# --------------------------------------------------------------------------------------
# fp8 (E4M3) forward GEMMs — opt-in (``train.fp8.enabled`` / ``LIBAI_B200_FP8=1``)
# --------------------------------------------------------------------------------------
_FP8 = os.environ.get("LIBAI_B200_FP8", "0") == "1"
_FP8_EPOCH = 0


def set_fp8(enabled: bool) -> None:
    """Run the forward GEMMs of the linear layers with E4M3 operands (per-tensor dynamic scaling, fp32 accumulation
    in registers, bf16 outputs); backward GEMMs stay bf16 on the saved bf16 operands."""
    global _FP8
    _FP8 = bool(enabled)


def fp8_enabled() -> bool:
    return _FP8


def fp8_weight_epoch() -> int:
    return _FP8_EPOCH


def bump_fp8_weight_epoch() -> None:
    """Invalidate cached quantised weights (called by the optimizers after they rewrote the parameters in place —
    the native update kernels do not bump ``Tensor._version``)."""
    global _FP8_EPOCH
    _FP8_EPOCH += 1


# --------------------------------------------------------------------------------------
# bias gradient of the MLP's first linear accumulated by the dgrad call straight into the bias' fp32 main_grad: on one
# GPU an ordered column-sum pass launched with the dgrad GEMM, under tensor parallelism inside the all-gather GEMM's
# epilogue.  Off: the layer returns the column sums as a separate bf16 gradient.
# --------------------------------------------------------------------------------------
_FUSED_BIAS_GRAD = os.environ.get("LIBAI_B200_FUSED_BIAS_GRAD", "1") == "1"


def fused_bias_grad() -> bool:
    return _FUSED_BIAS_GRAD


def set_fused_bias_grad(enabled: bool) -> None:
    global _FUSED_BIAS_GRAD
    _FUSED_BIAS_GRAD = bool(enabled)
