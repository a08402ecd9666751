"""The native ops' argument checks, run on the real extension without a GPU.

The extension loads and dispatches on a machine without one.  With CPU tensors every valid argument set reaches the
last rule, that the op's reference tensor is a CUDA tensor; every mutation of one argument is rejected by its own rule
before that.  A tensor on another device is a ``meta`` tensor here, so each rejection path runs with nothing launched.
"""
import os

import pytest
import torch

from libai_b200.ops import build as ops_build
from tests import op_args_cases as C

CASES = C.cases("cpu")


@pytest.fixture(scope="module")
def ext():
    if not os.path.exists(ops_build.NVCC):
        pytest.skip("needs nvcc to build the extension")
    torch.ops.load_library(ops_build.build(force=False))
    return torch.ops.libai_b200


def _error(fn):
    with pytest.raises(RuntimeError) as e:
        fn()
    return str(e.value).splitlines()[0]


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_valid_arguments_fail_only_for_not_being_on_a_cuda_device(ext, case):
    msg = _error(lambda: getattr(ext, case.op)(*case.values()))
    assert msg.startswith(f"{case.op}: ") and "must be a CUDA tensor" in msg, msg


MUTATIONS = [(c, m) for c in CASES for m in c.mutations]


@pytest.mark.parametrize("case,mutation", MUTATIONS, ids=[f"{c.id}-{n}-{k}" for c, (n, k, _) in MUTATIONS])
def test_each_mutation_is_rejected_by_its_own_rule(ext, case, mutation):
    name, kind, fragment = mutation
    msg = _error(lambda: getattr(ext, case.op)(*C.mutated(case, name, kind, "meta")))
    assert fragment in msg, msg
    assert "must be a CUDA tensor" not in msg, msg
