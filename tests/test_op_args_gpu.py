"""The native ops' argument checks on the GPU: every valid argument set of ``tests/op_args_cases.py`` runs and returns
its documented output shapes, and every mutation of one argument is rejected before a launch (another device is the
host here).  ``test_op_args_cpu.py`` shows on the same table that each mutation fails its own rule."""
import pytest
import torch

from tests import op_args_cases as C

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


@pytest.fixture(scope="module")
def cases():
    return {c.id: c for c in C.cases(DEV)}


IDS = [c.id for c in C.cases("meta")]
MUTATIONS = [(c.id, m) for c in C.cases("meta") for m in c.mutations]


@pytest.mark.parametrize("cid", IDS)
def test_valid_arguments_run(ext, cases, cid):
    case = cases[cid]
    out = getattr(ext, case.op)(*case.values())
    torch.cuda.synchronize()
    if case.outputs is None:
        assert out is None
        return
    outs = out if isinstance(out, (tuple, list)) else (out,)
    assert [tuple(t.shape) for t in outs] == case.outputs
    assert all(t.device == torch.device(DEV) for t in outs)


@pytest.mark.parametrize("cid,mutation", MUTATIONS, ids=[f"{c}-{n}-{k}" for c, (n, k, _) in MUTATIONS])
def test_each_mutation_is_rejected(ext, cases, cid, mutation):
    case = cases[cid]
    name, kind, fragment = mutation
    with pytest.raises(RuntimeError, match=fragment):
        getattr(ext, case.op)(*C.mutated(case, name, kind, "cpu"))
