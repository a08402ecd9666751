"""The native autograd wrappers of ``linear`` and ``mlp`` on the CPU, with the extension replaced by a small PyTorch
stub of the kernels they call: every ``requires_grad`` subset of the inputs (the bias alone included) must run the
backward and return the gradients fp64 autograd returns, within the bounds of ``tests/autograd_ref.py``."""
import itertools

import pytest
import torch

from libai_b200.ops import functional as OF
from tests import autograd_ref as AR
from tests import dense_ref as R


class StubExt:
    """The kernels ``_LinearFn`` / ``_MLPFn`` call, in fp32 PyTorch with the kernels' output dtypes.  Like the
    bindings' schemas, ``act_bwd`` and ``dgrad_actgrad`` take a required pre-activation."""

    @staticmethod
    def _act(v, act):
        y, _ = R.act_ref(v.double(), act)
        return y.float()

    @staticmethod
    def _dact(v, act):
        _, d = R.act_ref(v.double(), act)
        return d.float()

    def linear_fwd(self, x, w, bias, act, need_pre):
        pre = x.float() @ w.float().t()
        if bias is not None:
            pre = pre + bias.float()
        return self._act(pre, act).to(x.dtype), (pre.to(x.dtype) if need_pre else None)

    def linear_bias_residual(self, x, w, bias, residual):
        y = x.float() @ w.float().t() + residual.float()
        return (y if bias is None else y + bias.float()).to(x.dtype)

    def gemm(self, a, b, layout, bias, out, accumulate, dtype):
        A, B = R.gemm_operands(a.float(), b.float(), layout)
        c = A @ B.t()
        if out is None:
            return c.to(dtype)
        if accumulate:
            out.add_(c)
        else:
            out.copy_(c)
        return out

    def act_bwd(self, gy, pre, act):
        if pre is None:
            raise RuntimeError("act_bwd(): argument 'pre' must be Tensor, not None")
        return (gy.float() * self._dact(pre, act)).to(gy.dtype)

    def dgrad_actgrad(self, gy, w, pre, act, bias_grad):
        if pre is None:
            raise RuntimeError("dgrad_actgrad(): argument 'pre' must be Tensor, not None")
        d = ((gy.float() @ w.float()) * self._dact(pre, act)).to(gy.dtype)
        if bias_grad is not None:
            bias_grad.add_(d.float().sum(0))
        return d

    def colsum(self, x, accum=None):
        s = x.float().sum(0)
        if accum is None:
            return s
        return accum.add_(s)


@pytest.fixture
def stub(monkeypatch):
    """``functional`` dispatching to the stub for CPU tensors."""
    ext = StubExt()
    monkeypatch.setattr(OF, "use_native", lambda *tensors: True)
    monkeypatch.setattr(OF, "load_ext", lambda required=True: ext)
    return ext


def rand(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).bfloat16()


def subsets(names):
    return [s for n in range(1, len(names) + 1) for s in itertools.combinations(names, n)]


def check_param_grad(t, ref, bound, what):
    """A gradient returned to autograd in the parameter's dtype: one more rounding of that dtype."""
    assert t.grad is not None, f"{what}: no gradient"
    R.check(t.grad, ref, R.ROUND[t.dtype] * ref.abs() + bound * (1 + R.ROUND[t.dtype]), what)


@pytest.mark.parametrize("act", [None, "gelu", "gelu_tanh", "relu", "silu", "quick_gelu"])
@pytest.mark.parametrize("grads", subsets("xwb"), ids="".join)
def test_linear_every_requires_grad_subset(stub, act, grads):
    M, K, N = 21, 24, 16
    x0, w0, b0, gy = rand(M, K, seed=1), rand(N, K, seed=2, scale=0.3), rand(N, seed=3), rand(M, N, seed=4)
    x, w, b = (t.clone().requires_grad_(n in grads) for t, n in ((x0, "x"), (w0, "w"), (b0, "b")))
    y = OF.linear(x, w, b, act)
    assert y.grad_fn is not None and type(y.grad_fn).__name__ == "_LinearFnBackward", "the native wrapper did not run"
    y.backward(gy)
    ref = AR.linear_ref(x0, w0, b0, gy, act)
    R.check(y, *ref["y"], "y")
    for t, n, key in ((x, "x", "gx"), (w, "w", "gw"), (b, "b", "gb")):
        if n in grads:
            check_param_grad(t, *ref[key], f"act {act} grads {grads} {key}")
        else:
            assert t.grad is None


@pytest.mark.parametrize("act", ["gelu", "relu"])
@pytest.mark.parametrize("grads", subsets(["x", "w1", "b1", "w2", "b2", "res"]), ids="-".join)
def test_mlp_every_requires_grad_subset(stub, act, grads):
    M, K, Fh = 21, 24, 40
    x0, w10, b10 = rand(M, K, seed=1), rand(Fh, K, seed=2, scale=0.3), rand(Fh, seed=3)
    w20, b20, r0, gy = rand(K, Fh, seed=4, scale=0.3), rand(K, seed=5), rand(M, K, seed=6), rand(M, K, seed=7)
    leaves = {n: t.clone().requires_grad_(n in grads)
              for n, t in (("x", x0), ("w1", w10), ("b1", b10), ("w2", w20), ("b2", b20), ("res", r0))}
    y = OF.mlp(leaves["x"], leaves["w1"], leaves["b1"], leaves["w2"], act, leaves["b2"], leaves["res"])
    assert type(y.grad_fn).__name__ == "_MLPFnBackward", "the native wrapper did not run"
    y.backward(gy)
    ref = AR.mlp_ref(x0, w10, b10, w20, gy, act, b20, r0)
    R.check(y, *ref["y"], "y")
    for n, t in leaves.items():
        if n in grads:
            check_param_grad(t, *ref["g" + n], f"act {act} grads {grads} g{n}")
        else:
            assert t.grad is None


def test_linear_bias_only_accumulates_into_main_grad(stub):
    """BitFit / LoRA ``bias="all"``: frozen weight, trainable bias with an fp32 main_grad, two micro-batches."""
    M, K, N = 21, 24, 16
    x, w = rand(M, K, seed=1), rand(N, K, seed=2, scale=0.3)
    b = rand(N, seed=3).requires_grad_(True)
    base = torch.randn(N, generator=torch.Generator().manual_seed(9))
    b.main_grad = base.clone()
    want, bound = base.double(), torch.zeros(N, dtype=torch.float64)
    for step in range(2):
        gy = rand(M, N, seed=10 + step)
        OF.linear(x, w, b, "gelu").backward(gy)
        assert b.grad is None and b.grad_added_to_main_grad
        ref, e = AR.linear_ref(x, w, b.detach(), gy, "gelu")["gb"]
        want, bound = want + ref, bound + e
        bound = bound + R.ROUND[torch.float32] * want.abs()
    R.check(b.main_grad, want, bound, "bias main_grad after two micro-batches")
