"""Where every native linear-type autograd node sends each parameter's gradient, on the CPU with the extension replaced
by PyTorch stubs (``tests/test_autograd_cpu.py``) and the tensor-parallel collectives by their world-size-1 forms
(all-gather and reduce-scatter are the identity).

For every ``requires_grad`` subset of a node's inputs, with and without an fp32 ``main_grad`` on the trainable
parameters, each test checks:

* the gradients against the fp64 references of ``tests/autograd_ref.py``, whether they land in ``main_grad`` (with
  ``grad_added_to_main_grad`` set and no ``.grad``) or reach autograd in the parameter's dtype;
* the extension calls the node issues, in order, written out below;
* the node's ``count_launch`` tally (``gpu_launches`` of the benchmark line).
"""
import types

import pytest
import torch
import torch.nn.functional as F

from libai_b200 import ops
from libai_b200.ops import comm_gemm as CG
from libai_b200.ops import functional as OF
from libai_b200.ops import gated_mlp as GM
from tests import autograd_ref as AR
from tests import dense_ref as R
from tests.test_autograd_cpu import StubExt, check_param_grad, rand, subsets

M, K, FH = 21, 24, 16
LAYOUT = {0: "NT", 1: "NN", 2: "TN"}


class RecordingExt(StubExt):
    """The stub kernels plus SwiGLU, each call recorded as one line: the op, its GEMM layout, and the ``main_grad``
    it accumulates into (``+name``)."""

    def __init__(self):
        self.calls = []
        self.names = {}      # data_ptr of a main_grad -> its parameter's name

    def dst(self, t):
        return f" +{self.names.get(t.data_ptr(), '?')}" if t is not None else ""

    def linear_fwd(self, x, w, bias, act, need_pre):
        self.calls.append("linear_fwd" + (" pre" if need_pre else ""))
        return super().linear_fwd(x, w, bias, act, need_pre)

    def linear_bias_residual(self, x, w, bias, residual):
        self.calls.append("linear_bias_residual")
        return super().linear_bias_residual(x, w, bias, residual)

    def gemm(self, a, b, layout, bias, out, accumulate, dtype):
        assert (out is not None) == accumulate
        self.calls.append(f"gemm {LAYOUT[layout]}" + self.dst(out))
        return super().gemm(a, b, layout, bias, out, accumulate, dtype)

    def act_bwd(self, gy, pre, act):
        self.calls.append("act_bwd")
        return super().act_bwd(gy, pre, act)

    def dgrad_actgrad(self, gy, w, pre, act, bias_grad):
        self.calls.append("dgrad_actgrad" + self.dst(bias_grad))
        return super().dgrad_actgrad(gy, w, pre, act, bias_grad)

    def colsum(self, x, accum=None):
        self.calls.append("colsum" + self.dst(accum))
        return super().colsum(x, accum)

    def swiglu_packed_fwd(self, gu):
        self.calls.append("swiglu_fwd")
        g, u = gu.double().chunk(2, 1)
        return (F.silu(g) * u).to(gu.dtype)

    def swiglu_packed_bwd(self, dh, gu):
        self.calls.append("swiglu_bwd")
        g, u = gu.double().chunk(2, 1)
        s, d = torch.sigmoid(g), dh.double()
        return torch.cat([d * u * s * (1 + g * (1 - s)), d * g * s], 1).to(dh.dtype)


class WorldOfOne:
    """``comm_gemm.ag_gemm`` / ``gemm_rs`` / ``ag_wgrad`` on one rank, with the launch counts of the real ones.  The
    gathered buffer ``ag_gemm`` returns holds NaN unless ``fill_local`` asked for its (here: all) local rows."""

    def __init__(self, ext):
        self.ext = ext

    def ag_gemm(self, x_shard, w, bias, act, group, layout=0, need_pre=False, pre_in=None, colsum=None,
                fill_local=False):
        ext = self.ext
        ext.calls.append(f"ag_gemm {LAYOUT[layout]}" + (" pre" if need_pre else "") + (" act'" if pre_in is not None
                         else "") + ext.dst(colsum) + (" fill" if fill_local else ""))
        ops.count_launch(2 if fill_local else 1)
        if layout == 0:
            assert pre_in is None and colsum is None
            y, pre = StubExt.linear_fwd(ext, x_shard, w, bias, OF._ACT_IDS[act], need_pre)
        elif pre_in is None:
            assert bias is None and act is None and colsum is None and not need_pre
            y, pre = StubExt.gemm(ext, x_shard, w, 1, None, None, False, torch.bfloat16), None
        else:
            assert bias is None and not need_pre
            y, pre = StubExt.dgrad_actgrad(ext, x_shard, w, pre_in, OF._ACT_IDS[act], colsum), None
        gathered = x_shard.clone() if fill_local else torch.full_like(x_shard, float("nan"))
        return y, pre, gathered

    def gemm_rs(self, x, w, bias, residual, group, layout=0):
        self.ext.calls.append(f"gemm_rs {LAYOUT[layout]}")
        ops.count_launch()
        A, B = R.gemm_operands(x.float(), w.float(), layout)
        y = A @ B.t()
        for t in (bias, residual):
            if t is not None:
                y = y + t.float()
        return y.to(x.dtype)

    def ag_wgrad(self, gy, x_shard, out, accumulate, group):
        self.ext.calls.append("ag_wgrad" + (self.ext.dst(out) if accumulate else ""))
        ops.count_launch()
        c = gy.float().t() @ x_shard.float()
        out.add_(c) if accumulate else out.copy_(c)


@pytest.fixture
def ext(monkeypatch):
    ext = RecordingExt()
    comm = WorldOfOne(ext)
    monkeypatch.setattr(OF, "use_native", lambda *tensors: True)
    for mod in (OF, GM, CG):
        monkeypatch.setattr(mod, "load_ext", lambda required=True: ext)
    for name in ("ag_gemm", "gemm_rs", "ag_wgrad"):
        monkeypatch.setattr(CG, name, getattr(comm, name))
    monkeypatch.setattr(CG, "_state", lambda group: types.SimpleNamespace(rank=0, world=1))
    return ext


@pytest.fixture(params=[True, False], ids=["fused_bias_grad", "unfused_bias_grad"])
def fused_bias_grad(request, monkeypatch):
    monkeypatch.setattr(ops, "_FUSED_BIAS_GRAD", request.param)
    return request.param


@pytest.fixture(params=[True, False], ids=["save_gathered", "regather"])
def save_gathered(request, monkeypatch):
    monkeypatch.setattr(CG, "_SAVE_GATHERED", request.param)
    return request.param


def make_leaves(ext, values, params, grads, main_grad, one_buffer=()):
    """Leaves named as ``values``; the ``params`` among them are ``Parameter``s, those in ``one_buffer`` adjacent in one
    buffer (as after the optimizer's setup).  With ``main_grad`` each trainable parameter gets a random fp32
    ``main_grad``, adjacent too for ``one_buffer``.  Returns (leaves, main_grad bases)."""
    flat = torch.cat([values[n].reshape(-1) for n in one_buffer]) if one_buffer else None
    mflat = torch.randn(flat.numel(), generator=torch.Generator().manual_seed(99)) if one_buffer else None
    leaves, bases, off = {}, {}, 0
    for i, (n, v) in enumerate(values.items()):
        if n in one_buffer:
            data, mdata = flat[off: off + v.numel()].view(v.shape), mflat[off: off + v.numel()].view(v.shape)
            off += v.numel()
        else:
            data = v.clone()
            mdata = torch.randn(v.shape, generator=torch.Generator().manual_seed(100 + i))
        leaves[n] = (torch.nn.Parameter(data, requires_grad=n in grads) if n in params
                     else data.requires_grad_(n in grads))
        if main_grad and n in params and n in grads:
            leaves[n].main_grad = mdata
            bases[n] = mdata.clone()
            ext.names[mdata.data_ptr()] = n
    return leaves, bases


def check_grads(leaves, grads, bases, to_main, ref, what):
    """Each leaf's gradient: in ``main_grad`` for the names in ``to_main``, from autograd for the other trainable ones,
    none for the frozen ones; a ``main_grad`` that gets no gradient stays as it was."""
    for n, t in leaves.items():
        flag = getattr(t, "grad_added_to_main_grad", False)
        if n not in grads:
            assert t.grad is None and not flag, f"{what}: frozen {n} got a gradient"
        elif n in to_main:
            assert t.grad is None and flag, f"{what}: {n} did not go to main_grad"
            r, e = ref["g" + n]
            want = bases[n].double() + r
            R.check(t.main_grad, want, e + R.ROUND[torch.float32] * want.abs(), f"{what} {n} main_grad")
        else:
            assert not flag, f"{what}: {n} flagged but returned to autograd"
            check_param_grad(t, *ref["g" + n], f"{what} g{n}")
            if n in bases:
                assert torch.equal(t.main_grad, bases[n]), f"{what}: {n} main_grad changed"


def run(ext, fn, leaves, gy):
    ops.reset_launch_count()
    y = fn(*leaves.values())
    y.backward(gy)
    return y, ops.launch_count()


def dst(n, to_main):
    return f" +{n}" if n in to_main else ""


# ----------------------------------------------------------------------------------------------------- single device
@pytest.mark.parametrize("main_grad", [True, False], ids=["main_grad", "autograd"])
@pytest.mark.parametrize("act", [None, "gelu"])
@pytest.mark.parametrize("grads", subsets("xwb"), ids="".join)
def test_linear(ext, grads, act, main_grad):
    values = dict(x=rand(M, K, seed=1), w=rand(FH, K, seed=2, scale=0.3), b=rand(FH, seed=3))
    gy = rand(M, FH, seed=4)
    leaves, bases = make_leaves(ext, values, "wb", grads, main_grad)
    y, tally = run(ext, lambda x, w, b: OF.linear(x, w, b, act), leaves, gy)
    ref = AR.linear_ref(values["x"], values["w"], values["b"], gy, act)
    R.check(y, *ref["y"], "y")
    to_main = set(bases)
    want = ["linear_fwd pre" if act else "linear_fwd"] + (["act_bwd"] if act else []) + (
        ["gemm NN"] if "x" in grads else []) + ([f"gemm TN{dst('w', to_main)}"] if "w" in grads else []) + (
        [f"colsum{dst('b', to_main)}"] if "b" in grads else [])
    assert ext.calls == want
    assert tally == len(want)
    check_grads(leaves, grads, bases, to_main, ref, f"linear act {act} grads {grads}")


@pytest.mark.parametrize("main_grad", [True, False], ids=["main_grad", "autograd"])
@pytest.mark.parametrize("grads", subsets(["x", "w", "b", "res"]), ids="-".join)
def test_linear_bias_residual(ext, grads, main_grad):
    values = dict(x=rand(M, K, seed=1), w=rand(FH, K, seed=2, scale=0.3), b=rand(FH, seed=3), res=rand(M, FH, seed=5))
    gy = rand(M, FH, seed=4)
    leaves, bases = make_leaves(ext, values, "wb", grads, main_grad)
    y, tally = run(ext, OF.linear_bias_residual, leaves, gy)
    ref = AR.linear_ref(values["x"], values["w"], values["b"], gy, None)
    ref["gres"] = (gy.double(), torch.zeros(M, FH, dtype=torch.float64))
    yr = ref["y"][0] + values["res"].double()
    R.check(y, yr, ref["y"][1] + (AR.U8 + 2.0 ** -23) * yr.abs(), "y")
    to_main = set(bases)
    want = ["linear_bias_residual"] + (["gemm NN"] if "x" in grads else []) + (
        [f"gemm TN{dst('w', to_main)}"] if "w" in grads else []) + ([f"colsum{dst('b', to_main)}"] if "b" in grads
                                                                    else [])
    assert ext.calls == want
    assert tally == len(want)
    check_grads(leaves, grads, bases, to_main, ref, f"linear_bias_residual grads {grads}")


MLP_INPUTS = ["x", "w1", "b1", "w2", "b2", "res"]


def mlp_values():
    return dict(x=rand(M, K, seed=1), w1=rand(FH, K, seed=2, scale=0.3), b1=rand(FH, seed=3),
                w2=rand(K, FH, seed=4, scale=0.3), b2=rand(K, seed=5), res=rand(M, K, seed=6))


@pytest.mark.parametrize("main_grad", [True, False], ids=["main_grad", "autograd"])
@pytest.mark.parametrize("grads", subsets(MLP_INPUTS), ids="-".join)
def test_mlp(ext, grads, main_grad, fused_bias_grad):
    values, gy = mlp_values(), rand(M, K, seed=7)
    leaves, bases = make_leaves(ext, values, ["w1", "b1", "w2", "b2"], grads, main_grad)
    y, tally = run(ext, lambda x, w1, b1, w2, b2, res: OF.mlp(x, w1, b1, w2, "gelu", b2, res), leaves, gy)
    ref = AR.mlp_ref(values["x"], values["w1"], values["b1"], values["w2"], gy, "gelu", values["b2"], values["res"])
    R.check(y, *ref["y"], "y")
    to_main = set(bases)
    fused_b1 = fused_bias_grad and "b1" in to_main
    want = ["linear_fwd pre", "linear_bias_residual", "dgrad_actgrad" + (" +b1" if fused_b1 else "")] + (
        [f"gemm TN{dst('w2', to_main)}"] if "w2" in grads else []) + (
        [f"gemm TN{dst('w1', to_main)}"] if "w1" in grads else []) + (
        [f"colsum{dst('b1', to_main)}"] if "b1" in grads and not fused_b1 else []) + (
        ["gemm NN"] if "x" in grads else []) + ([f"colsum{dst('b2', to_main)}"] if "b2" in grads else [])
    assert ext.calls == want
    assert tally == len(want)
    check_grads(leaves, grads, bases, to_main, ref, f"mlp grads {grads}")


GATED_INPUTS = ["x", "wg", "wu", "wd"]


def gated_values():
    return dict(x=rand(M, K, seed=1), wg=rand(FH, K, seed=2, scale=0.3), wu=rand(FH, K, seed=3, scale=0.3),
                wd=rand(K, FH, seed=4, scale=0.3))


def gated_to_main(ext, leaves, bases):
    """The gate and up weights' gradients go to main_grad only when both own one (the fused [2F, K] view over them)."""
    to_main = set(bases)
    if {"wg", "wu"} <= to_main:
        ext.names[leaves["wg"].main_grad.data_ptr()] = "wg|wu"
    else:
        to_main -= {"wg", "wu"}
    return to_main


@pytest.mark.parametrize("main_grad", [True, False], ids=["main_grad", "autograd"])
@pytest.mark.parametrize("grads", subsets(GATED_INPUTS), ids="-".join)
def test_gated_mlp(ext, grads, main_grad):
    values, gy = gated_values(), rand(M, K, seed=7)
    leaves, bases = make_leaves(ext, values, ["wg", "wu", "wd"], grads, main_grad, one_buffer=("wg", "wu"))
    to_main = gated_to_main(ext, leaves, bases)
    y, tally = run(ext, GM.gated_mlp, leaves, gy)
    ref = AR.gated_mlp_ref(values["x"], values["wg"], values["wu"], values["wd"], gy)
    R.check(y, *ref["y"], "y")
    gate_up = "wg" in grads or "wu" in grads
    want = ["gemm NT", "swiglu_fwd", "gemm NT", "gemm NN"] + (
        [f"gemm TN{dst('wd', to_main)}"] if "wd" in grads else []) + ["swiglu_bwd"] + (
        ["gemm NN"] if "x" in grads else []) + (
        ["gemm TN" + (" +wg|wu" if "wg" in to_main else "")] if gate_up else [])
    assert ext.calls == want
    # the backward counts its dgrad of x whether or not it runs
    assert tally == 6 + ("wd" in grads) + gate_up
    check_grads(leaves, grads, bases, to_main, ref, f"gated_mlp grads {grads}")


# ------------------------------------------------------------------------------------------------ tensor parallel
@pytest.mark.parametrize("main_grad", [True, False], ids=["main_grad", "autograd"])
@pytest.mark.parametrize("act", [None, "gelu"])
@pytest.mark.parametrize("grads", subsets("xwb"), ids="".join)
def test_column_parallel_linear(ext, grads, act, main_grad, save_gathered):
    values = dict(x=rand(M, K, seed=1), w=rand(FH, K, seed=2, scale=0.3), b=rand(FH, seed=3))
    gy = rand(M, FH, seed=4)
    leaves, bases = make_leaves(ext, values, "wb", grads, main_grad)
    y, tally = run(ext, lambda x, w, b: CG.column_parallel_linear(x, w, b, act, None), leaves, gy)
    ref = AR.linear_ref(values["x"], values["w"], values["b"], gy, act)
    R.check(y, *ref["y"], "y")
    to_main = set(bases)
    snapshot = save_gathered and "w" in grads
    want = ["ag_gemm NT" + (" pre" if act else "")] + (["act_bwd"] if act else []) + (
        ["gemm_rs NN"] if "x" in grads else []) + (
        [("gemm TN" if snapshot else "ag_wgrad") + dst("w", to_main)] if "w" in grads else []) + (
        [f"colsum{dst('b', to_main)}"] if "b" in grads else [])
    assert ext.calls == want
    assert tally == len(want) + 2 * snapshot          # the gathered snapshot: a clone and a copy
    check_grads(leaves, grads, bases, to_main, ref, f"column_parallel_linear act {act} grads {grads}")


@pytest.mark.parametrize("main_grad", [True, False], ids=["main_grad", "autograd"])
@pytest.mark.parametrize("grads", subsets(["x", "w", "b", "res"]), ids="-".join)
def test_row_parallel_linear(ext, grads, main_grad):
    values = dict(x=rand(M, K, seed=1), w=rand(FH, K, seed=2, scale=0.3), b=rand(FH, seed=3), res=rand(M, FH, seed=5))
    gy = rand(M, FH, seed=4)
    leaves, bases = make_leaves(ext, values, "wb", grads, main_grad)
    y, tally = run(ext, lambda x, w, b, res: CG.row_parallel_linear(x, w, b, res, None), leaves, gy)
    ref = AR.linear_ref(values["x"], values["w"], values["b"], gy, None)
    ref["gres"] = (gy.double(), torch.zeros(M, FH, dtype=torch.float64))
    yr = ref["y"][0] + values["res"].double()
    R.check(y, yr, ref["y"][1] + (AR.U8 + 2.0 ** -23) * yr.abs(), "y")
    to_main = set(bases)
    want = ["gemm_rs NT", "ag_gemm NN" + (" fill" if "w" in grads else "")] + (
        [f"gemm TN{dst('w', to_main)}"] if "w" in grads else []) + ([f"colsum{dst('b', to_main)}"] if "b" in grads
                                                                    else [])
    assert ext.calls == want
    assert tally == len(want) + ("w" in grads)        # the fill of the gathered buffer's local rows
    check_grads(leaves, grads, bases, to_main, ref, f"row_parallel_linear grads {grads}")


@pytest.mark.parametrize("main_grad", [True, False], ids=["main_grad", "autograd"])
@pytest.mark.parametrize("grads", subsets(MLP_INPUTS), ids="-".join)
def test_tp_mlp(ext, grads, main_grad, fused_bias_grad, save_gathered):
    values, gy = mlp_values(), rand(M, K, seed=7)
    leaves, bases = make_leaves(ext, values, ["w1", "b1", "w2", "b2"], grads, main_grad)
    y, tally = run(ext, lambda x, w1, b1, w2, b2, res: CG.tp_mlp(x, w1, b1, w2, b2, res, "gelu", None), leaves, gy)
    ref = AR.mlp_ref(values["x"], values["w1"], values["b1"], values["w2"], gy, "gelu", values["b2"], values["res"])
    R.check(y, *ref["y"], "y")
    to_main = set(bases)
    fused_b1 = fused_bias_grad and "b1" in to_main
    snapshot = save_gathered and "w1" in grads
    want = ["ag_gemm NT pre", "gemm_rs NT",
            "ag_gemm NN act'" + (" +b1" if fused_b1 else "") + (" fill" if "w2" in grads else "")] + (
        [f"gemm TN{dst('w2', to_main)}"] if "w2" in grads else []) + (
        [f"colsum{dst('b2', to_main)}"] if "b2" in grads else []) + (["gemm_rs NN"] if "x" in grads else []) + (
        [("gemm TN" if snapshot else "ag_wgrad") + dst("w1", to_main)] if "w1" in grads else []) + (
        [f"colsum{dst('b1', to_main)}"] if "b1" in grads and not fused_b1 else [])
    assert ext.calls == want
    assert tally == len(want) + ("w2" in grads) + 2 * snapshot
    check_grads(leaves, grads, bases, to_main, ref, f"tp_mlp grads {grads}")


@pytest.mark.parametrize("main_grad", [True, False], ids=["main_grad", "autograd"])
@pytest.mark.parametrize("grads", subsets(GATED_INPUTS + ["res"]), ids="-".join)
def test_tp_gated_mlp(ext, grads, main_grad):
    values, gy = dict(gated_values(), res=rand(M, K, seed=6)), rand(M, K, seed=7)
    leaves, bases = make_leaves(ext, values, ["wg", "wu", "wd"], grads, main_grad, one_buffer=("wg", "wu"))
    to_main = gated_to_main(ext, leaves, bases)
    y, tally = run(ext, lambda x, wg, wu, wd, res: GM.tp_gated_mlp(x, wg, wu, wd, res, None), leaves, gy)
    ref = AR.gated_mlp_ref(values["x"], values["wg"], values["wu"], values["wd"], gy, values["res"])
    R.check(y, *ref["y"], "y")
    want = ["ag_gemm NT", "swiglu_fwd", "gemm_rs NT", "ag_gemm NN" + (" fill" if "wd" in grads else "")] + (
        [f"gemm TN{dst('wd', to_main)}"] if "wd" in grads else []) + ["swiglu_bwd"] + (
        ["gemm_rs NN"] if "x" in grads else []) + (
        ["ag_wgrad" + (" +wg|wu" if "wg" in to_main else "")] if "wg" in grads or "wu" in grads else [])
    assert ext.calls == want
    assert tally == len(want) + ("wd" in grads)
    check_grads(leaves, grads, bases, to_main, ref, f"tp_gated_mlp grads {grads}")
