"""The per-element comparator of tests/dense_ref.py has teeth: it accepts correctly rounded results and rejects each of
the defects a dense kernel typically has.  Also checks that the GPU suite's norm hidden sizes cover every case the norm
kernels dispatch on."""
import os
import re

import pytest
import torch
import torch.nn.functional as F

from tests import dense_ref as R
from tests.test_dense_kernels_gpu import NORM_HIDDEN

NORM_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "libai_b200", "csrc", "norm.cu")


def _data(M, N, K, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g).bfloat16()
    b = torch.randn(N, K, generator=g).bfloat16()
    bias = torch.randn(N, generator=g).bfloat16()
    return a, b, bias


def _exact(a, b, bias=None):
    acc = a.double() @ b.double().t()
    return acc if bias is None else acc + bias.double()


def _rejects(fn):
    with pytest.raises(R.Mismatch):
        fn()


@pytest.mark.parametrize("M,N,K", [(65, 72, 1032), (8, 200, 256), (1, 8, 8)])
def test_correctly_rounded_gemm_is_accepted(M, N, K):
    a, b, bias = _data(M, N, K)
    R.check_gemm(_exact(a, b).bfloat16(), a, b, "bf16")
    R.check_gemm(_exact(a, b).float(), a, b, "fp32")
    for act in R.ACTS:
        v = _exact(a, b, bias)
        y, _ = R.act_ref(v, act)
        R.check_gemm(y.bfloat16(), a, b, f"act {act}", bias=bias, act=act, pre=v.bfloat16())


def test_dropped_k_tail_is_rejected():
    a, b, _ = _data(65, 72, 1032)
    _rejects(lambda: R.check_gemm(_exact(a[:, :1024], b[:, :1024]).bfloat16(), a, b, "8 K columns dropped"))
    a, b, _ = _data(65, 72, 256)
    _rejects(lambda: R.check_gemm(_exact(a[:, :192], b[:, :192]).bfloat16(), a, b, "one 64-wide K tile dropped"))


def test_zeroed_last_row_of_ragged_tile_is_rejected():
    a, b, _ = _data(65, 72, 64)
    out = _exact(a, b).bfloat16()
    out[-1] = 0
    _rejects(lambda: R.check_gemm(out, a, b, "last row zeroed"))


def test_shifted_bias_is_rejected():
    a, b, bias = _data(63, 200, 56)
    out = _exact(a, b, bias.roll(1)).bfloat16()
    _rejects(lambda: R.check_gemm(out, a, b, "bias shifted", bias=bias))


def test_activation_skipped_for_negative_inputs_is_rejected():
    a, b, bias = _data(63, 72, 72)
    v = _exact(a, b, bias)
    for act in (1, 2, 3, 4, 5):
        y, _ = R.act_ref(v, act)
        out = torch.where(v < 0, v, y).bfloat16()
        _rejects(lambda: R.check_gemm(out, a, b, f"act {act} skipped", bias=bias, act=act))


def test_swapped_swiglu_halves_are_rejected():
    g = torch.Generator().manual_seed(1)
    gu = torch.randn(7, 2 * 64, generator=g).bfloat16()
    gate, up = gu[:, :64], gu[:, 64:]
    y, y_b = R.swiglu_ref(gate, up)
    R.check(y.bfloat16(), y, R.ROUND[torch.bfloat16] * y.abs() + y_b, "correct")
    swapped = (F.silu(up.double()) * gate.double()).bfloat16()
    _rejects(lambda: R.check(swapped, y, R.ROUND[torch.bfloat16] * y.abs() + y_b, "halves swapped"))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_norm_without_mean_is_rejected(dtype):
    g = torch.Generator().manual_seed(2)
    x = (torch.randn(9, 200, generator=g) + 0.5).to(dtype)
    gamma = (1 + 0.1 * torch.randn(200, generator=g)).to(dtype)
    beta = (0.1 * torch.randn(200, generator=g)).to(dtype)
    mean, rstd = R.norm_stats(x, False, 1e-5)
    good = ((x.double() - mean) * rstd * gamma.double() + beta.double())
    R.check_norm_fwd(good.to(dtype), mean[:, 0].float(), rstd[:, 0].float(), x, gamma, beta, False, 1e-5, "correct")
    bad = (x.double() * rstd * gamma.double() + beta.double())
    _rejects(lambda: R.check_norm_fwd(bad.to(dtype), mean[:, 0].float(), rstd[:, 0].float(), x, gamma, beta, False,
                                      1e-5, "mean left out"))


def test_nan_is_rejected_and_reported():
    ref = torch.ones(3, 4, dtype=torch.float64)
    out = ref.clone()
    out[2, 1] = float("nan")
    with pytest.raises(R.Mismatch, match=r"worst at \(2, 1\): out=nan"):
        R.check(out, ref, 1.0, "nan")


def _cases(func):
    """VPL values of the LB_CASE list in the body of `func` in norm.cu."""
    src = open(NORM_CU).read()
    body = src[src.index(f"bool {func}("):]
    body = body[body.index("switch (vpl)"):body.index("default:", body.index("switch (vpl)"))]
    return {int(v) for v in re.findall(r"LB_CASE\((\d+)\)", body)}


def test_gpu_norm_sizes_cover_every_dispatch_case():
    fwd, bwd, bwd_bf16 = _cases("fwd_dispatch"), _cases("bwd_dispatch"), _cases("bwd_dispatch_bf16")
    assert fwd and bwd and bwd_bf16 <= bwd
    fast = {h // 256 for h in NORM_HIDDEN if h % 256 == 0}
    assert fwd <= fast, sorted(fwd - fast)
    assert bwd <= fast, sorted(bwd - fast)
    fwd_generic = [h for h in NORM_HIDDEN if h % 256 or h // 256 not in fwd]
    bwd_generic = [h for h in NORM_HIDDEN if h % 256 or h // 256 not in bwd]
    assert len(fwd_generic) >= 2 and len(bwd_generic) >= 2, (fwd_generic, bwd_generic)
