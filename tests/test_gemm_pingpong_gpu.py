"""The ping-pong GEMM schedule (bf16 outputs of the NT forward and NN dgrad GEMMs) on the H100: every element must be
bit-identical to the 288-thread kernel that `gemm_schedule(1)` forces, for every epilogue, ragged M and N, tile counts
below, between and above one and two per SM (odd, so one consumer warpgroup gets one more tile than the other), outputs
inside wider buffers, CUDA-graph replay and repeated runs.  A few GPT-2 medium shapes are also checked per element
against fp64 (tests/dense_ref.py)."""
import contextlib

import pytest
import torch

from tests import dense_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    e = ops.load_ext(required=True)
    assert e.gemm_schedule(0) == 0
    yield e
    e.gemm_schedule(0)


@contextlib.contextmanager
def old_kernel(ext):
    prev = ext.gemm_schedule(1)
    try:
        yield
    finally:
        ext.gemm_schedule(prev)


def rand(*shape, seed, dtype=torch.bfloat16, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, device=DEV, generator=g) * scale).to(dtype)


def same_as_old_kernel(ext, fn, what):
    """fn() with the ping-pong schedule (twice) and with the 288-thread kernel: all results bitwise equal."""
    def as_tuple(r):
        return r if isinstance(r, tuple) else (r,)

    new, again = as_tuple(fn()), as_tuple(fn())
    with old_kernel(ext):
        old = as_tuple(fn())
    for i, (x, y, z) in enumerate(zip(new, again, old)):
        assert torch.equal(x, y), f"{what}: output {i} not bit-identical run to run"
        assert torch.equal(x, z), (f"{what}: output {i} differs from the 288-thread kernel at "
                                   f"{int((x != z).sum())} of {x.numel()} elements")


# (M, N, K): ragged M and N (N % 8 == 0 but not a multiple of 64 / 128) with 128 x 128 tile counts of 1, 16 and 2
# (< 132), 136 (between one and two per SM: the second consumer idles on most SMs), 320 (CTAs of 2 and 3 tiles) and 525
# (odd, about 4 per SM)
SHAPES = [(1, 8, 8), (1000, 200, 1032), (129, 72, 64), (2125, 1024, 1024), (4000, 1160, 192), (2600, 3080, 128)]


@pytest.mark.parametrize("layout", [0, 1], ids=["NT", "NN"])
@pytest.mark.parametrize("bias", [False, True], ids=["plain", "bias"])
def test_gemm_matches_old_kernel(ext, layout, bias):
    for i, (M, N, K) in enumerate(SHAPES):
        a = rand(M, K, seed=i)
        b = rand(N, K, seed=i + 1) if layout == 0 else rand(K, N, seed=i + 1)
        bv = rand(N, seed=i + 2) if bias else None
        same_as_old_kernel(ext, lambda: ext.gemm(a, b, layout, bv, None, False, torch.bfloat16),
                           f"layout {layout} {M}x{N}x{K} bias {bias}")


@pytest.mark.parametrize("layout", [0, 1], ids=["NT", "NN"])
def test_explicit_tile_widths(ext, layout):
    # 128 takes the ping-pong kernel, the other widths the 288-thread kernel: all give the same bits
    M, N, K = 1000, 200, 1032
    a = rand(M, K, seed=1)
    b = rand(N, K, seed=2) if layout == 0 else rand(K, N, seed=2)
    ref = ext.gemm_tuned(a, b, layout, 128, 1, False)
    A, B = R.gemm_operands(a, b, layout)
    R.check_gemm(ref, A, B, f"layout {layout} bn 128")
    for bn in (0, 64, 192, 256):
        assert torch.equal(ext.gemm_tuned(a, b, layout, bn, 1, False), ref), f"bn {bn}"
    with old_kernel(ext):
        assert torch.equal(ext.gemm_tuned(a, b, layout, 128, 1, False), ref)


@pytest.mark.parametrize("act", list(R.ACTS))
def test_linear_fwd_bias_act_pre_matches_old_kernel(ext, act):
    for i, (M, N, K) in enumerate(SHAPES):
        x, w, bias = rand(M, K, seed=i), rand(N, K, seed=i + 1, scale=0.3), rand(N, seed=i + 2)
        same_as_old_kernel(ext, lambda: ext.linear_fwd(x, w, bias, act, True), f"act {act} {M}x{N}x{K} pre")
        same_as_old_kernel(ext, lambda: ext.linear_fwd(x, w, None, act, False)[0], f"act {act} {M}x{N}x{K}")


def test_linear_bias_residual_matches_old_kernel(ext):
    for i, (M, N, K) in enumerate(SHAPES):
        x, w, bias, res = rand(M, K, seed=i), rand(N, K, seed=i + 1), rand(N, seed=i + 2), rand(M, N, seed=i + 3,
                                                                                                  scale=8.0)
        same_as_old_kernel(ext, lambda: ext.linear_bias_residual(x, w, bias, res), f"bias+residual {M}x{N}x{K}")
        same_as_old_kernel(ext, lambda: ext.linear_bias_residual(x, w, None, res), f"residual {M}x{N}x{K}")


@pytest.mark.parametrize("act", list(R.ACTS))
def test_dgrad_actgrad_and_bias_grad_match_old_kernel(ext, act):
    for i, (M, N, K) in enumerate(SHAPES):
        gy, w, pre = rand(M, K, seed=i), rand(K, N, seed=i + 1, scale=0.3), rand(M, N, seed=i + 2, scale=2.0)
        base = rand(N, seed=i + 3, dtype=torch.float32)

        def run():
            bg = base.clone()
            return ext.dgrad_actgrad(gy, w, pre, act, bg), bg

        same_as_old_kernel(ext, run, f"dgrad act {act} {M}x{N}x{K}")


def test_out_inside_wider_buffer_keeps_sentinels(ext):
    for layout in (0, 1):
        for i, (M, N, K) in enumerate(SHAPES[1:]):
            a = rand(M, K, seed=i)
            b = rand(N, K, seed=i + 1) if layout == 0 else rand(K, N, seed=i + 1)
            bias = rand(N, seed=i + 2)

            def run():
                buf = torch.full((M + 3, N + 24), 123.0, device=DEV, dtype=torch.bfloat16)
                view = buf[1:M + 1, 8:8 + N]          # 16 bytes into a row, row stride N + 24
                assert view.data_ptr() % 16 == 0
                ext.gemm(a, b, layout, bias, view, False, torch.bfloat16)
                return buf

            same_as_old_kernel(ext, run, f"wide out layout {layout} {M}x{N}x{K}")
            buf = run()
            keep = torch.ones_like(buf, dtype=torch.bool)
            keep[1:M + 1, 8:8 + N] = False
            assert bool((buf[keep] == 123.0).all()), f"layout {layout} {M}x{N}x{K}: wrote outside the view"
            R.check_gemm(buf[1:M + 1, 8:8 + N], *R.gemm_operands(a, b, layout), f"wide out {M}x{N}x{K}", bias=bias)


def test_cuda_graph_replay(ext):
    M, N, K = 4000, 1160, 192
    x, w, bias = rand(M, K, seed=1), rand(N, K, seed=2, scale=0.3), rand(N, seed=3)
    gy, w2, pre = rand(M, N, seed=4), rand(N, K, seed=5, scale=0.3), rand(M, K, seed=6)
    eager = (*ext.linear_fwd(x, w, bias, 1, True), ext.dgrad_actgrad(gy, w2, pre, 1, None))
    s = torch.cuda.Stream(device=DEV)
    s.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(s):
        ext.linear_fwd(x, w, bias, 1, True)
        ext.dgrad_actgrad(gy, w2, pre, 1, None)
    torch.cuda.current_stream(DEV).wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y, p = ext.linear_fwd(x, w, bias, 1, True)
        d = ext.dgrad_actgrad(gy, w2, pre, 1, None)
    for _ in range(2):
        for t in (y, p, d):
            t.fill_(0)
        g.replay()
        torch.cuda.synchronize()
        for got, want in zip((y, p, d), eager):
            assert torch.equal(got, want)


# GPT-2 medium (8 x 1024 tokens, hidden 1024, ffn 4096) against fp64
def test_gpt2_medium_shapes_against_fp64(ext):
    T, H, F = 8192, 1024, 4096
    x = rand(T, H, seed=1)
    w_fc1, b_fc1 = rand(F, H, seed=2, scale=0.03), rand(F, seed=3, scale=0.1)
    y, pre = ext.linear_fwd(x, w_fc1, b_fc1, 1, True)
    R.check_gemm(y, x, w_fc1, "fc1 forward", bias=b_fc1, act=1, pre=pre)
    w_proj, b_proj, res = rand(H, H, seed=4, scale=0.03), rand(H, seed=5, scale=0.1), rand(T, H, seed=6)
    R.check_gemm(ext.linear_bias_residual(x, w_proj, b_proj, res), x, w_proj, "proj forward", bias=b_proj, residual=res)
    w_fc2, gy = rand(H, F, seed=7, scale=0.03), rand(T, H, seed=8)
    R.check_gemm(ext.dgrad_actgrad(gy, w_fc2, pre, 1, None), gy, w_fc2.t(), "fc2 dgrad", act=1, dpre=pre)
    w_qkv = rand(3 * H, H, seed=9, scale=0.03)
    R.check_gemm(ext.gemm(x, w_qkv, 0, None, None, False, torch.bfloat16), x, w_qkv, "qkv forward")
