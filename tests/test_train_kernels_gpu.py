"""The fused Adam / AdamW update, the embedding kernels, the E4M3 quantiser and the fp8 forward GEMM on the H100 against
the per-element references of tests/train_ref.py, which states the bounds.  The embedding kernels are checked bit for
bit; the Adam update's low-precision copy must be exactly the round-to-nearest-even of its own new master."""
import math

import pytest
import torch

from libai_b200.optim import Adam, AdamW
from tests import dense_ref as R
from tests import train_ref as T

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# (M, N, K) of fp8 forward GEMMs on the heuristic path: GPT-2 345M's QKV, fc1 and fc2 at 8 x 1024 tokens (tile widths
# 64, 64, 128), then the smallest found shapes where the heuristic takes 192 and 256 (tests/test_train_kernels_cpu.py
# checks this against a mirror of the heuristic)
FP8_HEURISTIC_SHAPES = [(8192, 3072, 1024), (8192, 4096, 1024), (8192, 1024, 4096), (256, 8704, 8192),
                        (256, 12800, 49152)]


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


def sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def rand(*shape, seed, dtype=torch.bfloat16, scale=1.0):
    return (torch.randn(*shape, device=DEV, generator=gen(seed)) * scale).to(dtype)


# ---------------------------------------------------------------------------------------------------- fused_adamw
def adam_inputs(n, seed, scale):
    """fp32 master, grad, m, v; the gradient (after ``scale``) holds zeros, values whose square is near the fp32
    overflow (|g| = 1e19, g^2 = 1e38) or below the smallest normal (|g| = 1e-20), and values of both signs."""
    master = rand(n, seed=seed, dtype=torch.float32)
    g = rand(n, seed=seed + 1, dtype=torch.float32, scale=1e-2)
    special = torch.tensor([0.0, 1e19, -1e19, 1e-20, -1e-20, 3e18, 0.0, -0.0], device=DEV)
    k = min(n, special.numel())
    g[:k] = special[:k]
    if n > 64:
        g[n // 2:n // 2 + k] = special[:k]
    grad = (g.double() / scale).float()
    m = rand(n, seed=seed + 2, dtype=torch.float32, scale=1e-3)
    v = rand(n, seed=seed + 3, dtype=torch.float32, scale=1e-3).square()
    return master, grad, m, v


def adam_sizes():
    return [4, 1000, sms() * 8 * 256 * 4 + 1028]     # the last is past the grid cap (every thread loops)


@pytest.mark.parametrize("lp_dtype", [None, torch.bfloat16, torch.float16], ids=["no_lp", "bf16", "fp16"])
@pytest.mark.parametrize("wd", [0.0, 0.1])
@pytest.mark.parametrize("scale", [1.0, 0.37, 2.0 ** -16])
@pytest.mark.parametrize("decoupled", [True, False])
def test_fused_adamw_per_element(ext, decoupled, scale, wd, lp_dtype):
    for n in adam_sizes():
        master, grad, m, v = adam_inputs(n, seed=n, scale=scale)
        lp = None if lp_dtype is None else torch.empty(n, dtype=lp_dtype, device=DEV)
        scale_t = torch.tensor([scale], dtype=torch.float32, device=DEV)
        for step in (1, 2, 1000):
            hp = T.adam_hparams(1e-2, 0.9, 0.999, 1e-8, wd, step)
            old = tuple(t.clone() for t in (master, grad, m, v))
            ext.fused_adamw(master, grad, m, v, lp, scale_t, 1e-2, 0.9, 0.999, 1e-8, wd, 1 - 0.9 ** step,
                            1 - 0.999 ** step, decoupled)
            T.check_adam((master, m, v), old, T.f32(scale), hp, decoupled, f"n {n} step {step}", lp=lp)
            # the next step starts from the kernel's own state, with a fresh gradient
            grad = adam_inputs(n, seed=n + step, scale=scale)[1]


def test_fused_adamw_run_to_run_identical(ext):
    n = 1 << 20
    outs = []
    for _ in range(2):
        master, grad, m, v = adam_inputs(n, seed=5, scale=1.0)
        lp = torch.empty(n, dtype=torch.bfloat16, device=DEV)
        ext.fused_adamw(master, grad, m, v, lp, torch.ones(1, device=DEV), 1e-3, 0.9, 0.999, 1e-8, 0.01, 0.1, 0.001,
                        True)
        outs.append((master, m, v, lp))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def _groups(dtype):
    """Two parameter groups whose sizes are not multiples of 8, on the GPU in ``dtype``."""
    torch.manual_seed(0)
    shapes = [[(7, 3), (13,), (1,)], [(5, 11), (9,)]]
    return [[torch.nn.Parameter((torch.randn(s) * 0.5).to(DEV, dtype)) for s in g] for g in shapes]


@pytest.mark.parametrize("loss_scale", [1.0, 1024.0])
@pytest.mark.parametrize("clip", [None, 0.05])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "fp16", "fp32"])
@pytest.mark.parametrize("opt_cls", [AdamW, Adam])
def test_optimizer_steps_per_element(opt_cls, dtype, clip, loss_scale):
    groups = _groups(dtype)
    pg = []
    for gi, ps in enumerate(groups):
        d = {"params": ps, "weight_decay": 0.1 * gi}
        if clip is not None:
            d.update(clip_grad_max_norm=clip, clip_grad_norm_type=2.0)
        pg.append(d)
    opt = opt_cls(pg, lr=1e-2, eps=1e-6)
    opt.setup()
    opt.grad_scale = 1.0 / loss_scale
    for step in range(1, 4):
        opt.zero_grad()
        for ps in groups:
            for p in ps:
                p.grad = (torch.randn(p.shape, device=DEV) * loss_scale).to(dtype)
        opt.sync_gradients()
        opt.clip_grad()
        coef = opt._clip_coef
        scale = T.f32(float((coef * opt.grad_scale).float())) if coef is not None else T.f32(opt.grad_scale)
        before = []
        for fg in opt._groups:
            before.append(tuple(t.clone() for t in (fg.master_view(), fg.grad_shard(), fg.state["exp_avg"],
                                                    fg.state["exp_avg_sq"])))
        opt.step()
        for gi, (fg, old) in enumerate(zip(opt._groups, before)):
            hp = T.adam_hparams(1e-2, 0.9, 0.999, 1e-6, 0.1 * gi, step)
            new = (fg.master_view(), fg.state["exp_avg"], fg.state["exp_avg_sq"])
            lp = fg.lp_shard() if fg.master is not None else None
            T.check_adam(new, old, scale, hp, opt_cls.decoupled, f"{opt_cls.__name__} {dtype} group {gi} step {step}",
                         lp=lp)


def test_fused_adamw_rejects_bad_arguments(ext):
    n = 1000
    master, grad, m, v = adam_inputs(n, seed=1, scale=1.0)
    one = torch.ones(1, device=DEV)
    args = (1e-3, 0.9, 0.999, 1e-8, 0.0, 0.1, 0.001, True)
    bad = [
        (master, grad, m[:996], v, None, one),                                    # short m
        (master, grad.double(), m, v, None, one),                                 # fp64 grad
        (master, grad, m, v.cpu(), None, one),                                    # v on the host
        (master, grad, m, torch.empty(2 * n, device=DEV)[1:n + 1], None, one),    # misaligned v
        (master, grad, m, v, torch.empty(n, dtype=torch.float32, device=DEV), one),   # fp32 lp_out
        (master, grad, m, v, torch.empty(996, dtype=torch.bfloat16, device=DEV), one),  # short lp_out
        (master, grad, m, v, torch.empty(n + 1, dtype=torch.bfloat16, device=DEV)[1:], one),  # misaligned lp_out
        (master, grad, m, v, None, torch.ones(2, device=DEV)),                     # two-element scale
        (master, grad, m, v, None, torch.ones(1)),                                # host scale
    ]
    for b in bad:
        with pytest.raises(RuntimeError, match="fused_adamw"):
            ext.fused_adamw(*b, *args)


# ------------------------------------------------------------------------------------------------------- embedding
def emb_ids(T_, V, seed, kind="random"):
    if kind == "distinct":
        return torch.randperm(V, device=DEV, generator=gen(seed))[:T_]
    if kind == "pad":
        return torch.full((T_,), 7, dtype=torch.long, device=DEV)
    ids = torch.randint(-3, V + 3, (T_,), device=DEV, generator=gen(seed))      # negative and past-the-end ids too
    ids[: min(T_, 40)] = 11                                                       # a run of equal ids
    return ids


@pytest.mark.parametrize("T_", [1, 1000, 16384])
@pytest.mark.parametrize("H", [8, 136, 1024, 4096])
def test_embedding_per_element(ext, H, T_):
    V = 5000 if H < 4096 else 2000
    table = rand(V, H, seed=1)
    ids = emb_ids(T_, V, seed=H + T_)
    what = f"H {H} T {T_}"
    for start in (0, 1234):
        T.check_bits(ext.embedding_fwd(ids, table, start), T.embedding_fwd_ref(ids, table, start), what + " fwd")
    gy = rand(T_, H, seed=3)
    base = rand(V, H, seed=4, dtype=torch.float32)
    grad = base.clone()
    ext.embedding_bwd(ids, gy, grad, 0)
    T.check_bits(grad, T.embedding_bwd_ref(ids, gy, base, 0), what + " bwd")
    again = base.clone()
    ext.embedding_bwd(ids, gy, again, 0)
    assert torch.equal(again, grad), "embedding_bwd not bit-identical run to run"
    # two vocabulary shards: their gradients, concatenated, are the unsharded gradient exactly
    half = V // 2
    shards = []
    for lo, hi in ((0, half), (half, V)):
        g = base[lo:hi].clone()
        ext.embedding_bwd(ids, gy, g, lo)
        T.check_bits(g, T.embedding_bwd_ref(ids, gy, base[lo:hi], lo), what + f" shard at {lo}")
        shards.append(g)
    T.check_bits(torch.cat(shards), grad, what + " shards vs unsharded")


@pytest.mark.parametrize("kind", ["pad", "distinct"])
def test_embedding_bwd_pad_token_and_distinct_ids(ext, kind):
    V, H = 20000, 1024
    T_ = 16384
    ids = emb_ids(T_, V, seed=9, kind=kind)
    gy = rand(T_, H, seed=5)
    base = rand(V, H, seed=6, dtype=torch.float32)
    grad = base.clone()
    ext.embedding_bwd(ids, gy, grad, 0)
    T.check_bits(grad, T.embedding_bwd_ref(ids, gy, base, 0), kind)


def test_embedding_main_grad_and_grad_return_paths():
    from libai_b200.ops import functional as OFn

    V, H = 3000, 136
    ids = emb_ids(2 * 500, V, seed=2).view(2, 500)
    table = torch.nn.Parameter(rand(V, H, seed=1))
    base = rand(V, H, seed=7, dtype=torch.float32)
    table.main_grad = base.clone()
    out = OFn.embedding(ids, table, 100)
    T.check_bits(out.reshape(-1, H), T.embedding_fwd_ref(ids, table.detach(), 100), "functional fwd")
    gy = rand(2, 500, H, seed=8)
    out.backward(gy)
    assert table.grad is None
    T.check_bits(table.main_grad, T.embedding_bwd_ref(ids, gy.reshape(-1, H), base, 100), "main_grad path")
    t2 = torch.nn.Parameter(table.detach().clone())
    OFn.embedding(ids, t2, 100).backward(gy)
    want = T.embedding_bwd_ref(ids, gy.reshape(-1, H), torch.zeros(V, H, device=DEV), 100).bfloat16()
    T.check_bits(t2.grad, want, "grad return path")


def test_embedding_bwd_rejects_arguments_on_different_devices(ext):
    ids = torch.randint(0, 100, (64,))
    gy = rand(64, 16, seed=1)
    grad = torch.zeros(100, 16, device=DEV)
    with pytest.raises(RuntimeError, match="embedding_bwd"):
        ext.embedding_bwd(ids, gy, grad, 0)                          # host ids
    with pytest.raises(RuntimeError, match="embedding_bwd"):
        ext.embedding_bwd(ids.to(DEV), gy, grad.cpu(), 0)            # host grad


# ------------------------------------------------------------------------------------------------------ quantiser
def quant_sizes():
    return [1, 7, 8, 1003, sms() * 8 * 256 * 8 + 13]                 # the last is past the 8-blocks-per-SM cap


def quant(ext, x):
    """quantize_e4m3 twice: the results must be bit-identical."""
    (q, d), (q2, d2) = ext.quantize_e4m3(x), ext.quantize_e4m3(x)
    assert torch.equal(q.view(torch.uint8), q2.view(torch.uint8)) and torch.equal(d, d2), "not bit-identical"
    return q, d


@pytest.mark.parametrize("i", range(5))
def test_quantize_per_element(ext, i):
    n = quant_sizes()[i]
    x = rand(n, seed=n, scale=3.0)
    q, d = quant(ext, x)
    T.check_quant(q, d, x, f"n {n}")


def test_quantize_zero_tensor_signed_zeros_and_subnormals(ext):
    z = torch.zeros(1003, dtype=torch.bfloat16, device=DEV)
    q, d = quant(ext, z)
    assert bool((q.float() == 0).all()) and math.isfinite(float(d)) and float(d) > 0
    T.check_quant(q, d, z, "all zero")
    x = rand(1003, seed=1)
    x[::5] = 0.0
    x[1::5] = -0.0
    q, d = quant(ext, x)
    T.check_quant(q, d, x, "±0")
    sub = torch.tensor([1e-39, -2e-39, 5e-40, -1e-40] * 25, dtype=torch.bfloat16, device=DEV)
    assert bool((sub.float().abs() < 2.0 ** -126).all()) and bool((sub != 0).all())
    q, d = quant(ext, sub)
    T.check_quant(q, d, sub, "all subnormal")      # read as zero: q = 0
    mixed = rand(1003, seed=2)
    mixed[::3] = sub[0]
    q, d = quant(ext, mixed)
    T.check_quant(q, d, mixed, "subnormals among normals")


def test_quantize_single_huge_element(ext):
    for big in (3.0e38, -2.0 ** 127, 2.0 ** 126 * 1.5, 1e30):
        x = rand(1003, seed=3)
        x[517] = big
        q, d = quant(ext, x)
        T.check_quant(q, d, x, f"huge element {big:g}")


def test_quantize_amax_ignores_nan(ext):
    """fmaxf ignores NaN: the scale comes from the finite elements."""
    x = rand(1003, seed=4, scale=2.0)
    x[100] = float("nan")
    x[1001] = float("nan")                          # in the n % 8 tail
    q, d = ext.quantize_e4m3(x)
    finite = torch.nan_to_num(x.float(), nan=0.0)
    _, deq_ref, deq_b, q_lo, q_hi = T.quant_ref(finite)
    R.check(d, torch.tensor([deq_ref]), deq_b, "deq with NaN inputs")
    keep = ~torch.isnan(x.float())
    R.check(q.double()[keep], ((q_lo + q_hi) / 2)[keep], ((q_hi - q_lo) / 2)[keep], "q with NaN inputs")


# ------------------------------------------------------------------------------------------------------- fp8 GEMM
FP8_TILE_SHAPES = [(1, 8, 16), (63, 72, 48), (65, 200, 1040), (1000, 264, 4096), (1000, 8, 1040), (65, 264, 16),
                   (63, 200, 4096)]


def fp8_operands(M, N, K, seed, wscale=0.05):
    x = rand(M, K, seed=seed)
    w = rand(N, K, seed=seed + 1, scale=wscale)
    return x, w


@pytest.mark.parametrize("bn", [64, 128, 192, 256])
def test_fp8_gemm_every_tile_width(ext, bn):
    for i, (M, N, K) in enumerate(FP8_TILE_SHAPES):
        x, w = fp8_operands(M, N, K, seed=i)
        (xq, dx), (wq, dw) = ext.quantize_e4m3(x), ext.quantize_e4m3(w)
        y, _ = ext.linear_fp8_fwd(xq, wq, dx, dw, None, 0, False, None, bn)
        T.check_fp8_gemm(y, xq, wq, dx, dw, f"bn {bn} {M}x{N}x{K}")


@pytest.mark.parametrize("act", list(R.ACTS))
def test_fp8_gemm_epilogues(ext, act):
    for i, (M, N, K) in enumerate([(1000, 264, 1040), (63, 72, 48), (1, 200, 4096)]):
        x, w = fp8_operands(M, N, K, seed=10 + i, wscale=0.3)
        bias = rand(N, seed=20 + i)
        (xq, dx), (wq, dw) = ext.quantize_e4m3(x), ext.quantize_e4m3(w)
        for bn in (0, 64, 256):
            y, pre = ext.linear_fp8_fwd(xq, wq, dx, dw, bias, act, True, None, bn)
            T.check_fp8_gemm(y, xq, wq, dx, dw, f"act {act} bn {bn} {M}x{N}x{K}", bias=bias, act=act, pre=pre)
            y, _ = ext.linear_fp8_fwd(xq, wq, dx, dw, None, act, False, None, bn)
            T.check_fp8_gemm(y, xq, wq, dx, dw, f"act {act} bn {bn} {M}x{N}x{K} no bias", act=act)


def test_fp8_gemm_bias_and_residual(ext):
    for i, (M, N, K) in enumerate([(1000, 264, 1040), (65, 8, 4096), (1, 72, 16)]):
        x, w = fp8_operands(M, N, K, seed=30 + i)
        bias, res = rand(N, seed=40 + i), rand(M, N, seed=50 + i, scale=8.0)
        (xq, dx), (wq, dw) = ext.quantize_e4m3(x), ext.quantize_e4m3(w)
        for bn in (0, 128, 192):
            y, _ = ext.linear_fp8_fwd(xq, wq, dx, dw, bias, 0, False, res, bn)
            T.check_fp8_gemm(y, xq, wq, dx, dw, f"bias+residual bn {bn}", bias=bias, residual=res)
            y, _ = ext.linear_fp8_fwd(xq, wq, dx, dw, None, 0, False, res, bn)
            T.check_fp8_gemm(y, xq, wq, dx, dw, f"residual bn {bn}", residual=res)


def test_fp8_gemm_residual_refuses_activation_and_pre(ext):
    """A residual epilogue has no activation and no pre-activation copy: asking for either is refused (the
    pre-activation tensor used to come back unwritten)."""
    x, w = fp8_operands(65, 72, 48, seed=1)
    (xq, dx), (wq, dw) = ext.quantize_e4m3(x), ext.quantize_e4m3(w)
    res = rand(65, 72, seed=2)
    with pytest.raises(RuntimeError, match="residual"):
        ext.linear_fp8_fwd(xq, wq, dx, dw, None, 0, True, res)
    with pytest.raises(RuntimeError, match="residual"):
        ext.linear_fp8_fwd(xq, wq, dx, dw, None, 1, False, res)


def test_fp8_gemm_zero_input(ext):
    """amax = 0: q = 0 and a finite deq, so the output is act(bias) exactly."""
    M, N, K = 63, 200, 1040
    x = torch.zeros(M, K, dtype=torch.bfloat16, device=DEV)
    w = rand(N, K, seed=3)
    bias = rand(N, seed=4)
    (xq, dx), (wq, dw) = ext.quantize_e4m3(x), ext.quantize_e4m3(w)
    for act in R.ACTS:
        y, pre = ext.linear_fp8_fwd(xq, wq, dx, dw, bias, act, True, None)
        T.check_fp8_gemm(y, xq, wq, dx, dw, f"zero input act {act}", bias=bias, act=act, pre=pre)
        assert torch.equal(pre, bias.expand(M, N))


@pytest.mark.parametrize("shape", FP8_HEURISTIC_SHAPES)
def test_fp8_gemm_heuristic_path(ext, shape):
    """The default tile width at model shapes; every row and the first and last 264 columns are checked."""
    M, N, K = shape
    x, w = fp8_operands(M, N, K, seed=M + N, wscale=0.02)
    (xq, dx), (wq, dw) = ext.quantize_e4m3(x), ext.quantize_e4m3(w)
    y, _ = ext.linear_fp8_fwd(xq, wq, dx, dw, None, 0, False, None)
    y2, _ = ext.linear_fp8_fwd(xq, wq, dx, dw, None, 0, False, None)
    assert torch.equal(y, y2), "not bit-identical run to run"
    for cols in (slice(0, 264), slice(N - 264, N)):
        T.check_fp8_gemm(y[:, cols].contiguous(), xq, wq[cols], dx, dw, f"{M}x{N}x{K} columns {cols}")


# ------------------------------------------------------------------------------------------------ fp8 weight cache
def _fp8_linear_step(graph):
    """A native linear layer with the fp8 forward on, an AdamW step, then the next forward: it must use
    quantize_e4m3 of the new weight bit for bit (eagerly, and inside a CUDA-graph capture)."""
    from libai_b200 import ops
    from libai_b200.ops import functional as OFn

    ext = ops.load_ext(required=True)
    torch.manual_seed(0)
    w = torch.nn.Parameter((torch.randn(264, 1040) * 0.05).to(DEV, torch.bfloat16))
    x = rand(128, 1040, seed=1)
    opt = AdamW([{"params": [w]}], lr=1e-2)
    opt.setup()
    prev = ops.fp8_enabled()
    ops.set_fp8(True)
    try:
        y0 = OFn.linear(x, w, None)
        y0.float().square().mean().backward()
        opt.step()
        if graph:
            static = {}
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                OFn.linear(x, w, None)                      # warm-up outside the capture
            torch.cuda.current_stream().wait_stream(s)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                static["y"] = OFn.linear(x, w, None)
            opt.step()                                      # rewrites w after the capture: the replay must see it
            g.replay()
            torch.cuda.synchronize()
            y1 = static["y"]
        else:
            y1 = OFn.linear(x, w, None)
    finally:
        ops.set_fp8(prev)
    (xq, dx), (wq, dw) = ext.quantize_e4m3(x), ext.quantize_e4m3(w.detach())
    want, _ = ext.linear_fp8_fwd(xq, wq, dx, dw, None, 0, False, None)
    return y1, want


@pytest.mark.parametrize("graph", [False, True])
def test_fp8_weight_cache_follows_the_optimizer(graph):
    y1, want = _fp8_linear_step(graph)
    T.check_bits(y1.reshape(want.shape), want, "forward after optimizer.step()")
