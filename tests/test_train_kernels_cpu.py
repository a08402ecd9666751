"""The per-element references of tests/train_ref.py have teeth: an fp32 emulation of each kernel passes its bound, and
each of the defects these kernels typically have is rejected.  Also: the optimizers remove the fp16 loss scale when
gradient clipping is off, and the tile-width mirror used to pick the GPU file's fp8 GEMM shapes matches gemm_sm90.cu."""
import os
import re

import pytest
import torch

from libai_b200.optim import LAMB, SGD, Adam, AdamW
from tests import train_ref as T
from tests.dense_ref import Mismatch
from tests.test_train_kernels_gpu import FP8_HEURISTIC_SHAPES

GEMM_CU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "libai_b200", "csrc", "gemm_sm90.cu")


def _rejects(fn, exc=(Mismatch, AssertionError)):
    with pytest.raises(exc):
        fn()


# ------------------------------------------------------------------------------------------------------------ Adam
def adam_fp32(master, grad, m, v, scale, hp, decoupled, defect=None):
    """fp32 emulation of one adamw_kernel step (correctly rounded division and root), with an optional planted defect."""
    f = lambda x: torch.tensor(x, dtype=torch.float32)
    lr, b1, b2, eps, wd, bc1, bc2 = (f(hp[k]) for k in ("lr", "b1", "b2", "eps", "wd", "bc1", "bc2"))
    if defect == "no bias correction":
        bc1 = bc2 = f(1.0)
    coupled = (defect == "decay swapped") == decoupled
    g = grad if defect == "scale after moments" else grad * f(scale)
    if coupled:
        g = g + wd * master
    m2 = b1 * m + (1 - b1) * g
    v2 = b2 * v + (1 - b2) * g * g
    den = torch.sqrt(v2 / bc2 + eps) if defect == "eps inside sqrt" else torch.sqrt(v2 / bc2) + eps
    upd = (m2 / bc1) / den
    if not coupled:
        upd = upd + wd * master
    if defect == "scale after moments":
        upd = upd * f(scale)
    return master - lr * upd, m2, v2


def _adam_state(n=1000, seed=0, gscale=1e-3):
    g = torch.Generator().manual_seed(seed)
    master = torch.randn(n, generator=g)
    grad = torch.randn(n, generator=g) * gscale
    m = torch.randn(n, generator=g) * gscale * 0.1
    v = torch.rand(n, generator=g) * gscale ** 2 * 0.1
    return master, grad, m, v


@pytest.mark.parametrize("decoupled", [True, False])
@pytest.mark.parametrize("step", [1, 2, 1000])
@pytest.mark.parametrize("scale", [1.0, 0.37, 1 / 65536])
def test_adam_fp32_emulation_is_accepted(decoupled, step, scale):
    old = _adam_state(gscale=1e-3 / scale)
    hp = T.adam_hparams(1e-2, 0.9, 0.999, 1e-3, 0.1, step)
    new = adam_fp32(*old, scale, hp, decoupled)
    T.check_adam(new, old, T.f32(scale), hp, decoupled, "fp32 emulation", lp=new[0].bfloat16())
    T.check_lp(new[0].half(), new[0], "fp16")


@pytest.mark.parametrize("decoupled", [True, False])
@pytest.mark.parametrize("defect,step", [("no bias correction", 1), ("no bias correction", 2),
                                         ("bias correction one step late", 1), ("bias correction one step late", 2),
                                         ("eps inside sqrt", 1), ("eps inside sqrt", 1000), ("decay swapped", 1),
                                         ("decay swapped", 1000), ("scale after moments", 2)])
def test_adam_defects_are_rejected(decoupled, defect, step):
    old = _adam_state()
    scale = 0.37
    hp = T.adam_hparams(1e-2, 0.9, 0.999, 1e-3, 0.1, step)
    if defect == "bias correction one step late":
        new = adam_fp32(*old, scale, T.adam_hparams(1e-2, 0.9, 0.999, 1e-3, 0.1, step + 1), decoupled)
    else:
        new = adam_fp32(*old, scale, hp, decoupled, defect=defect)
    _rejects(lambda: T.check_adam(new, old, T.f32(scale), hp, decoupled, defect))


def test_truncated_lp_out_is_rejected():
    master = _adam_state()[0]
    trunc = (master.view(torch.int32) & ~0xFFFF).view(torch.float32).bfloat16()
    _rejects(lambda: T.check_lp(trunc, master, "truncated bf16"))
    T.check_lp(master.bfloat16(), master, "rounded bf16")


# ------------------------------------------------------------------------------------------------------- embedding
def embedding_bwd_defect(ids, gy, grad, vocab_start, defect):
    """Sequential (per-token) fp32 emulation with a planted defect."""
    out = grad.clone()
    rows = grad.shape[0]
    flat = ids.reshape(-1).tolist()
    runs = {}
    for t, i in enumerate(flat):
        runs.setdefault(i, []).append(t)
    for i, toks in sorted(runs.items()):
        r = i - vocab_start
        if defect == "vocab_start off by one":
            r = i - vocab_start - 1
        if defect == "last token of a run dropped" and len(toks) > 1:
            toks = toks[:-1]
        if not 0 <= r < rows:
            continue
        acc = torch.zeros(grad.shape[1])
        for t in toks:
            acc = acc + gy[t].float()
        out[r] = out[r] + acc
    return out


def _emb_data(T_=200, H=16, rows=50, start=20, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(-5, rows + 2 * start, (T_,), generator=g)
    ids[:9] = start + 3                                     # a run of equal ids
    gy = torch.randn(T_, H, generator=g).bfloat16()
    grad = torch.randn(rows, H, generator=g)
    return ids, gy, grad, start


def test_embedding_bwd_emulation_matches_sequential_sum():
    ids, gy, grad, start = _emb_data()
    T.check_bits(T.embedding_bwd_ref(ids, gy, grad, start), embedding_bwd_defect(ids, gy, grad, start, None), "emulation")


@pytest.mark.parametrize("defect", ["last token of a run dropped", "vocab_start off by one"])
def test_embedding_bwd_defects_are_rejected(defect):
    ids, gy, grad, start = _emb_data()
    bad = embedding_bwd_defect(ids, gy, grad, start, defect)
    _rejects(lambda: T.check_bits(bad, T.embedding_bwd_ref(ids, gy, grad, start), defect))


def test_embedding_fwd_defects_are_rejected():
    ids, _, _, start = _emb_data()
    table = torch.randn(50, 16).bfloat16()
    ref = T.embedding_fwd_ref(ids, table, start)
    local = ids - start
    inside = (local >= 0) & (local < 50)
    assert bool((ref[~inside] == 0).all()) and torch.equal(ref[inside], table[local[inside]])
    shifted = T.embedding_fwd_ref(ids, table, start + 1)
    _rejects(lambda: T.check_bits(shifted, ref, "vocab_start off by one"))
    row0 = table[torch.where(inside, local, torch.zeros_like(local))]          # out-of-shard ids gathered from row 0
    _rejects(lambda: T.check_bits(row0, ref, "out-of-shard ids from row 0"))


# ------------------------------------------------------------------------------------------------------ quantiser
def quant_fp32(x, defect=None):
    """fp32 emulation of quantize_e4m3 (saturating RNE cast), with an optional planted defect."""
    xf = x.float().reshape(-1)
    body = xf[: xf.numel() // 8 * 8] if defect == "amax without the tail" else xf
    amax = torch.clamp(body.abs().max(), min=T.f32(1e-12))
    scale = torch.tensor(448.0) / amax
    y = xf * scale
    if defect == "truncated":
        q = torch.sign(y).double() * _e4m3_floor(y.abs().double().clamp(max=448))
    elif defect == "saturating to NaN":
        q = T.e4m3(y.double().clamp(-448, 448))
        q[y.abs().double() >= 448] = float("nan")
    else:
        q = T.e4m3(y.double().clamp(-448, 448))
    return q, (amax / 448.0).reshape(1)


def _e4m3_floor(a):
    """Largest E4M3 value <= a (a >= 0, <= 448): truncation."""
    grid = torch.arange(0, 127, dtype=torch.uint8).view(torch.float8_e4m3fn).double()      # every finite non-negative
    idx = torch.searchsorted(grid, a, right=True) - 1
    return grid[idx.clamp(min=0)]


@pytest.mark.parametrize("n", [1, 7, 8, 1003])
def test_quant_fp32_emulation_is_accepted(n):
    x = (torch.randn(n, generator=torch.Generator().manual_seed(n)) * 3).bfloat16()
    q, deq = quant_fp32(x)
    T.check_quant(q, deq, x, f"n {n}")


def test_quant_defects_are_rejected():
    x = (torch.randn(1003, generator=torch.Generator().manual_seed(0)) * 3).bfloat16()
    x[-1] = 50.0                                            # the maximum sits in the n % 8 tail
    for defect in ("amax without the tail", "truncated", "saturating to NaN"):
        q, deq = quant_fp32(x, defect)
        _rejects(lambda: T.check_quant(q, deq, x, defect))


def test_quant_reference_flushes_subnormals_and_floors_amax():
    x = torch.tensor([1e-39, -2e-39, 0.0, -0.0, 3e-39, 0.0, 0.0, 0.0, 1e-39]).bfloat16()
    assert bool((x.float().abs() < 2.0 ** -126).all())
    amax, deq, _, q_lo, q_hi = T.quant_ref(x)
    assert amax == 0.0 and deq == T.f32(1e-12) / 448 and bool((q_lo == 0).all()) and bool((q_hi == 0).all())


# ------------------------------------------------------------------------------------------------------- fp8 GEMM
def _fp8_data(M, N, K, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g).bfloat16()
    w = (torch.randn(N, K, generator=g) * 0.05).bfloat16()
    xq, dx = quant_fp32(x)
    wq, dw = quant_fp32(w)
    bias = torch.randn(N, generator=g).bfloat16()
    return xq.reshape(M, K), wq.reshape(N, K), dx, dw, bias


def _fp8_out(xq, wq, alpha, bias=None, bias_first=False, k=None):
    k = xq.shape[1] if k is None else k
    acc = xq[:, :k].double() @ wq[:, :k].double().t()
    if bias is None:
        return (acc * alpha).bfloat16()
    if bias_first:
        return ((acc + bias.double()) * alpha).bfloat16()
    return (acc * alpha + bias.double()).bfloat16()


@pytest.mark.parametrize("M,N,K", [(63, 72, 1040), (1, 8, 48), (65, 200, 4096)])
def test_fp8_gemm_emulation_is_accepted(M, N, K):
    xq, wq, dx, dw, bias = _fp8_data(M, N, K)
    alpha = T.fp8_alpha(dx, dw)
    T.check_fp8_gemm(_fp8_out(xq, wq, alpha), xq, wq, dx, dw, "plain")
    T.check_fp8_gemm(_fp8_out(xq, wq, alpha, bias), xq, wq, dx, dw, "bias", bias=bias)


@pytest.mark.parametrize("M,N,K", [(63, 72, 1040), (65, 200, 4096)])
def test_fp8_gemm_defects_are_rejected(M, N, K):
    xq, wq, dx, dw, bias = _fp8_data(M, N, K)
    alpha = T.fp8_alpha(dx, dw)
    _rejects(lambda: T.check_fp8_gemm(_fp8_out(xq, wq, float(dx)), xq, wq, dx, dw, "deq_w missing"))
    _rejects(lambda: T.check_fp8_gemm(_fp8_out(xq, wq, float(dw)), xq, wq, dx, dw, "deq_x missing"))
    _rejects(lambda: T.check_fp8_gemm(_fp8_out(xq, wq, alpha, k=K - 16), xq, wq, dx, dw, "last 16 K missing"))
    _rejects(lambda: T.check_fp8_gemm(_fp8_out(xq, wq, alpha, bias, bias_first=True), xq, wq, dx, dw,
                                      "bias before dequantisation", bias=bias))


# -------------------------------------------------------------------------------------------- loss scale, no clip
@pytest.mark.parametrize("opt_cls,kw", [(SGD, dict(lr=0.1, momentum=0.9)), (AdamW, dict(lr=0.1, eps=1e-3)),
                                        (Adam, dict(lr=0.1, eps=1e-3, weight_decay=0.1)),
                                        (LAMB, dict(lr=0.1, eps=1e-3, weight_decay=0.1))])
def test_loss_scale_is_removed_without_clipping(opt_cls, kw):
    """grad_scale = 1/1024 (what DynamicLossScaler sets) on gradients of loss * 1024 must step exactly like the same
    optimizer on unscaled gradients: both factors are powers of two."""
    torch.manual_seed(0)
    a, b = torch.nn.Linear(4, 2), torch.nn.Linear(4, 2)
    b.load_state_dict(a.state_dict())
    oa, ob = opt_cls(list(a.parameters()), **kw), opt_cls(list(b.parameters()), **kw)
    oa.grad_scale = 1.0 / 1024
    for _ in range(3):
        x = torch.randn(8, 4)
        for model, opt, s in ((a, oa, 1024.0), (b, ob, 1.0)):
            opt.zero_grad()
            (model(x).square().mean() * s).backward()
            opt.step()
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert torch.equal(pa, pb), (opt_cls.__name__, (pa - pb).abs().max())


# ---------------------------------------------------------------------------------------------- tile-width mirror
def test_tile_width_mirror_matches_the_source():
    src = open(GEMM_CU).read()
    start = src.index("  if (bn == 0) {\n    double best")
    body = src[start:src.index("const int n_blocks", start)]
    assert re.search(r"cands\[4\] = \{256, 192, 128, 64\}", body)
    assert "if (c > 64 && N <= c / 2) continue;" in body
    per_col = re.search(r"per_col = c == 256 \? ([\d.]+) : \(c == 192 \? ([\d.]+) : \(c == 128 \? ([\d.]+) : ([\d.]+)\)\)",
                        body)
    assert per_col and tuple(float(v) for v in per_col.groups()) == tuple(T.TILE_PER_COL[c] for c in T.TILE_CANDS)
    epi = re.search(r"epi != 0 \? [\d.]+ : \(c == 256 \? ([\d.]+) : \(c == 192 \? ([\d.]+) : \(c == 128 \? ([\d.]+) : "
                    r"([\d.]+)\)\)\)", body)
    assert epi and tuple(float(v) for v in epi.groups()) == tuple(T.TILE_EPILOGUE_BF16[c] for c in T.TILE_CANDS)
    assert re.search(r"waves \* \(c \* k_blocks \* per_col \+ epilogue\)", body)
    assert "constexpr int BLOCK_M = 128;" in src and "constexpr int BLOCK_K = 64;" in src
    # the fp8 entry hands the kernel K / 2 bf16 columns
    assert re.search(r"gemm_impl\(xq, wq, out, M, N, K / 2,", src)


def test_gpu_fp8_shapes_reach_every_tile_width_on_the_heuristic_path():
    widths = {T.pick_bn(M, N, K, fp8=True) for M, N, K in FP8_HEURISTIC_SHAPES}
    assert widths == {64, 128, 192, 256}, widths
