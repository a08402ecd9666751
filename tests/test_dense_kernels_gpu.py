"""The dense kernels on the H100 against fp64, element by element (tests/dense_ref.py states the bounds): the GEMM at
every tile width, split-K, the heuristic path at model shapes and every epilogue; LayerNorm / RMSNorm at every
dispatched hidden size and past the grids' row caps; vocab-parallel cross-entropy; the packed SwiGLU; column sums and
the squared norm.  Every default-path call is also run twice and must give identical bits."""
import pytest
import torch
import torch.nn.functional as F

from tests import dense_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# 256 * every VPL the norm kernels dispatch on, then sizes that take the generic kernels (Swin, Qwen2-0.5B, ragged,
# ViT-g, Qwen2-7B); 5120 and 8192 are fast forward, generic backward
NORM_HIDDEN = [256 * v for v in (1, 2, 3, 4, 5, 6, 8, 10, 12, 16, 20, 32)] + [96, 200, 896, 1001, 1408, 3584]


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


def sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def rand(*shape, seed, dtype=torch.bfloat16, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, device=DEV, generator=g) * scale).to(dtype)


def twice(fn):
    """fn() run twice; the results must be bitwise equal."""
    a, b = fn(), fn()
    for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
        assert torch.equal(x, y), "not bit-identical run to run"
    return a


def operands(M, N, K, layout, seed):
    """ext.gemm operands of a layout; a TN left operand [K, M] with M % 8 != 0 is a column slice of a wider buffer
    (TMA needs 16-byte row strides)."""
    if layout == 0:
        return rand(M, K, seed=seed), rand(N, K, seed=seed + 1)
    if layout == 1:
        return rand(M, K, seed=seed), rand(K, N, seed=seed + 1)
    return rand(K, (M + 7) // 8 * 8, seed=seed)[:, :M], rand(K, N, seed=seed + 1)


# ------------------------------------------------------------------------------------------------------------------ GEMM
# ragged shapes, the sizes paired rather than crossed: M in {1, 8, 63, 65, 129, 1000}, N in {8, 72, 200, 264},
# K in {8, 56, 64, 72, 1032}
TILE_SHAPES = [(1, 8, 8), (8, 72, 56), (63, 200, 64), (65, 264, 72), (129, 200, 1032), (1000, 264, 56),
               (1000, 72, 1032), (65, 8, 1032)]


@pytest.mark.parametrize("bn", [64, 128, 192, 256])
@pytest.mark.parametrize("layout", [0, 1, 2])
def test_gemm_every_tile_width(ext, layout, bn):
    for i, (M, N, K) in enumerate(TILE_SHAPES):
        a, b = operands(M, N, K, layout, seed=i)
        A, B = R.gemm_operands(a, b, layout)
        R.check_gemm(ext.gemm_tuned(a, b, layout, bn, 1, False), A, B, f"layout {layout} bn {bn} {M}x{N}x{K} bf16")
        R.check_gemm(ext.gemm_tuned(a, b, layout, bn, 1, True), A, B, f"layout {layout} bn {bn} {M}x{N}x{K} fp32")


@pytest.mark.parametrize("layout", [0, 1, 2])
def test_gemm_split_k(ext, layout):
    for M, N, K in [(129, 200, 1032), (65, 72, 72), (1000, 264, 1032)]:
        a, b = operands(M, N, K, layout, seed=M)
        A, B = R.gemm_operands(a, b, layout)
        k_blocks = (K + 63) // 64
        for splits in (2, 3, k_blocks + 5):
            R.check_gemm(ext.gemm_tuned(a, b, layout, 128, splits, True), A, B,
                         f"layout {layout} {M}x{N}x{K} splits {splits}")


# (N, K) of the qkv, o, packed gate|up and down projections; the LM heads at decode-time M only
MODEL_SHAPES = {
    "llama-7b": [(12288, 4096), (4096, 4096), (22016, 4096), (4096, 11008)],
    "llama-3-8b": [(6144, 4096), (28672, 4096), (4096, 14336)],
    "qwen2-7b": [(4608, 3584), (37888, 3584), (3584, 18944)],
    "qwen2-0.5b": [(1152, 896)],
    "lm-heads": [(32000, 4096), (151936, 896)],
}


@pytest.mark.parametrize("model", list(MODEL_SHAPES))
def test_gemm_heuristic_path_at_model_shapes(ext, model):
    for j, (N, K) in enumerate(MODEL_SHAPES[model]):
        w = rand(N, K, seed=j, scale=0.05)
        for M in ((1, 16) if model == "lm-heads" else (1, 16, 4096)):
            x = rand(M, K, seed=M + j)
            what = f"{model} {M}x{N}x{K}"
            R.check_gemm(twice(lambda: ext.gemm(x, w, 0, None, None, False, torch.bfloat16)), x, w, what + " gemm")
            y, _ = twice(lambda: ext.linear_fwd(x, w, None, 0, False))
            R.check_gemm(y, x, w, what + " linear_fwd")
            if M == 4096:
                gy = rand(M, N, seed=7)
                # dgrad gy[M, N] @ w[N, K] and wgrad gy^T x -> [N, K] in fp32 (fresh and accumulated)
                R.check_gemm(twice(lambda: ext.gemm(gy, w, 1, None, None, False, torch.bfloat16)), gy, w.t(),
                             what + " dgrad")
                R.check_gemm(twice(lambda: ext.gemm(gy, x, 2, None, None, False, torch.float32)), gy.t(), x.t(),
                             what + " wgrad")
                base = rand(N, K, seed=9, dtype=torch.float32)
                acc = twice(lambda: ext.gemm(gy, x, 2, None, base.clone(), True, torch.float32))
                R.check_gemm(acc, gy.t(), x.t(), what + " wgrad accumulate", base=base)


@pytest.mark.parametrize("act", list(R.ACTS))
def test_linear_fwd_bias_act_and_pre(ext, act):
    for M, N, K in [(1000, 264, 72), (65, 200, 1032), (1, 8, 8)]:
        x, w, bias = rand(M, K, seed=1), rand(N, K, seed=2, scale=0.3), rand(N, seed=3)
        y, pre = twice(lambda: ext.linear_fwd(x, w, bias, act, True))
        R.check_gemm(y, x, w, f"act {act} {M}x{N}x{K}", bias=bias, act=act, pre=pre if act else None)
        y, _ = ext.linear_fwd(x, w, None, act, False)
        R.check_gemm(y, x, w, f"act {act} {M}x{N}x{K} no bias", act=act)


def test_linear_bias_residual(ext):
    for M, N, K in [(129, 200, 1032), (1, 72, 64), (1000, 264, 56)]:
        x, w, bias, res = rand(M, K, seed=1), rand(N, K, seed=2), rand(N, seed=3), rand(M, N, seed=4, scale=8.0)
        R.check_gemm(twice(lambda: ext.linear_bias_residual(x, w, bias, res)), x, w, "bias+residual", bias=bias,
                     residual=res)
        R.check_gemm(ext.linear_bias_residual(x, w, None, res), x, w, "residual", residual=res)


@pytest.mark.parametrize("act", list(R.ACTS))
def test_dgrad_actgrad_and_bias_grad(ext, act):
    for M, N, K in [(777, 264, 200), (1, 72, 1032), (4096, 1024, 256)]:
        gy, w, pre = rand(M, K, seed=1), rand(K, N, seed=2, scale=0.3), rand(M, N, seed=3, scale=2.0)
        out = twice(lambda: ext.dgrad_actgrad(gy, w, pre, act, None))
        R.check_gemm(out, gy, w.t(), f"dgrad act {act} {M}x{N}x{K}", act=act, dpre=pre)
        base = rand(N, seed=4, dtype=torch.float32)
        bg = base.clone()
        out2 = ext.dgrad_actgrad(gy, w, pre, act, bg)
        assert torch.equal(out2, out)
        o = out.double()
        ref = base.double() + o.sum(0)
        R.check(bg, ref, R.ROUND[torch.float32] * ref.abs() + (M + 8) * R.ACC * o.abs().sum(0), f"bias_grad act {act}")
        bg2 = base.clone()
        ext.dgrad_actgrad(gy, w, pre, act, bg2)
        assert torch.equal(bg, bg2)


@pytest.mark.parametrize("layout", [0, 1, 2])
def test_gemm_out_overwrites_unless_accumulating(ext, layout):
    M, N, K = 129, 200, 1032
    a, b = operands(M, N, K, layout, seed=5)
    A, B = R.gemm_operands(a, b, layout)
    out = torch.full((M, N), 7.0, device=DEV)
    assert ext.gemm(a, b, layout, None, out, False, torch.float32).data_ptr() == out.data_ptr()
    R.check_gemm(out, A, B, f"layout {layout} out= overwrite")
    base = rand(M, N, seed=6, dtype=torch.float32)
    acc = base.clone()
    ext.gemm(a, b, layout, None, acc, True, torch.float32)
    R.check_gemm(acc, A, B, f"layout {layout} out= accumulate", base=base)
    R.check_gemm(twice(lambda: ext.gemm(a, b, layout, None, None, False, torch.float32)), A, B,
                 f"layout {layout} fp32 out")


def test_linear_fwd_row_strided_input(ext):
    M, N, K = 1000, 264, 72
    buf = rand(M, K + 24, seed=8)
    x = buf[:, 8:8 + K]                      # starts 16 bytes into each row
    assert not x.is_contiguous() and x.data_ptr() % 16 == 0
    w, bias = rand(N, K, seed=9), rand(N, seed=10)
    y, pre = ext.linear_fwd(x, w, bias, 1, True)
    R.check_gemm(y, x, w, "row-strided x", bias=bias, act=1, pre=pre)


# ----------------------------------------------------------------------------------------------------------------- norms
NORM_DTYPES = [(torch.bfloat16, torch.bfloat16), (torch.bfloat16, torch.float32), (torch.float32, torch.float32)]


def norm_rows(H):
    """1, 7, 777 and a count past the forward grid's cap (4 blocks of 8 rows per SM); wide rows stop past the backward
    caps (2 blocks of 8 rows per SM) to keep memory and time down."""
    return [1, 7, 777, 4 * sms() * 8 + 37] if H < 4096 else [1, 7, 2 * sms() * 8 + 5]


@pytest.mark.parametrize("H", NORM_HIDDEN)
@pytest.mark.parametrize("dtypes", NORM_DTYPES, ids=["bf16-bf16", "bf16-fp32", "fp32-fp32"])
@pytest.mark.parametrize("rms", [False, True], ids=["layernorm", "rmsnorm"])
def test_norm_matches_fp64_and_is_deterministic(ext, H, dtypes, rms):
    xdt, wdt = dtypes
    eps = 1e-5
    gamma = (1 + 0.2 * rand(H, seed=1, dtype=torch.float32)).to(wdt)
    beta = None if rms else (0.2 * rand(H, seed=2, dtype=torch.float32)).to(wdt)
    for rows in norm_rows(H):
        what = f"H {H} rows {rows} {'rms' if rms else 'ln'} {xdt}/{wdt}"
        x = (rand(rows, H, seed=rows, dtype=torch.float32) * 2 + 0.5).to(xdt)
        gy = rand(rows, H, seed=rows + 1, dtype=xdt)
        y, mean, rstd = twice(lambda: ext.norm_fwd(x, gamma, beta, eps, rms))
        R.check_norm_fwd(y, mean, rstd, x, gamma, beta, rms, eps, what)
        gx, dg, db = twice(lambda: ext.norm_bwd(gy, x, gamma, mean, rstd, rms, not rms, None, None, None))
        (gx_r, gx_b), (dg_r, dg_b), (db_r, db_b) = R.norm_bwd_ref(gy, x, gamma, rms, eps)
        R.check(gx, gx_r, R.ROUND[xdt] * gx_r.abs() + gx_b + R.FLUSH, what + " gx")
        R.check(dg, dg_r, R.ROUND[torch.float32] * dg_r.abs() + dg_b + R.FLUSH, what + " dgamma")
        if not rms:
            R.check(db, db_r, R.ROUND[torch.float32] * db_r.abs() + db_b + R.FLUSH, what + " dbeta")
        if rows != 777:
            continue
        # dγ / dβ accumulated into slices of an fp32 main-grad buffer, and the skip connection's gradient added to gx
        flat = rand(3 * H, seed=3, dtype=torch.float32)
        base = flat.clone()
        gadd = rand(rows, H, seed=4, dtype=xdt)
        dga, dba = flat[H:2 * H], (None if rms else flat[2 * H:])
        gx2, _, _ = ext.norm_bwd(gy, x, gamma, mean, rstd, rms, not rms, dga, dba, gadd)
        ref = gx_r + gadd.double()
        R.check(gx2, ref, R.ROUND[xdt] * (ref.abs() + gx_r.abs()) + gx_b + R.FLUSH, what + " gx + gadd")
        ref = base[H:2 * H].double() + dg_r
        R.check(dga, ref, R.ROUND[torch.float32] * ref.abs() + dg_b + R.FLUSH, what + " dgamma accumulated")
        if not rms:
            ref = base[2 * H:].double() + db_r
            R.check(dba, ref, R.ROUND[torch.float32] * ref.abs() + db_b + R.FLUSH, what + " dbeta accumulated")
        assert torch.equal(flat[:H], base[:H])


def test_norm_rejects_bad_gamma_beta_on_the_host(ext):
    x = rand(4, 256, seed=1)
    g = torch.ones(256, device=DEV, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="gamma must be contiguous with H = 256"):
        ext.norm_fwd(x, g[:255], None, 1e-5, True)
    with pytest.raises(RuntimeError, match="gamma must be contiguous"):
        ext.norm_fwd(x, torch.ones(512, device=DEV, dtype=torch.bfloat16)[::2], None, 1e-5, True)
    with pytest.raises(RuntimeError, match="gamma must be contiguous"):
        ext.norm_fwd(x, g.cpu(), None, 1e-5, True)
    with pytest.raises(RuntimeError, match="beta must have gamma's dtype"):
        ext.norm_fwd(x, g, g.float(), 1e-5, False)
    with pytest.raises(RuntimeError, match="beta must be contiguous with H = 256"):
        ext.norm_fwd(x, g, g[:128], 1e-5, False)
    with pytest.raises(RuntimeError, match="unsupported dtypes x Float with gamma BFloat16"):
        ext.norm_fwd(x.float(), g, None, 1e-5, True)
    y, mean, rstd = ext.norm_fwd(x, g, None, 1e-5, True)
    with pytest.raises(RuntimeError, match="gamma must be contiguous with H = 256"):
        ext.norm_bwd(x, x, g[:100], mean, rstd, True, False, None, None, None)
    with pytest.raises(RuntimeError, match="unsupported dtypes x Float with gamma BFloat16"):
        ext.norm_bwd(x.float(), x.float(), g, mean, rstd, True, False, None, None, None)


def test_norm_unsupported_dtype_pair_takes_the_reference_path():
    from libai_b200.ops import functional as OF

    x = rand(5, 200, seed=1, dtype=torch.float32)
    w = (1 + 0.2 * rand(200, seed=2, dtype=torch.float32)).bfloat16()
    b = (0.2 * rand(200, seed=3, dtype=torch.float32)).bfloat16()
    mean, rstd = R.norm_stats(x, True, 1e-6)
    ref = x.double() * rstd * w.double()
    R.check(OF.rms_norm(x, w, 1e-6), ref, 2 ** -20 * ref.abs() + 2 ** -20, "rms_norm fp32 x, bf16 weight")
    ref = F.layer_norm(x.double(), (200,), w.double(), b.double(), 1e-5)
    R.check(OF.layer_norm(x, w, b, 1e-5), ref, 2 ** -20 * ref.abs() + 2 ** -20, "layer_norm fp32 x, bf16 weight")


# --------------------------------------------------------------------------------------------------------- cross-entropy
@pytest.mark.parametrize("V", [8, 1000, 1003, 32000, 50304, 151936])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_cross_entropy_matches_fp64(ext, V, dtype):
    for T in (1, 513):
        for shard in (0, 1):
            vocab_start = shard * V
            logits = (rand(T, V, seed=T + V, dtype=torch.float32) * 10).clamp(-30, 30).to(dtype)
            g = torch.Generator(device=DEV).manual_seed(V)
            labels = torch.randint(0, 2 * V, (T,), device=DEV, generator=g)
            labels[::5] = -100
            if T > 1:
                # thread 0's whole first 8-chunk (its first element when V % 8 != 0); V = 8 keeps one finite logit
                logits[0, :min(8, V - 1)] = float("-inf")
                logits[1, ::3] = float("-inf")
                logits[2, 1::2] = float("-inf")
                labels[0] = vocab_start + V - 1
                labels[1] = vocab_start + 1
                labels[2] = vocab_start
            mx, se, tgt = twice(lambda: ext.ce_stats(logits, labels, vocab_start))
            lse = mx + torch.log(se)
            loss = lse - tgt
            gloss = rand(T, seed=3, dtype=torch.float32)
            buf = logits.clone()
            assert ext.ce_bwd(buf, labels, lse, gloss, vocab_start).data_ptr() == buf.data_ptr()
            d = twice(lambda: ext.ce_bwd(logits.clone(), labels, lse, gloss, vocab_start))
            assert torch.equal(d, buf)
            R.check_ce(loss, d, logits, labels, vocab_start, gloss, f"V {V} T {T} start {vocab_start} {dtype}")


# ---------------------------------------------------------------------------------------------- SwiGLU and activations
@pytest.mark.parametrize("F_", [8, 2816, 11008, 14336, 18944])
def test_swiglu_packed_matches_fp64(ext, F_):
    for rows in (1, 777):
        gu = rand(rows, 2 * F_, seed=rows, scale=3.0)
        gy = rand(rows, F_, seed=rows + 1)
        gate, up = gu[:, :F_], gu[:, F_:]
        y_r, y_b, dg_r, dg_b, du_r, du_b = R.swiglu_ref(gate, up, gy)
        y = twice(lambda: ext.swiglu_packed_fwd(gu))
        R.check(y, y_r, R.ROUND[torch.bfloat16] * y_r.abs() + y_b + R.FLUSH, f"swiglu fwd F {F_} rows {rows}")
        dgu = twice(lambda: ext.swiglu_packed_bwd(gy, gu))
        R.check(dgu[:, :F_], dg_r, R.ROUND[torch.bfloat16] * dg_r.abs() + dg_b + R.FLUSH, f"swiglu dgate F {F_}")
        R.check(dgu[:, F_:], du_r, R.ROUND[torch.bfloat16] * du_r.abs() + du_b + R.FLUSH, f"swiglu dup F {F_}")


def all_bf16(limit=2.0 ** 16):
    """Every finite bf16 value with |x| <= limit, padded to a multiple of 8 elements."""
    x = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).to(DEV)
    x = x[torch.isfinite(x) & (x.float().abs() <= limit)]
    return torch.cat([x, x[: (-x.numel()) % 8]]).view(-1, 8)


def flushed(x):
    """x in fp64 with subnormals as zero, which is what the kernels (built with --use_fast_math) see: relu'(x) of a
    positive subnormal is 0."""
    v = x.double()
    return torch.where(v.abs() < 2.0 ** -126, torch.zeros_like(v), v)


@pytest.mark.parametrize("act", list(R.ACTS))
def test_activations_exhaustive_bf16(ext, act):
    x = all_bf16()
    v = flushed(x)
    ref, dref = R.act_ref(v, act)
    fa, ga = R.act_approx(v, act)
    y = ext.bias_act_fwd(x, None, act)
    R.check(y, ref, R.ROUND[torch.bfloat16] * ref.abs() + fa + R.FLUSH, f"act {act} fwd")
    one = torch.ones_like(x)
    for gx in (ext.act_bwd(one, x, act), ext.bias_act_bwd(one, x, None, act)):
        R.check(gx, dref, R.ROUND[torch.bfloat16] * dref.abs() + ga + R.FLUSH, f"act {act} grad")


def test_swiglu_gate_exhaustive_bf16(ext):
    x = all_bf16()
    gu = torch.cat([x, torch.ones_like(x)], 1)        # F = 8: gate = every bf16 value, up = 1
    y_r, y_b, dg_r, dg_b, du_r, du_b = R.swiglu_ref(flushed(x), torch.ones_like(x), torch.ones_like(x))
    R.check(ext.swiglu_packed_fwd(gu), y_r, R.ROUND[torch.bfloat16] * y_r.abs() + y_b + R.FLUSH, "swiglu gate fwd")
    dgu = ext.swiglu_packed_bwd(torch.ones_like(x), gu)
    R.check(dgu[:, :8], dg_r, R.ROUND[torch.bfloat16] * dg_r.abs() + dg_b + R.FLUSH, "swiglu gate dgate")
    R.check(dgu[:, 8:], du_r, R.ROUND[torch.bfloat16] * du_r.abs() + du_b + R.FLUSH, "swiglu gate dup")


def test_gated_mlp_matches_fp64_autograd():
    """GatedMLPFn on adjacent gate / up weights: y, gx and the three main_grads against fp64 autograd through
    down(silu(gate(x)) * up(x)).  The bound carries the bf16 rounding of every stored intermediate forward to first
    order, along with each GEMM's accumulation term."""
    from libai_b200.layers._param import param_defaults
    from libai_b200.models.llama_model import LlamaMLP
    from libai_b200.ops import gated_mlp
    from libai_b200.optim import AdamW

    H, Fh, T = 512, 1408, 300
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=11):
        mlp = LlamaMLP(H, Fh)
    opt = AdamW([{"params": list(mlp.parameters())}], lr=1e-3)
    opt.setup()
    wg, wu, wd = mlp.gate_proj.weight, mlp.up_proj.weight, mlp.down_proj.weight
    assert gated_mlp.fused_gate_up_views(wg, wu)[1] is not None
    x0, gy = rand(T, H, seed=1), rand(T, H, seed=2, scale=0.1)
    base = [p.main_grad.clone() for p in (wg, wu, wd)]
    x = x0.clone().requires_grad_(True)
    y = gated_mlp.gated_mlp(x, wg, wu, wd)
    y.backward(gy)

    u8 = R.ROUND[torch.bfloat16]
    X, G, Wg, Wu, Wd = (t.detach().double() for t in (x0, gy, wg, wu, wd))
    xr = X.clone().requires_grad_(True)
    wgr, wur, wdr = (t.clone().requires_grad_(True) for t in (Wg, Wu, Wd))
    gate, up = xr @ wgr.t(), xr @ wur.t()
    h = F.silu(gate) * up
    yr = h @ wdr.t()
    yr.backward(G)
    gt, u, hd = gate.detach(), up.detach(), h.detach()
    s = torch.sigmoid(gt)
    silu, dsilu = gt * s, s * (1 + gt * (1 - s))
    rel = R.EXPF_APPROX * (1 + gt.abs())
    # forward: error of gate / up (GEMM + bf16 store), of h, of y
    e_g = u8 * gt.abs() + H * R.ACC * (X.abs() @ Wg.abs().t())
    e_u = u8 * u.abs() + H * R.ACC * (X.abs() @ Wu.abs().t())
    e_h = u8 * hd.abs() + 1.13 * u.abs() * e_g + silu.abs() * e_u + hd.abs() * rel
    e_y = u8 * yr.detach().abs() + (Fh * R.ACC * hd.abs() + e_h) @ Wd.abs().t()
    R.check(y, yr.detach(), e_y, "gated mlp y")
    # backward: dh = gy Wd, then the SwiGLU backward, then gx and the weight gradients
    dh = G @ Wd
    e_dh = u8 * dh.abs() + H * R.ACC * (G.abs() @ Wd.abs())
    dgate, dup = dh * u * dsilu, dh * silu
    e_dgate = (u8 * dgate.abs() + (u * dsilu).abs() * e_dh + (dh * dsilu).abs() * e_u + 0.5 * (dh * u).abs() * e_g
               + (dh * u).abs() * s * (1 - s) * (1 + 2 * gt.abs()) * rel)
    e_dup = u8 * dup.abs() + silu.abs() * e_dh + 1.13 * dh.abs() * e_g + dup.abs() * rel
    e_gx = u8 * xr.grad.abs() + (2 * Fh * R.ACC * dgate.abs() + e_dgate) @ Wg.abs() \
        + (2 * Fh * R.ACC * dup.abs() + e_dup) @ Wu.abs()
    R.check(x.grad, xr.grad, e_gx, "gated mlp gx")
    for p, b0, ref, e in ((wg, base[0], wgr.grad, (T * R.ACC * dgate.abs() + e_dgate).t() @ X.abs()),
                          (wu, base[1], wur.grad, (T * R.ACC * dup.abs() + e_dup).t() @ X.abs()),
                          (wd, base[2], wdr.grad, G.abs().t() @ (T * R.ACC * hd.abs() + e_h))):
        want = b0.double() + ref
        R.check(p.main_grad, want, R.ROUND[torch.float32] * want.abs() + e, "gated mlp main_grad")


# ------------------------------------------------------------------------------------------------------------ reductions
def test_colsum_matches_fp64_and_is_deterministic(ext):
    for N in (2, 10, 4096, 11008):
        for M in (1, 777, 70000):
            x = rand(M, N, seed=M + N, scale=4.0)
            ref = torch.zeros(N, dtype=torch.float64, device=DEV)
            mag = torch.zeros_like(ref)
            for r0 in range(0, M, 8192):
                c = x[r0:r0 + 8192].double()
                ref += c.sum(0)
                mag += c.abs().sum(0)
            bound = (M + 8) * R.ACC * mag + R.FLUSH
            out = twice(lambda: ext.colsum(x))
            R.check(out, ref, R.ROUND[torch.bfloat16] * ref.abs() + bound, f"colsum {M}x{N}")
            base = rand(N, seed=1, dtype=torch.float32)
            accs = []
            for _ in range(2):
                acc = base.clone()
                ext.colsum(x, acc)
                accs.append(acc)
            assert torch.equal(accs[0], accs[1])
            want = base.double() + ref
            R.check(accs[0], want, R.ROUND[torch.float32] * want.abs() + bound, f"colsum {M}x{N} accumulate")


def test_sqnorm_covers_the_tail(ext):
    for n in (1, 3, 2 ** 20 + 3):
        x = rand(n, seed=n, dtype=torch.float32)
        x[-min(n, 3):] = 100.0                   # the n % 4 tail carries most of the sum when n is small
        ref = (x.double() ** 2).sum()
        # each thread sums at most n / 256 squares (float4 loads), then fixed trees over threads, blocks and partials
        bound = (n / 256 + 64) * R.ACC * ref
        R.check(twice(lambda: ext.sqnorm(x)), ref.reshape(1), bound, f"sqnorm n {n}")


# ------------------------------------------------------------------------------------------------------------ end to end
def test_qwen2_05b_width_llama_training_is_bit_identical_run_to_run():
    """hidden 896 (Qwen2-0.5B): its norms take the generic kernels, 14 heads over 2 K/V heads of d = 64."""
    from libai_b200.config import DictConfig
    from libai_b200.layers._param import param_defaults
    from libai_b200.models import LlamaForCausalLM

    cfg = DictConfig(dict(hidden_layers=2, vocab_size=512, hidden_size=896, intermediate_size=4864,
                          num_attention_heads=14, num_key_value_heads=2, max_position_embeddings=256,
                          rms_norm_eps=1e-6, initializer_range=0.02, use_scaled_init_for_output_weights=True,
                          scale_mask_softmax_fusion=False, amp_enabled=True, bos_token_id=1, eos_token_id=2,
                          pad_token_id=0))

    def run():
        from libai_b200.optim import AdamW

        with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
            model = LlamaForCausalLM(cfg)
        model = model.to(DEV).train()
        params = list(model.parameters())
        opt = AdamW([{"params": params}], lr=1e-3)
        opt.setup()           # fp32 main_grad slices: the norm gradients are reduced into them, as in training
        g = torch.Generator(device=DEV).manual_seed(7)
        losses = []
        for _ in range(3):
            ids = torch.randint(3, 512, (4, 192), device=DEV, generator=g)
            opt.zero_grad()
            loss = model(ids, labels=ids)["lm_loss"]
            loss.backward()
            opt.step()
            losses.append(loss.detach().float())
        return torch.stack(losses), [t.detach().clone() for p in params for t in (p, p.main_grad)]

    l1, p1 = run()
    l2, p2 = run()
    assert torch.isfinite(l1).all()
    assert torch.equal(l1, l2)
    assert all(torch.equal(a, b) for a, b in zip(p1, p2))
