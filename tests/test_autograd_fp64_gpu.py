"""The autograd wrappers of ``libai_b200.ops.functional`` (and the transformer blocks built on them) on the H100 against
fp64, element by element: forward output and every gradient, through the public functions, at the edges where a
wrapper can pick the wrong saved tensor, GEMM layout, accumulation target or upstream-gradient layout.

Function-level bounds come from ``tests/dense_ref.py`` (GEMM, norms, cross-entropy, SwiGLU), ``tests/attention_ref.py``
(flash attention, Philox masks, rotary) and ``tests/autograd_ref.py`` (linear / mlp), carried forward to first order.
A gradient that autograd returns in a parameter's dtype adds one rounding of that dtype; one accumulated into an fp32
``main_grad`` adds ``2^-24`` of every partial sum.

Block-level checks compare with a ``copy.deepcopy(...).double()`` of the same module under a comparative criterion
(see ``check_block``); the sensitivity tests at the end make one wrapper subtly wrong and require that criterion to
reject it."""
import copy
import struct

import pytest
import torch
from torch import nn

from libai_b200 import ops
from libai_b200.ops import functional as OF
from tests import attention_ref as AT
from tests import autograd_ref as AR
from tests import dense_ref as R
from tests import window_attention_ref as WR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U8 = R.ROUND[torch.bfloat16]
U32 = R.ROUND[torch.float32]
ACTS = [None, "gelu", "gelu_tanh", "relu", "silu", "quick_gelu"]


def rand(*shape, seed, dtype=torch.bfloat16, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, device=DEV, generator=g) * scale).to(dtype)


def upstream(shape, seed):
    """The upstream-gradient layouts autograd hands a wrapper: contiguous, an expanded stride-0 one (what
    ``y.sum().backward()`` produces, here with distinct values along the last axis) and a permuted view."""
    n = len(shape)
    return [("contiguous", rand(*shape, seed=seed)),
            ("expanded", rand(shape[-1], seed=seed + 1).expand(*shape)),
            ("permuted", rand(*reversed(shape), seed=seed + 2).permute(*reversed(range(n))))]


def as_grad(t, ref, bound, what):
    """A gradient autograd returns in ``t``'s dtype: one more rounding of that dtype."""
    assert t.grad is not None, f"{what}: no gradient"
    u = R.ROUND[t.dtype]
    R.check(t.grad, ref, u * ref.abs() + (1 + u) * bound, what)


def generator_state():
    """(seed, offset) of the default CUDA generator."""
    return struct.unpack("<QQ", bytes(torch.cuda.get_rng_state(DEV).tolist()))


def flat_params(*params, seed=0):
    """Parameters in an AdamW flat buffer (fp32 ``main_grad`` slices) whose ``main_grad`` starts from a random base;
    returns the optimizer and the bases."""
    from libai_b200.optim import AdamW

    opt = AdamW([{"params": list(params)}], lr=1e-3)
    opt.setup()
    bases = []
    for i, p in enumerate(params):
        p.main_grad.copy_(rand(*p.shape, seed=seed + i, dtype=torch.float32))
        bases.append(p.main_grad.clone())
    return opt, bases


def accumulated(base, grads):
    """fp64 ``base + sum(grads)`` and the rounding bound of adding them one by one into fp32."""
    want, bound = base.double(), torch.zeros_like(base, dtype=torch.float64)
    for ref, e in grads:
        want = want + ref
        bound = bound + e + U32 * want.abs()
    return want, bound + R.FLUSH


# ------------------------------------------------------------------------------------------------------------- linear
LINEAR_GRADS = ["xwb", "xw", "xb", "wb", "x", "w", "b", "xw-nobias", "x-nobias", "w-nobias"]


@pytest.mark.parametrize("grads", LINEAR_GRADS)
@pytest.mark.parametrize("act", ACTS)
def test_linear(act, grads):
    """Every activation, bias or none, every requires_grad subset (bias only: a frozen weight under BitFit or LoRA with
    trainable biases), a 3-D strided input and every upstream layout."""
    B, S, K, N = 3, 67, 72, 136
    x0 = rand(S, B, K + 16, seed=1)[:, :, 8:8 + K].transpose(0, 1)        # [B, S, K], neither row- nor batch-contiguous
    w0 = rand(N, K, seed=2, scale=0.3)
    b0 = None if "nobias" in grads else rand(N, seed=3)
    need = grads.split("-")[0]
    for layout, gy in upstream((B, S, N), seed=10):
        x = x0.detach().requires_grad_("x" in need)
        w = w0.clone().requires_grad_("w" in need)
        b = None if b0 is None else b0.clone().requires_grad_("b" in need)
        y = OF.linear(x, w, b, act)
        assert type(y.grad_fn).__name__ == "_LinearFnBackward"
        y.backward(gy)
        what = f"linear act={act} grads={grads} gy={layout}"
        ref = AR.linear_ref(x0.reshape(-1, K), w0, b0, gy.reshape(-1, N), act)
        R.check(y.reshape(-1, N), *ref["y"], what + " y")
        if "x" in need:
            R.check(x.grad.reshape(-1, K), *ref["gx"], what + " gx")
        for t, key in ((w, "gw"), (b, "gb")):
            if t is not None and t.requires_grad:
                as_grad(t, *ref[key], what + " " + key)


def test_linear_main_grad_two_micro_batches():
    """Weight and bias gradients accumulate into the fp32 main_grad on top of what was there; sync_gradients() then has
    nothing left to fold."""
    M, K, N = 203, 72, 136
    w, b = nn.Parameter(rand(N, K, seed=1, scale=0.3)), nn.Parameter(rand(N, seed=2))
    opt, (wb, bb) = flat_params(w, b, seed=50)
    gws, gbs = [], []
    for mb in range(2):
        x = rand(M, K, seed=10 + mb).requires_grad_(True)
        gy = rand(M, N, seed=20 + mb)
        OF.linear(x, w, b, "gelu").backward(gy)
        ref = AR.linear_ref(x.detach(), w.detach(), b.detach(), gy, "gelu")
        gws.append(ref["gw"])
        gbs.append(ref["gb"])
    assert w.grad is None and b.grad is None and w.grad_added_to_main_grad and b.grad_added_to_main_grad
    for p, base, gs, what in ((w, wb, gws, "w"), (b, bb, gbs, "b")):
        R.check(p.main_grad, *accumulated(base, gs), f"{what}.main_grad after two micro-batches")
    before = [w.main_grad.clone(), b.main_grad.clone()]
    opt.sync_gradients()
    assert torch.equal(w.main_grad, before[0]) and torch.equal(b.main_grad, before[1])


@pytest.mark.parametrize("fused_bias_grad", [True, False])
@pytest.mark.parametrize("epilogue", ["b2+residual", "plain"])
def test_mlp(epilogue, fused_bias_grad):
    M, K, Fh = 203, 72, 264
    x0 = rand(M, K, seed=1)
    w1, b1 = nn.Parameter(rand(Fh, K, seed=2, scale=0.3)), nn.Parameter(rand(Fh, seed=3))
    w2, b2 = nn.Parameter(rand(K, Fh, seed=4, scale=0.2)), nn.Parameter(rand(K, seed=5))
    opt, bases = flat_params(w1, b1, w2, b2, seed=60)
    res0 = rand(M, K, seed=6) if epilogue != "plain" else None
    old = ops.fused_bias_grad()
    ops.set_fused_bias_grad(fused_bias_grad)
    try:
        sums = {k: [] for k in ("gw1", "gb1", "gw2", "gb2")}
        for mb, (layout, gy) in enumerate(upstream((M, K), seed=30)[:2]):
            x = x0.clone().requires_grad_(True)
            res = None if res0 is None else res0.clone().requires_grad_(True)
            y = OF.mlp(x, w1, b1, w2, "gelu", b2 if res is not None else None, res)
            assert type(y.grad_fn).__name__ == "_MLPFnBackward"
            y.backward(gy)
            ref = AR.mlp_ref(x0, w1.detach(), b1.detach(), w2.detach(), gy, "gelu", b2.detach() if res is not None else None,
                             res0)
            what = f"mlp {epilogue} fused_bias_grad={fused_bias_grad} gy={layout}"
            R.check(y, *ref["y"], what + " y")
            R.check(x.grad, *ref["gx"], what + " gx")
            if res is not None:
                assert torch.equal(res.grad, gy.contiguous()), what + " the residual's gradient is gy itself"
            for k in sums:
                sums[k].append(ref[k])
        sums["gb2"] = sums["gb2"] if res0 is not None else []
        for p, base, k in zip((w1, b1, w2, b2), bases, ("gw1", "gb1", "gw2", "gb2")):
            assert p.grad is None
            R.check(p.main_grad, *accumulated(base, sums[k]), f"mlp {epilogue} {k} main_grad")
    finally:
        ops.set_fused_bias_grad(old)


@pytest.mark.parametrize("has_bias", [True, False])
@pytest.mark.parametrize("grad_to", ["autograd", "main_grad"])
def test_linear_bias_residual(grad_to, has_bias):
    """With ``grad_to="main_grad"`` the weight and bias own fp32 main_grad slices, and the three upstream layouts
    accumulate into them as three micro-batches would."""
    B, S, K, N = 2, 101, 72, 136
    x0, w0, b0, r0 = rand(B, S, K, seed=1), rand(N, K, seed=2, scale=0.3), rand(N, seed=3), rand(B, S, N, seed=4)
    if grad_to == "main_grad":
        params = [nn.Parameter(w0.clone())] + ([nn.Parameter(b0.clone())] if has_bias else [])
        _, bases = flat_params(*params, seed=70)
        w, b = params[0], (params[1] if has_bias else None)
        sums = {"gw": [], "gb": []}
    for layout, gy in upstream((B, S, N), seed=40):
        x, r = x0.clone().requires_grad_(), r0.clone().requires_grad_()
        if grad_to == "autograd":
            w = w0.clone().requires_grad_()
            b = b0.clone().requires_grad_() if has_bias else None
        y = OF.linear_bias_residual(x, w, b, r)
        assert type(y.grad_fn).__name__ == "_LinearFnBackward"
        y.backward(gy)
        what = f"linear_bias_residual {grad_to} bias={has_bias} gy={layout}"
        ref = AR.linear_ref(x0.reshape(-1, K), w0, b0 if has_bias else None, gy.reshape(-1, N), None)
        yr = ref["y"][0] + r0.reshape(-1, N).double()
        # the bound of x @ w^T + bias, plus the residual's fp32 add and the bf16 rounding of the sum
        R.check(y.reshape(-1, N), yr, ref["y"][1] + (U8 + 2.0 ** -23) * yr.abs(), what + " y")
        R.check(x.grad.reshape(-1, K), *ref["gx"], what + " gx")
        if grad_to == "autograd":
            as_grad(w, *ref["gw"], what + " gw")
            if has_bias:
                as_grad(b, *ref["gb"], what + " gb")
        else:
            sums["gw"].append(ref["gw"])
            sums["gb"].append(ref["gb"])
        assert torch.equal(r.grad, gy.contiguous()), what + " the residual's gradient is gy itself"
    if grad_to == "main_grad":
        for p, base, k in zip(params, bases, ("gw", "gb")):
            assert p.grad is None and p.grad_added_to_main_grad, f"linear_bias_residual {k} did not go to main_grad"
            R.check(p.main_grad, *accumulated(base, sums[k]), f"linear_bias_residual bias={has_bias} {k} main_grad")


# -------------------------------------------------------------------------------------------------------------- norms
def norm_fwd_ref(x, gamma, beta, rms, eps, out_dtype):
    """fp64 LayerNorm / RMSNorm of x [R, H] and its bound (the forward bound of dense_ref.check_norm_fwd)."""
    H = x.shape[1]
    c = (H + 8) * R.ACC
    xd = x.double()
    mean, rstd = R.norm_stats(x, rms, eps)
    xh = (xd - mean) * rstd
    g = gamma.double()
    ref = xh * g + (0.0 if beta is None else beta.double())
    dmean = 0.0 if rms else c * xd.abs().mean(1, keepdim=True)
    dxh = rstd * dmean + c * xh.abs()
    return ref, R.ROUND[out_dtype] * ref.abs() + g.abs() * dxh + c * ref.abs() + R.FLUSH


NORM_DTYPES = [(torch.bfloat16, torch.bfloat16), (torch.bfloat16, torch.float32), (torch.float32, torch.float32)]


@pytest.mark.parametrize("dtypes", NORM_DTYPES, ids=["bf16-bf16", "bf16-fp32", "fp32-fp32"])
@pytest.mark.parametrize("kind", ["layer_norm", "rms_norm", "skip:norm", "skip:skip", "skip:both"])
def test_norm(kind, dtypes):
    """layer_norm / rms_norm, and layer_norm_with_skip with only the norm output, only the skip output or both used."""
    xdt, wdt = dtypes
    B, S, H, eps = 2, 101, 384, 1e-5
    rms = kind == "rms_norm"
    x0 = (rand(B, S, H, seed=1, dtype=torch.float32) * 2 + 0.5).to(xdt)
    g0 = (1 + 0.2 * rand(H, seed=2, dtype=torch.float32)).to(wdt)
    b0 = None if rms else (0.2 * rand(H, seed=3, dtype=torch.float32)).to(wdt)
    for layout, gy in upstream((B, S, H), seed=10):
        gy, gs = gy.to(xdt), rand(B, S, H, seed=20, dtype=xdt)
        x = x0.clone().requires_grad_()
        g = g0.clone().requires_grad_()
        b = None if b0 is None else b0.clone().requires_grad_()
        use_norm, use_skip = True, False
        if kind == "rms_norm":
            y = OF.rms_norm(x, g, eps)
            outs, grads = [y], [gy]
        elif kind == "layer_norm":
            y = OF.layer_norm(x, g, b, eps)
            outs, grads = [y], [gy]
        else:
            y, s = OF.layer_norm_with_skip(x, g, b, eps)
            use = kind.split(":")[1]
            use_norm, use_skip = use in ("norm", "both"), use in ("skip", "both")
            outs = [y] * use_norm + [s] * use_skip
            grads = [gy] * use_norm + [gs] * use_skip
        assert type(y.grad_fn).__name__ == "_LayerNormFnBackward"
        torch.autograd.backward(outs, grads)
        what = f"{kind} {xdt}/{wdt} gy={layout}"
        x2 = x0.reshape(-1, H)
        R.check(y.reshape(-1, H), *norm_fwd_ref(x2, g0, b0, rms, eps, xdt), what + " y")
        g2 = (gy if use_norm else torch.zeros_like(gy)).reshape(-1, H)
        (gx_r, gx_b), (dg_r, dg_b), (db_r, db_b) = R.norm_bwd_ref(g2, x2, g0, rms, eps)
        ref = gx_r + (gs.reshape(-1, H).double() if use_skip else 0.0)
        R.check(x.grad.reshape(-1, H), ref, R.ROUND[xdt] * (ref.abs() + gx_r.abs()) + gx_b + R.FLUSH, what + " gx")
        as_grad(g, dg_r, U32 * dg_r.abs() + dg_b + R.FLUSH, what + " dgamma")
        if b is not None:
            as_grad(b, db_r, U32 * db_r.abs() + db_b + R.FLUSH, what + " dbeta")


@pytest.mark.parametrize("beta_main_grad", [True, False], ids=["both-main_grad", "gamma-only-main_grad"])
def test_norm_main_grad_two_micro_batches(beta_main_grad):
    """γ and β both in the flat buffer: reduced into main_grad by the kernel.  γ in it but β not: both come back as
    autograd gradients, and sync_gradients() folds γ's into its main_grad exactly once."""
    R_, H, eps = 203, 384, 1e-5
    g = nn.Parameter((1 + 0.2 * rand(H, seed=2, dtype=torch.float32)).bfloat16())
    b = nn.Parameter((0.2 * rand(H, seed=3, dtype=torch.float32)).bfloat16())
    opt, bases = flat_params(*((g, b) if beta_main_grad else (g,)), seed=70)
    dgs, dbs = [], []
    for mb in range(2):
        x = (rand(R_, H, seed=10 + mb, dtype=torch.float32) * 2 + 0.5).bfloat16().requires_grad_()
        gy = rand(R_, H, seed=20 + mb)
        y, s = OF.layer_norm_with_skip(x, g, b, eps)
        torch.autograd.backward([y, s], [gy, gy])
        _, (dg_r, dg_b), (db_r, db_b) = R.norm_bwd_ref(gy, x.detach(), g.detach(), False, eps)
        dgs.append((dg_r, dg_b))
        dbs.append((db_r, db_b))
    if beta_main_grad:
        assert g.grad is None and b.grad is None
        R.check(g.main_grad, *accumulated(bases[0], dgs), "dgamma main_grad")
        R.check(b.main_grad, *accumulated(bases[1], dbs), "dbeta main_grad")
        return
    # autograd sums the two bf16 gradients in bf16: a rounding per micro-batch and one for the sum
    for p, gs, what in ((g, dgs, "dgamma"), (b, dbs, "dbeta")):
        ref = gs[0][0] + gs[1][0]
        bound = sum((U32 * r.abs() + e) * (1 + U8) + U8 * r.abs() for r, e in gs) + U8 * ref.abs() + R.FLUSH
        R.check(p.grad, ref, bound, what + " .grad")
    grad = g.grad.clone()
    opt.sync_gradients()
    assert g.grad is None
    assert torch.equal(g.main_grad, bases[0] + grad.float()), "γ's gradient must be folded exactly once"
    opt.sync_gradients()
    assert torch.equal(g.main_grad, bases[0] + grad.float())


# --------------------------------------------------------------------------------------------- bias + act, dropout
@pytest.mark.parametrize("has_bias", [True, False])
@pytest.mark.parametrize("act", ACTS)
def test_bias_act(act, has_bias):
    B, S, N = 2, 101, 136
    x0, b0 = rand(B, S, N, seed=1, scale=2.0), (rand(N, seed=2) if has_bias else None)
    aid = AR.ACT_IDS[act]
    for layout, gy in upstream((B, S, N), seed=10):
        x = x0.clone().requires_grad_()
        b = None if b0 is None else b0.clone().requires_grad_()
        y = OF.bias_gelu(x, b) if act == "gelu" else OF.bias_act(x, b, act)
        assert type(y.grad_fn).__name__ == "_BiasActFnBackward"
        y.backward(gy)
        what = f"bias_act {act} bias={has_bias} gy={layout}"
        v = x0.reshape(-1, N).double() + (0.0 if b0 is None else b0.double())
        e_v = 2.0 ** -24 * v.abs()                                    # x + bias in fp32
        yr, _ = R.act_ref(v, aid)
        fa, _ = R.act_approx(v, aid)
        lip = 1.0 if aid in (0, 3) else R.ACT_LIPSCHITZ
        R.check(y.reshape(-1, N), yr, U8 * yr.abs() + lip * e_v + fa + R.FLUSH, what + " y")
        gx, e_gx = AR._act_grad(gy.reshape(-1, N).double(), v, e_v, aid)
        R.check(x.grad.reshape(-1, N), gx, e_gx, what + " gx")
        if b is not None:
            # the bias gradient is the column sum of the kernel's bf16 gx
            M = gx.shape[0]
            as_grad(b, gx.sum(0), (M + 8) * R.ACC * gx.abs().sum(0) + e_gx.sum(0), what + " gb")


DROPOUT_CASES = ["p0", "eval", "p0.1", "p0.1-no-residual", "p0.1-no-bias", "p0.1-salt", "dropout"]


@pytest.mark.parametrize("case", DROPOUT_CASES)
def test_bias_dropout_add(case):
    B, S, N = 2, 101, 136
    x0, b0, r0 = rand(B, S, N, seed=1, scale=3.0), rand(N, seed=2), rand(B, S, N, seed=3)
    has_bias = case not in ("p0.1-no-bias", "dropout")
    has_res = case not in ("p0.1-no-residual", "dropout")
    p = 0.0 if case == "p0" else 0.1
    training = case != "eval"
    salt = 5 if case == "p0.1-salt" else 0
    for layout, gy in upstream((B, S, N), seed=10):
        x = x0.clone().requires_grad_()
        b = b0.clone().requires_grad_() if has_bias else None
        r = r0.clone().requires_grad_() if has_res else None
        gen = generator_state()
        if case == "dropout":
            y = OF.dropout(x, p, training)
        elif salt:
            y = OF._BiasDropoutAddFn.apply(x, b, r, p, salt)
        else:
            y = OF.bias_dropout_add(x, b, r, p, training)
        dropped = p > 0 and training
        assert type(y.grad_fn).__name__ == ("_BiasDropoutAddFnBackward" if dropped else "_BiasAddFnBackward")
        y.backward(gy)
        what = f"bias_dropout_add {case} gy={layout}"
        xb = x0.reshape(-1, N).double() + (b0.double() if has_bias else 0.0)
        G = gy.reshape(-1, N).double()
        keep, scale = torch.ones_like(xb, dtype=torch.bool), 1.0
        if dropped:
            # the mask of the generator's (seed ^ salt, offset): the backward must replay it from the saved state
            thr, scale = AT.bdr_drop_threshold(p)
            keep = AT.bdr_keep_mask(AT.salted_seed(gen[0], salt), gen[1], xb.numel(), thr, device=DEV).reshape(xb.shape)
        yr = torch.where(keep, xb * scale, torch.zeros_like(xb)) + (r0.reshape(-1, N).double() if has_res else 0.0)
        # fp32 x + b, * scale and + residual each round at 2^-24 of their result (2^-23 per term with room); bf16 output
        dev = 2.0 ** -23 * (2 * xb.abs() * scale * keep + yr.abs())
        R.check(y.reshape(-1, N), yr, U8 * yr.abs() + (1 + U8) * dev + R.FLUSH, what + " y")
        gx = torch.where(keep, G * scale, torch.zeros_like(G))
        e_gx = U8 * gx.abs() + 2.0 ** -23 * gx.abs()
        R.check(x.grad.reshape(-1, N), gx, e_gx, what + " gx")
        if has_bias:
            M = gx.shape[0]
            as_grad(b, gx.sum(0), (M + 8) * R.ACC * gx.abs().sum(0) + e_gx.sum(0) + R.FLUSH, what + " gb")
        if has_res:
            assert torch.equal(r.grad, gy.contiguous()), what + " the residual's gradient is gy itself"


# ----------------------------------------------------------------------------------------------------------- attention
ATTN_CASES = ["bias[1,A]", "bias[B,1]", "bias[Sq,Sk]", "bias-fp32[B,A]", "alibi", "kv_start+kv_lens", "gqa"]


@pytest.mark.parametrize("case", ATTN_CASES)
def test_attention(case):
    """attention(): a dense bias broadcast over batch and / or heads (its gradient summed over the broadcast axes and
    reshaped back, a key length that takes the row-padded bias layout), ALiBi, key windows, grouped heads."""
    B, A, Sq, Sk, D = 2, 4, 77, 203, 64
    G = 2 if case == "gqa" else A
    causal = case in ("alibi", "gqa")
    q0, k0, v0 = rand(B, A, Sq, D, seed=1), rand(B, G, Sk, D, seed=2), rand(B, G, Sk, D, seed=3)
    bias0 = alibi = kv_start = kv_lens = None
    if case.startswith("bias"):
        shape = {"bias[1,A]": (1, A, Sq, Sk), "bias[B,1]": (B, 1, Sq, Sk), "bias[Sq,Sk]": (Sq, Sk),
                 "bias-fp32[B,A]": (B, A, Sq, Sk)}[case]
        bias0 = rand(*shape, seed=4, scale=2.0, dtype=torch.float32 if "fp32" in case else torch.bfloat16)
    if case == "alibi":
        alibi = torch.tensor([2.0 ** (-8 * (h + 1) / A) for h in range(A)], device=DEV)
    if case == "kv_start+kv_lens":
        kv_start = torch.tensor([3, 50], dtype=torch.int32, device=DEV)
        kv_lens = torch.tensor([Sk, 120], dtype=torch.int32, device=DEV)
    # the bias as the kernels must see it, built from the caller's bias: bf16, broadcast to 4-D
    b_ref = None
    if bias0 is not None:
        b_ref = bias0.to(torch.bfloat16)
        while b_ref.dim() < 4:
            b_ref = b_ref.unsqueeze(0)
    scale = D ** -0.5
    vis = OF.visible_keys(Sq, Sk, causal=causal, kv_start=kv_start, kv_lens=kv_lens, device=DEV)
    (o_r, o_b), _ = AT.attention_fwd_ref(q0, k0, v0, scale=scale, vis=vis, bias=b_ref, alibi=alibi, tile=128)
    for layout, do in upstream((B, A, Sq, D), seed=20):
        q, k, v = (t.clone().requires_grad_() for t in (q0, k0, v0))
        bias = None if bias0 is None else bias0.clone().requires_grad_()
        o = OF.attention(q, k, v, causal=causal, bias=bias, alibi_slopes=alibi, kv_lens=kv_lens, kv_start=kv_start)
        assert type(o.grad_fn).__name__ == "_FlashAttnFnBackward"
        lse, b_seen = o.grad_fn.saved_tensors[4], o.grad_fn.saved_tensors[5]
        if bias0 is not None:
            assert b_seen.shape == b_ref.shape and torch.equal(b_seen, b_ref), "the kernels were handed another bias"
        o.backward(do)
        what = f"attention {case} do={layout}"
        R.check(o, o_r, o_b, what + " o")
        ref = AT.attention_bwd_ref(q0, k0, v0, do, o.detach(), lse, scale=scale, vis=vis, bias=b_ref, alibi=alibi)
        R.check(q.grad, *ref["dq"], what + " dq")
        R.check(k.grad, *ref["dk"], what + " dk")
        R.check(v.grad, *ref["dv"], what + " dv")
        if bias is not None:
            db, db_b = ref["dbias"]
            as_grad(bias, db.reshape(bias.shape), db_b.reshape(bias.shape), what + " dbias")


@pytest.mark.parametrize("heads", [(4, 4), (8, 2)], ids=["mha", "gqa"])
def test_attention_qkvpacked(heads):
    """The packed projection ([b, s, a, 3d] or grouped [b, s, g, r + 2, d]): one dqkv of the same layout, with key
    lengths."""
    A, G = heads
    B, S, D = 2, 203, 64
    r = A // G
    if A == G:
        qkv0 = rand(B, S, A, 3 * D, seed=1)
    else:
        qkv0 = rand(B, S, G, r + 2, D, seed=1)
    kv_lens = torch.tensor([S, 150], dtype=torch.int32, device=DEV)
    q4, k4, v4 = (t.permute(0, 2, 1, 3) for t in OF.split_qkv(qkv0))
    vis = OF.visible_keys(S, S, causal=True, kv_lens=kv_lens, device=DEV)
    (o_r, o_b), _ = AT.attention_fwd_ref(q4, k4, v4, scale=D ** -0.5, vis=vis, tile=128)
    for layout, do in upstream((B, S, A, D), seed=30):
        _check_packed(qkv0, q4, k4, v4, do, kv_lens, vis, o_r, o_b, A, G, f"attention_qkvpacked A/G={A}/{G} do={layout}")


def _check_packed(qkv0, q4, k4, v4, do, kv_lens, vis, o_r, o_b, A, G, what):
    B, S, D = qkv0.shape[0], qkv0.shape[1], q4.shape[-1]
    r = A // G
    qkv = qkv0.clone().requires_grad_()
    o = OF.attention_qkvpacked(qkv, causal=True, scale=D ** -0.5, kv_lens=kv_lens)
    o_saved, lse = o.grad_fn.saved_tensors[1], o.grad_fn.saved_tensors[2]
    o.backward(do)
    R.check(o.permute(0, 2, 1, 3), o_r, o_b, what + " o")
    ref = AT.attention_bwd_ref(q4, k4, v4, do.permute(0, 2, 1, 3), o_saved, lse, scale=D ** -0.5, vis=vis)
    (dq, dqb), (dk, dkb), (dv, dvb) = ref["dq"], ref["dk"], ref["dv"]
    if A == G:     # per head [q | k | v]
        want = torch.cat([dq, dk, dv], -1).permute(0, 2, 1, 3)
        bound = torch.cat([dqb, dkb, dvb], -1).permute(0, 2, 1, 3)
    else:          # per group q_0 .. q_{r-1}, k, v
        def grouped(t, tk, tv):
            return torch.cat([t.reshape(B, G, r, S, D).permute(0, 3, 1, 2, 4), tk.permute(0, 2, 1, 3)[:, :, :, None],
                              tv.permute(0, 2, 1, 3)[:, :, :, None]], 3)
        want, bound = grouped(dq, dk, dv), grouped(dqb, dkb, dvb)
    R.check(qkv.grad, want, bound, what + " dqkv")


@pytest.mark.parametrize("cosine", [False, True], ids=["swin", "swinv2"])
def test_window_attention(cosine):
    """window_attention(): gradients of qkv, the relative-position table and tau through the wrapper, with the
    tolerances of tests/window_attention_ref.py."""
    B, H, W, ws, shift, heads, d = 2, 8, 8, 4, 2, 3, 32
    g = torch.Generator().manual_seed(5)
    qkv0 = (torch.randn(B, H * W, 3 * heads * d, generator=g)).bfloat16().to(DEV)
    table0 = (0.5 * torch.randn((2 * ws - 1) ** 2, heads, generator=g)).to(DEV)
    tau0 = (10.0 * (1.0 + 0.1 * torch.rand(heads, generator=g))).to(DEV) if cosine else None
    scale = d ** -0.5
    o_ref, o_mag = WR.forward(qkv0, H, W, ws, shift, heads, scale, table0, tau0)
    for layout, dout in upstream((B, H * W, heads * d), seed=7):
        qkv, table = qkv0.clone().requires_grad_(), table0.clone().requires_grad_()
        tau = None if tau0 is None else tau0.clone().requires_grad_()
        o = OF.window_attention(qkv, H=H, W=W, window=ws, shift=shift, heads=heads, scale=scale, table=table, tau=tau)
        o.backward(dout)
        what = f"window dout={layout}"
        WR.assert_close(o, o_ref, o_mag, what + " O")
        (g_ref, g_mag), (t_ref, t_mag), (u_ref, u_mag) = WR.backward(dout.contiguous(), qkv0, H, W, ws, shift, heads,
                                                                     scale, table0, tau0)
        WR.assert_close(qkv.grad, g_ref, g_mag, what + " dqkv")
        WR.assert_close(table.grad, t_ref, t_mag, what + " dtable", tol=WR.DS_TOL, out_tol=2.0 ** -20)
        if cosine:
            WR.assert_close(tau.grad, u_ref, u_mag, what + " dtau", tol=WR.DS_TOL, out_tol=2.0 ** -20)


# -------------------------------------------------------------------------------------------------- cross-entropy
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_vocab_parallel_cross_entropy_masked_mean(dtype):
    """Per-token losses of [b, s, V] logits, ignored labels (outside the vocabulary) and a masked mean: the per-token
    upstream gradient is zero where the mask is."""
    B, S, V = 3, 67, 1000
    logits0 = (rand(B, S, V, seed=1, dtype=torch.float32) * 10).clamp(-30, 30).to(dtype)
    g = torch.Generator(device=DEV).manual_seed(2)
    labels = torch.randint(0, V, (B, S), device=DEV, generator=g)
    labels[:, ::7] = -100
    mask = (torch.rand(B, S, device=DEV, generator=g) > 0.3).float()
    logits = logits0.clone().requires_grad_()
    loss = OF.vocab_parallel_cross_entropy(logits, labels)
    total = (loss * mask).sum() / mask.sum()
    total.backward()
    gloss = (mask / mask.sum()).reshape(-1)
    # ce_bwd writes dlogits over the saved logits, which here are the leaf's own storage
    R.check_ce(loss.reshape(-1), logits.grad.reshape(-1, V), logits0.reshape(-1, V), labels.reshape(-1), 0, gloss,
               f"cross-entropy {dtype}")


# ------------------------------------------------------------------------------------------------------ embedding
def scatter_ref(ids_local, inside, gy, rows):
    """fp64 row sums of gy [T, H] into ``rows`` rows and their bound: each row's fp32 sum over its n tokens."""
    H = gy.shape[1]
    G = gy.double() * inside[:, None]
    idx = ids_local.clamp(0, rows - 1)
    ref = torch.zeros(rows, H, dtype=torch.float64, device=DEV).index_add_(0, idx, G)
    mag = torch.zeros_like(ref).index_add_(0, idx, G.abs())
    cnt = torch.zeros(rows, dtype=torch.float64, device=DEV).index_add_(0, idx, inside.double())
    return ref, (cnt[:, None] + 8) * R.ACC * mag + R.FLUSH


@pytest.mark.parametrize("main_grad", [True, False])
def test_embedding(main_grad):
    """A vocabulary shard [32, 128) of ids in [0, 160): rows outside give zeros and get no gradient."""
    rows, H, start = 96, 64, 32
    table = nn.Parameter(rand(rows, H, seed=1))
    opt, bases = flat_params(table, seed=80) if main_grad else (None, None)
    gen = torch.Generator(device=DEV).manual_seed(3)
    grads = []
    for mb in range(2 if main_grad else 1):
        ids = torch.randint(0, 160, (3, 67), device=DEV, generator=gen)
        ids[0, :5] = start                      # a row many tokens share
        out = OF.embedding(ids, table, start)
        local = ids - start
        inside = (local >= 0) & (local < rows)
        want = torch.where(inside[..., None], table.detach()[local.clamp(0, rows - 1)], torch.zeros_like(out))
        assert torch.equal(out, want)
        layout, gy = upstream((3, 67, H), seed=10 + mb)[mb]
        out.backward(gy)
        grads.append(scatter_ref(local.reshape(-1), inside.reshape(-1), gy.reshape(-1, H), rows))
    if main_grad:
        assert table.grad is None
        R.check(table.main_grad, *accumulated(bases[0], grads), "embedding main_grad after two micro-batches")
    else:
        as_grad(table, *grads[0], "embedding .grad")


def test_tied_embedding_lm_head():
    """The embedding table as the LM head's weight: its main_grad gets the embedding's scatter of the LM head's input
    gradient plus the LM head's weight gradient."""
    from libai_b200.layers.lm_logits import LMLogits

    V, H, B, S = 1000, 128, 2, 67
    table = nn.Parameter(rand(V, H, seed=1, scale=0.5))
    opt, (base,) = flat_params(table, seed=90)
    head = LMLogits(V)
    ids = torch.randint(0, V, (B, S), device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    x = OF.embedding(ids, table)
    logits = head(x, table)
    gy = rand(B, S, V, seed=3, scale=0.1)
    logits.backward(gy)
    xr = table.detach()[ids.reshape(-1)]
    ref = AR.linear_ref(xr, table.detach(), None, gy.reshape(-1, V), None)
    R.check(logits.reshape(-1, V), *ref["y"], "tied LM head logits")
    # the embedding scatters the LM head's bf16 input gradient, which is within ref["gx"]'s bound of its reference
    sc, sc_b = scatter_ref(ids.reshape(-1), torch.ones(B * S, dtype=torch.bool, device=DEV), ref["gx"][0], V)
    e_gx = torch.zeros(V, H, dtype=torch.float64, device=DEV).index_add_(0, ids.reshape(-1), ref["gx"][1])
    R.check(table.main_grad, *accumulated(base, [ref["gw"], (sc, sc_b + e_gx)]), "tied table main_grad")


# -------------------------------------------------------------------------------------------------------------- rotary
def rope_tables(P, D):
    inv = 1.0 / 10000.0 ** (torch.arange(0, D, 2, device=DEV, dtype=torch.float64) / D)
    ang = torch.arange(P, device=DEV, dtype=torch.float64)[:, None] * inv[None]
    emb = torch.cat([ang, ang], -1)
    return emb.cos().float(), emb.sin().float()


def rotate(x, cos, sin, backward):
    """The rotate-half rotation of x [..., D] (tables broadcast against it) in fp64 and its bound: two fp32 products
    and a sum, each rounding at 2^-24 of a value below |x1 c| + |x2 s| (2^-22 in all), then the bf16 rounding."""
    h = x.shape[-1] // 2
    xd, c, s = x.double(), cos.double(), sin.double()
    x1, x2, c1, c2, s1, s2 = xd[..., :h], xd[..., h:], c[..., :h], c[..., h:], s[..., :h], s[..., h:]
    if not backward:
        y1, y2 = x1 * c1 - x2 * s1, x2 * c2 + x1 * s2
        m1, m2 = (x1 * c1).abs() + (x2 * s1).abs(), (x2 * c2).abs() + (x1 * s2).abs()
    else:
        y1, y2 = x1 * c1 + x2 * s2, x2 * c2 - x1 * s1
        m1, m2 = (x1 * c1).abs() + (x2 * s2).abs(), (x2 * c2).abs() + (x1 * s1).abs()
    ref = torch.cat([y1, y2], -1)
    return ref, U8 * ref.abs() + (1 + U8) * 2.0 ** -22 * torch.cat([m1, m2], -1) + R.FLUSH


@pytest.mark.parametrize("positions", ["offset", "position_ids"])
@pytest.mark.parametrize("r", [1, 4])
def test_apply_rotary_qkv(r, positions):
    """Rotary on the packed projection: q and k rotated, v passed through, at ``pos_offset + i`` or at per-token
    ``position_ids``; the caller's upstream gradient must come back unchanged."""
    B, S, G, D, off = 2, 45, 2, 64, 17
    cos, sin = rope_tables(S + off + 5, D)
    shape = (B, S, G, r + 2, D) if r > 1 else (B, S, G, 3 * D)
    qkv0 = rand(*shape, seed=1, scale=4.0)
    pos = None
    if positions == "position_ids":
        pos = torch.randint(0, S + off, (B, S), device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
        pos = pos.to(torch.int32)
        c, s = cos[pos.long()], sin[pos.long()]                         # [B, S, D]
    else:
        c, s = cos[off:off + S][None].expand(B, S, D), sin[off:off + S][None].expand(B, S, D)
    c, s = c[:, :, None, None], s[:, :, None, None]
    for layout, gy in upstream(shape, seed=10):
        gy_before = gy.clone()
        qkv = qkv0.clone().requires_grad_()
        y = OF.apply_rotary_qkv(qkv, cos, sin, off, pos)
        assert type(y.grad_fn).__name__ == "_RopeQKVFnBackward"
        y.backward(gy)
        assert torch.equal(gy, gy_before), "the backward overwrote the caller's gradient"
        what = f"apply_rotary_qkv r={r} {positions} gy={layout}"
        # a 5-D view [B, S, G, r + 2, D] of either layout: rows :r+1 rotate, the last is v
        n = r + 2 if r > 1 else 3
        v5 = (lambda t: t.reshape(B, S, G, n, D))
        R.check(v5(y)[:, :, :, :n - 1], *rotate(v5(qkv0)[:, :, :, :n - 1], c, s, False), what + " y")
        assert torch.equal(v5(y)[:, :, :, n - 1], v5(qkv0)[:, :, :, n - 1])
        R.check(v5(qkv.grad)[:, :, :, :n - 1], *rotate(v5(gy)[:, :, :, :n - 1], c, s, True), what + " dqkv")
        assert torch.equal(v5(qkv.grad)[:, :, :, n - 1], v5(gy)[:, :, :, n - 1])


# -------------------------------------------------------------------------------------------------------------- SwiGLU
def test_swiglu_unpacked_non_contiguous():
    """swiglu(gate, up) on column slices of one [M, 2F] projection (neither contiguous)."""
    M, Fh = 203, 264
    gu0 = rand(M, 2 * Fh, seed=1, scale=3.0)
    for layout, gy in upstream((M, Fh), seed=10):
        gu = gu0.clone().requires_grad_()
        gate, up = gu[:, :Fh], gu[:, Fh:]
        assert not gate.is_contiguous()
        y = OF.swiglu(gate, up)
        assert type(y.grad_fn).__name__ == "_SwigluFnBackward"
        y.backward(gy)
        y_r, y_b, dg_r, dg_b, du_r, du_b = R.swiglu_ref(gu0[:, :Fh], gu0[:, Fh:], gy)
        R.check(y, y_r, U8 * y_r.abs() + y_b + R.FLUSH, f"swiglu gy={layout} y")
        R.check(gu.grad[:, :Fh], dg_r, U8 * dg_r.abs() + dg_b + R.FLUSH, f"swiglu gy={layout} dgate")
        R.check(gu.grad[:, Fh:], du_r, U8 * du_r.abs() + du_b + R.FLUSH, f"swiglu gy={layout} dup")


# ===================================================================================================== block level
# Whole-block first-order bounds are impractical, so a block is held to a comparative criterion.  Three copies of the
# block, with the same weights, run the same two micro-batches:
# * native: the sm_90a kernels, gradients accumulated into fp32 main_grad;
# * fp64 ("exact"): a copy in fp64 through the library's PyTorch path, with its attention, norms and cross-entropy
#   (which compute in fp32 there) replaced by the same math in fp64;
# * bf16 PyTorch path (LIBAI_B200_IMPL=ref): its gradients folded into fp32 main_grad after each micro-batch.  Its
#   attention is the library's math with the rounding points of the flash kernels (attention_ref_kernel_rounding):
#   fp32 scores, P rounded to bf16 for P V, delta = rowsum(dO O) from the bf16 O, dS rounded to bf16.  The library's
#   own PyTorch attention keeps all of these in fp32, and gradients that sum over every token (a bias, a norm's γ)
#   accumulate those roundings coherently.
# With E_ref the error of the PyTorch path against the fp64 copy, every row of the output and of each input gradient,
# and every row of every parameter's accumulated gradient (every output channel of a weight; a bias or a norm weight
# as a whole), must satisfy
#     max |native - fp64| <= 4 max |E_ref| + 2^-8 max |fp64| + FLUSH
# (the last terms: one bf16 rounding of the row's largest element, for rows the PyTorch path happens to get exact).
# A vector parameter is one row: with one element per row the maxima would be single draws of two independent
# rounding errors, and |E_native| > 4 |E_ref| would then hold by chance for about one element in six.
def _rows(t):
    t = t.detach()
    return t.reshape(1, -1) if t.dim() <= 1 else t.reshape(-1, t.shape[-1]) if t.dim() > 2 else t


def check_rows(native, ref, exact, what):
    n, r, e = (_rows(t).double() for t in (native, ref, exact))
    err_n = (n - e).abs().amax(1)
    err_r = (r - e).abs().amax(1)
    allowed = 4 * err_r + U8 * e.abs().amax(1) + R.FLUSH
    bad = ~(err_n <= allowed)
    if bool(bad.any()):
        i = int(torch.argmax(torch.where(bad, err_n / allowed, torch.zeros_like(err_n))))
        raise R.Mismatch(f"{what}: {int(bad.sum())} of {bad.numel()} rows outside 4 E_ref; worst row {i}: "
                         f"native {float(err_n[i]):.3e} ref {float(err_r[i]):.3e} allowed {float(allowed[i]):.3e}")


def _visible(q, k, causal, mask):
    """The keys OF.attention_ref keeps (the others are filled with -10000 there)."""
    sq, sk = q.shape[-2], k.shape[-2]
    vis = torch.ones(sq, sk, dtype=torch.bool, device=q.device).tril(diagonal=sk - sq) if causal else None
    if mask is not None:
        vis = mask.bool() if vis is None else vis & mask.bool()
    return vis


class _KernelRoundingAttn(torch.autograd.Function):
    """Softmax attention in fp32 with the flash kernels' bf16 roundings (P for P V, the stored O that delta reads, dS)."""

    @staticmethod
    def forward(ctx, q, k, v, bias, vis, scale):
        s = torch.matmul(q.float(), k.float().transpose(-1, -2)) * scale
        if bias is not None:
            s = s + bias.float()
        if vis is not None:
            s = s.masked_fill(~vis, -10000.0)
        p = torch.softmax(s, -1)
        pb = p.to(torch.bfloat16).float()
        o = torch.matmul(pb, v.float()).to(q.dtype)
        ctx.save_for_backward(q, k, v, p, pb, o)
        ctx.scale = scale
        ctx.bias_meta = None if bias is None else (bias.shape, bias.dtype)
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, p, pb, o = ctx.saved_tensors
        do = do.float()
        dp = torch.matmul(do, v.float().transpose(-1, -2))
        ds = p * (dp - (do * o.float()).sum(-1, keepdim=True))
        dsb = ds.to(torch.bfloat16).float()
        dq = (torch.matmul(dsb, k.float()) * ctx.scale).to(q.dtype)
        dk = (torch.matmul(dsb.transpose(-1, -2), q.float()) * ctx.scale).to(k.dtype)
        dv = torch.matmul(pb.transpose(-1, -2), do).to(v.dtype)
        db = None
        if ctx.bias_meta is not None and ctx.needs_input_grad[3]:
            shape, dtype = ctx.bias_meta
            db = ds.sum_to_size(shape).to(dtype)
        return dq, dk, dv, db, None, None


def attention_ref_kernel_rounding(q, k, v, *, causal, scale, mask=None, bias=None, dropout_p=0.0, training=False,
                                  fill=-10000.0):
    assert not (training and dropout_p > 0) and fill == -10000.0
    k, v = OF._expand_kv(k, q.shape[-3]), OF._expand_kv(v, q.shape[-3])
    return _KernelRoundingAttn.apply(q, k, v, bias, _visible(q, k, causal, mask), float(scale))


def attention_ref_fp64(q, k, v, *, causal, scale, mask=None, bias=None, dropout_p=0.0, training=False, fill=-10000.0):
    """OF.attention_ref in the inputs' (fp64) precision."""
    assert not (training and dropout_p > 0)
    k, v = OF._expand_kv(k, q.shape[-3]), OF._expand_kv(v, q.shape[-3])
    s = torch.matmul(q, k.transpose(-1, -2)) * scale
    if bias is not None:
        s = s + bias.to(s.dtype)
    vis = _visible(q, k, causal, mask)
    if vis is not None:
        s = s.masked_fill(~vis, fill)
    return torch.matmul(torch.softmax(s, -1), v)


def layer_norm_fp64(x, weight, bias, eps=1e-5):
    return torch.nn.functional.layer_norm(x, (x.shape[-1],), weight, bias, eps)


def rms_norm_fp64(x, weight, eps=1e-6):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * weight


def cross_entropy_fp64(logits, labels, vocab_start=0, group=None):
    assert group is None
    V = logits.shape[-1]
    local = labels - vocab_start
    inside = (local >= 0) & (local < V)
    tgt = logits.gather(-1, local.clamp(0, V - 1)[..., None])[..., 0]
    return torch.logsumexp(logits, -1) - torch.where(inside, tgt, torch.zeros_like(tgt))


def _run(model, forward, batches, *, impl, opt=None, monkeypatch):
    """Two micro-batches through ``model``: the first output, each input gradient, and every parameter's accumulated
    gradient (fp32 main_grad for the bf16 models, fp64 .grad for the fp64 copy)."""
    fp64 = impl == "fp64"
    with monkeypatch.context() as mp:
        if impl == "ref":
            mp.setenv("LIBAI_B200_IMPL", "ref")
            mp.setattr(OF, "attention_ref", attention_ref_kernel_rounding)
        if fp64:
            mp.setattr(OF, "attention_ref", attention_ref_fp64)
            mp.setattr(OF, "layer_norm", layer_norm_fp64)
            mp.setattr(OF, "rms_norm", rms_norm_fp64)
            mp.setattr(OF, "vocab_parallel_cross_entropy", cross_entropy_fp64)
        outs, gxs = [], []
        for inputs, gy in batches:
            leaves = [t.detach().double().requires_grad_() if fp64 and t.is_floating_point() else
                      t.detach().clone().requires_grad_() if t.is_floating_point() else t for t in inputs]
            y = forward(model, *leaves)
            y.backward(gy.double() if fp64 else gy)
            outs.append(y.detach())
            gxs.append([t.grad for t in leaves if t.is_floating_point()])
            if impl == "ref":
                opt._collect_autograd_grads()          # fp32 accumulation per micro-batch, as the native path does
        if impl == "native":
            opt.sync_gradients()
    params = {n: (p.grad if fp64 else p.main_grad) for n, p in model.named_parameters()}
    return outs[0], gxs, params


def check_block(build, forward, make_batches, monkeypatch, what):
    """Build the block in bf16, copy it (bf16 for the PyTorch path, fp64 for the reference), run all three on the same
    two micro-batches and apply the comparative criterion to output, input gradients and accumulated gradients."""
    from libai_b200.layers._param import param_defaults
    from libai_b200.optim import AdamW

    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
        model = build()
    model = model.to(DEV).eval()                                  # dropout is covered at function level
    exact = copy.deepcopy(model).double()
    ref = copy.deepcopy(model)
    opts = {}
    for name, m in (("native", model), ("ref", ref)):
        opts[name] = AdamW([{"params": list(m.parameters())}], lr=1e-3)
        opts[name].setup()
    batches = make_batches()
    y_n, gx_n, p_n = _run(model, forward, batches, impl="native", opt=opts["native"], monkeypatch=monkeypatch)
    y_r, gx_r, p_r = _run(ref, forward, batches, impl="ref", opt=opts["ref"], monkeypatch=monkeypatch)
    y_e, gx_e, p_e = _run(exact, forward, batches, impl="fp64", monkeypatch=monkeypatch)
    check_rows(y_n, y_r, y_e, what + " output")
    for mb in range(len(batches)):
        for i, (a, b, c) in enumerate(zip(gx_n[mb], gx_r[mb], gx_e[mb])):
            check_rows(a, b, c, f"{what} input {i} gradient (micro-batch {mb})")
    for name in p_e:
        assert p_e[name] is not None, f"{what}: {name} got no fp64 gradient"
        assert p_n[name] is not None and p_r[name] is not None, f"{what}: {name} has no main_grad"
        check_rows(p_n[name], p_r[name], p_e[name], f"{what} {name} main_grad")


H_, S_, B_ = 256, 203, 2


def hidden_batches(S=S_, seed=0, pad_lengths=None):
    """Two micro-batches of (hidden states, upstream gradient); padded rows (past ``pad_lengths``) get no gradient,
    as a masked loss would give them."""
    out = []
    for mb in range(2):
        x = rand(B_, S, H_, seed=seed + 10 * mb)
        gy = rand(B_, S, H_, seed=seed + 10 * mb + 1)
        if pad_lengths is not None:
            keep = torch.arange(S, device=DEV)[None, :] < torch.tensor(pad_lengths, device=DEV)[:, None]
            gy = gy * keep[..., None]
        out.append(([x], gy))
    return out


def gpt2_layer():
    from libai_b200.layers import TransformerLayer
    from libai_b200.layers.attention import AttnMaskType

    return TransformerLayer(H_, 4 * H_, 4, bias_gelu_fusion=True, bias_dropout_fusion=True,
                            scale_mask_softmax_fusion=True, apply_query_key_layer_scaling=True,
                            attn_mask_type=AttnMaskType.causal, layer_idx=1)


def test_block_gpt2_pre_ln(monkeypatch):
    check_block(gpt2_layer, lambda m, x: m(x), hidden_batches, monkeypatch, "GPT-2 layer")


def test_block_bert_post_ln_key_padding(monkeypatch):
    from libai_b200.layers import TransformerLayer
    from libai_b200.layers.attention import KeyPaddingMask

    lengths = [S_, 150]
    mask2d = (torch.arange(S_, device=DEV)[None, :] < torch.tensor(lengths, device=DEV)[:, None]).long()

    def build():
        return TransformerLayer(H_, 4 * H_, 4, bias_gelu_fusion=True, bias_dropout_fusion=True,
                                apply_residual_post_layernorm=True)

    def forward(m, x):
        # the padded query rows differ by design between the key-length kernel and the dense m_i m_j mask of the
        # PyTorch path; they carry no gradient and are left out of the comparison
        y = m(x, KeyPaddingMask(mask2d))
        return y * mask2d[..., None].to(y.dtype)

    check_block(build, forward, lambda: hidden_batches(pad_lengths=lengths), monkeypatch, "BERT post-LN layer")


def test_block_t5_decoder_cross_attention(monkeypatch):
    from libai_b200.layers import TransformerLayer
    from libai_b200.layers.attention import AttnMaskType

    S_enc = 77

    def build():
        return TransformerLayer(H_, 4 * H_, 4, is_decoder=True, bias_gelu_fusion=True, bias_dropout_fusion=True,
                                attn_mask_type=AttnMaskType.causal)

    def batches():
        return [([x[0], rand(B_, S_enc, H_, seed=100 + mb)], gy) for mb, (x, gy) in enumerate(hidden_batches(seed=5))]

    check_block(build, lambda m, x, enc: m(x, None, enc, None), batches, monkeypatch, "T5 decoder layer")


@pytest.mark.parametrize("kind", ["decoder", "encoder"])
def test_block_mt5_relative_position_bias(kind, monkeypatch):
    """The MT5 layer with its relative-position table: a gather, a permute to a [1, a, q, k] bias (the decoder adds
    its causal mask into it, the unmasked encoder hands the permuted view itself to _prep_bias), dbias summed over the
    batch and scattered back into the table.  The decoder also runs cross-attention over right-padded encoder states."""
    from libai_b200.layers._param import xavier_normal_
    from projects.MT5.mt5_model import TransformerLayer as MT5Layer

    S_enc, enc_lengths = 77, [77, 50]
    decoder = kind == "decoder"

    def build():
        return MT5Layer(H_, 704, 4, 64, 32, is_decoder=decoder, init_method=xavier_normal_, layer_idx=0,
                        has_relative_attention_bias=True)

    causal = torch.ones(S_, S_, dtype=torch.bool, device=DEV).tril()[None, None].expand(B_, 1, S_, S_)
    enc_mask = (torch.arange(S_enc, device=DEV)[None, :] < torch.tensor(enc_lengths, device=DEV)[:, None])
    enc_mask = enc_mask[:, None, None, :]

    def batches():
        out = hidden_batches(seed=7)
        if decoder:
            out = [([x[0], rand(B_, S_enc, H_, seed=200 + mb)], gy) for mb, (x, gy) in enumerate(out)]
        return out

    def forward(m, x, enc=None):
        if decoder:
            return m(x, causal, enc, enc_mask)[0]
        return m(x)[0]

    check_block(build, forward, batches, monkeypatch, f"MT5 {kind} layer")


def test_block_llama_gqa(monkeypatch):
    from libai_b200.models.llama_model import LlamaDecoderLayer, rotary_tables

    cos, sin = rotary_tables(32, S_, device=DEV)

    def build():
        return LlamaDecoderLayer(H_, 704, 8, num_key_value_heads=2, rms_norm_eps=1e-6, max_position_embeddings=S_)

    check_block(build, lambda m, x: m(x, cos_cached=cos, sin_cached=sin), hidden_batches, monkeypatch,
                "Llama GQA layer")


class EmbedHeadCE(nn.Module):
    """GPT's token + position embedding, final LayerNorm, tied LM head and cross-entropy with a masked mean."""

    def __init__(self, V, H, S):
        super().__init__()
        from libai_b200.layers import LayerNorm, VocabEmbedding

        self.word = VocabEmbedding(V, H)
        self.pos = VocabEmbedding(S, H)
        self.norm = LayerNorm(H)
        from libai_b200.layers.lm_logits import LMLogits

        self.head = LMLogits(V)

    def forward(self, ids, labels, mask):
        pos = torch.arange(ids.shape[1], device=ids.device)[None].expand_as(ids)
        h = self.norm(self.word(ids) + self.pos(pos))
        loss = OF.vocab_parallel_cross_entropy(self.head(h, self.word.weight), labels)
        return (loss.float() * mask).sum() / mask.sum()


def test_block_embedding_lm_head_cross_entropy(monkeypatch):
    V = 1000
    gen = torch.Generator(device=DEV).manual_seed(11)

    def batches():
        out = []
        for _ in range(2):
            ids = torch.randint(0, V, (B_, S_), device=DEV, generator=gen)
            mask = (torch.rand(B_, S_, device=DEV, generator=gen) > 0.3).float()
            out.append(([ids, ids.roll(-1, 1), mask], torch.ones((), device=DEV)))
        return out

    # the mask is a float input too: its gradient is each token's loss minus the mean, over the mask's sum
    check_block(lambda: EmbedHeadCE(V, H_, S_), lambda m, ids, labels, mask: m(ids, labels, mask), batches, monkeypatch,
                "embedding + LM head + CE")


# ===================================================================================================== sensitivity
# Each test makes one wrapper subtly wrong (Python only) and requires the block criterion above to reject it.
def _expect_rejected(monkeypatch, what):
    with pytest.raises(R.Mismatch):
        check_block(gpt2_layer, lambda m, x: m(x), hidden_batches, monkeypatch, what)


def _scaled_bias_grad(ext, g2, bias):
    """_bias_grad off by a factor (1 + 2^-5)."""
    mg = getattr(bias, "main_grad", None)
    s = ext.colsum(g2).float() * (1 + 2.0 ** -5)
    if mg is not None and mg.dtype == torch.float32:
        mg.add_(s)
        bias.grad_added_to_main_grad = True
        return None
    return s.to(bias.dtype)


def test_block_check_rejects_scaled_bias_gradient(monkeypatch):
    monkeypatch.setattr(OF, "_bias_grad", _scaled_bias_grad)
    _expect_rejected(monkeypatch, "bias gradient * (1 + 2^-5)")


def test_linear_checks_reject_scaled_bias_gradient(monkeypatch):
    """The scaled bias gradient is caught whether it returns to autograd or accumulates into main_grad."""
    monkeypatch.setattr(OF, "_bias_grad", _scaled_bias_grad)
    with pytest.raises(R.Mismatch, match="gb"):
        test_linear("gelu", "b")
    for grad_to in ("autograd", "main_grad"):
        with pytest.raises(R.Mismatch, match="gb"):
            test_linear_bias_residual(grad_to=grad_to, has_bias=True)


def test_block_check_rejects_scaled_attention_weight_gradients(monkeypatch):
    """The attention projections' weight gradients off by a factor (1 + 2^-5)."""
    orig = OF._LinearFn.backward

    def wrong(ctx, gy):
        w = ctx.saved_tensors[1]
        before = w.main_grad.clone()
        out = orig(ctx, gy)
        w.main_grad.add_((w.main_grad - before) * 2.0 ** -5)
        return out

    monkeypatch.setattr(OF._LinearFn, "backward", staticmethod(wrong))
    _expect_rejected(monkeypatch, "weight gradient * (1 + 2^-5)")


def test_block_check_rejects_scaled_norm_gradient(monkeypatch):
    """γ / β gradients of the LayerNorms off by a factor (1 + 2^-5)."""
    orig = OF._LayerNormFn.backward

    def wrong(ctx, gy, gskip=None):
        x2, weight, _, _ = ctx.saved_tensors
        grads = (weight.main_grad, ctx.bias_param.main_grad)
        before = [g.clone() for g in grads]
        out = orig(ctx, gy, gskip)
        for g, b in zip(grads, before):
            g.add_((g - b) * 2.0 ** -5)
        return out

    monkeypatch.setattr(OF._LayerNormFn, "backward", staticmethod(wrong))
    _expect_rejected(monkeypatch, "LayerNorm gradients * (1 + 2^-5)")


def test_block_check_rejects_dropped_skip_gradient(monkeypatch):
    orig = OF._LayerNormFn.backward

    def wrong(ctx, gy, gskip=None):
        return orig(ctx, gy, None)

    monkeypatch.setattr(OF._LayerNormFn, "backward", staticmethod(wrong))
    _expect_rejected(monkeypatch, "LayerNorm backward without gadd")


def test_block_check_rejects_linear_main_grad_added_twice(monkeypatch):
    orig = OF._LinearFn.backward
    seen = []

    def wrong(ctx, gy):
        w = ctx.saved_tensors[1]
        before = w.main_grad.clone() if getattr(w, "main_grad", None) is not None else None
        out = orig(ctx, gy)
        if before is not None and not seen:            # the first micro-batch's wgrad lands twice
            seen.append(True)
            w.main_grad.add_(w.main_grad - before)
        return out

    monkeypatch.setattr(OF._LinearFn, "backward", staticmethod(wrong))
    _expect_rejected(monkeypatch, "one micro-batch's main_grad added twice")


def test_block_check_rejects_swapped_head_dq(monkeypatch):
    orig = OF._FlashAttnPackedFn.backward

    def wrong(ctx, go):
        out = orig(ctx, go)
        dqkv = out[0]                                  # [b, s, a, 3d]: swap the dq of heads 0 and 1
        d = dqkv.shape[-1] // 3
        q0 = dqkv[:, :, 0, :d].clone()
        dqkv[:, :, 0, :d] = dqkv[:, :, 1, :d]
        dqkv[:, :, 1, :d] = q0
        return out

    monkeypatch.setattr(OF._FlashAttnPackedFn, "backward", staticmethod(wrong))
    _expect_rejected(monkeypatch, "dq of heads 0 and 1 swapped")
