"""fp64 references, with per-element bounds, of the linear-layer autograd wrappers in ``libai_b200.ops.functional``
(``linear`` and ``mlp``) and ``libai_b200.ops.gated_mlp``: forward output and every gradient, from the exact bf16
inputs and upstream gradient.  The tensor-parallel nodes of ``ops/comm_gemm.py`` on one rank compute the same.

The bounds carry each kernel's error forward to first order, with the constants of ``tests/dense_ref.py``:

* a GEMM over ``K`` accumulates in fp32: ``K * ACC * (|A| @ |B|^T)``; a bias or residual added in its fp32 epilogue
  rounds once more, ``2^-24`` of the sum;
* a stored bf16 intermediate (the saved pre-activation, the bf16 ``h`` of an MLP, the bf16 ``dpre``) adds ``ROUND`` of
  itself, and a later step sees its error times that step's sensitivity to it;
* the activation and its derivative carry their approximation errors (``act_approx``); an error in the pre-activation
  moves ``act'`` by at most ``ACT_CURVATURE`` times it, and relu's derivative may flip where the pre-activation lies
  within its error of zero;
* a column sum over ``M`` rows (the bias gradient) accumulates in fp32: ``(M + 8) * ACC * sum |terms|``.

Each function returns ``{name: (reference, bound)}``; the bound of a gradient that lands in a parameter excludes the
rounding of its destination (bf16 ``.grad`` or fp32 ``main_grad``), which the caller adds.
"""
import torch

from tests import dense_ref as R

# max |act''(x)| over the reals: 2 phi(0) = 0.80 for gelu and gelu_tanh, 0.5 for silu, 1.702 * 0.5 = 0.85 for
# quick_gelu; 1 bounds them all (relu has no second derivative: its flips are handled separately)
ACT_CURVATURE = 1.0
U8 = R.ROUND[torch.bfloat16]
ACT_IDS = {None: 0, "none": 0, "gelu": 1, "gelu_tanh": 2, "relu": 3, "silu": 4, "quick_gelu": 5}


def _act_grad(gin, pre, e_pre, act):
    """``gin * act'(pre)`` rounded to bf16 when the kernel reads a pre-activation ``pre`` known to ``e_pre`` and an
    incoming gradient ``gin`` known to ``e_gin`` (callers add that part); returns (ref, bound without e_gin)."""
    if act == 0:
        return gin, torch.zeros_like(gin)
    _, d = R.act_ref(pre, act)
    _, ga = R.act_approx(pre, act)
    ref = gin * d
    if act == 3:
        # the sign of a pre-activation within its error (or a subnormal, flushed) of zero may come out either way
        flip = pre.abs() <= e_pre + 2.0 ** -126
        return ref, U8 * ref.abs() + gin.abs() * flip
    return ref, U8 * ref.abs() + gin.abs() * (ACT_CURVATURE * e_pre + ga) + R.FLUSH


def linear_ref(x, w, bias, gy, act):
    """``act(x @ w^T + bias)`` of ``linear`` on x [M, K], w [N, K], bias [N] or None, upstream gy [M, N]: y, gx, gw, gb."""
    act = ACT_IDS.get(act, act)
    X, W, G = x.double(), w.double(), gy.double()
    M, K = X.shape
    N = W.shape[0]
    pre = X @ W.t()
    e_acc = K * R.ACC * (X.abs() @ W.abs().t())
    if bias is not None:
        pre = pre + bias.double()
        e_acc = e_acc + 2.0 ** -24 * pre.abs()
    y, _ = R.act_ref(pre, act)
    fa, _ = R.act_approx(pre, act)
    lip = 1.0 if act in (0, 3) else R.ACT_LIPSCHITZ
    out = {"y": (y, U8 * y.abs() + lip * e_acc + fa + R.FLUSH)}
    # the backward reads the bf16 copy of the fp32 pre-activation; without an activation gy goes straight to the GEMMs
    dpre, e_dpre = _act_grad(G, pre, U8 * pre.abs() + e_acc, act)
    gx = dpre @ W
    out["gx"] = (gx, U8 * gx.abs() + (N * R.ACC * dpre.abs() + e_dpre) @ W.abs() + R.FLUSH)
    out["gw"] = (dpre.t() @ X, (M * R.ACC * dpre.abs() + e_dpre).t() @ X.abs() + R.FLUSH)
    out["gb"] = (dpre.sum(0), (M + 8) * R.ACC * dpre.abs().sum(0) + e_dpre.sum(0) + R.FLUSH)
    return out


def mlp_ref(x, w1, b1, w2, gy, act, b2=None, residual=None):
    """``act(x @ w1^T + b1) @ w2^T (+ b2 + residual)`` of ``mlp``: y, gx, gw1, gb1, gw2, gb2, gres."""
    act = ACT_IDS.get(act, act)
    X, W1, W2, G = x.double(), w1.double(), w2.double(), gy.double()
    M, K = X.shape
    Fh, N = W1.shape[0], W2.shape[0]
    pre = X @ W1.t()
    e_acc = K * R.ACC * (X.abs() @ W1.abs().t())
    if b1 is not None:
        pre = pre + b1.double()
        e_acc = e_acc + 2.0 ** -24 * pre.abs()
    h, _ = R.act_ref(pre, act)
    fa, _ = R.act_approx(pre, act)
    lip = 1.0 if act in (0, 3) else R.ACT_LIPSCHITZ
    e_h = U8 * h.abs() + lip * e_acc + fa                      # h is stored in bf16 and is the second GEMM's operand
    y = h @ W2.t()
    e_y = Fh * R.ACC * (h.abs() @ W2.abs().t()) + e_h @ W2.abs().t()
    if b2 is not None:
        y = y + b2.double()
    if residual is not None:
        y = y + residual.double()
    if b2 is not None or residual is not None:
        e_y = e_y + 2.0 ** -23 * y.abs()
    out = {"y": (y, U8 * y.abs() + e_y + R.FLUSH)}
    # dgrad_actgrad: dh = gy @ w2 in fp32, times act'(bf16 pre), rounded to bf16 once
    dh = G @ W2
    e_dh = N * R.ACC * (G.abs() @ W2.abs())
    dpre, e_dpre = _act_grad(dh, pre, U8 * pre.abs() + e_acc, act)
    _, d = R.act_ref(pre, act)
    # dh's own error passes through act' (and, where relu's derivative flips, through the flipped 1)
    e_dpre = e_dpre + d.abs() * e_dh + (e_dh if act == 3 else 0.0)
    gx = dpre @ W1
    out["gx"] = (gx, U8 * gx.abs() + (Fh * R.ACC * dpre.abs() + e_dpre) @ W1.abs() + R.FLUSH)
    out["gw1"] = (dpre.t() @ X, (M * R.ACC * dpre.abs() + e_dpre).t() @ X.abs() + R.FLUSH)
    out["gb1"] = (dpre.sum(0), (M + 8) * R.ACC * dpre.abs().sum(0) + e_dpre.sum(0) + R.FLUSH)
    out["gw2"] = (G.t() @ h, G.abs().t() @ (M * R.ACC * h.abs() + e_h) + R.FLUSH)
    out["gb2"] = (G.sum(0), (M + 8) * R.ACC * G.abs().sum(0) + R.FLUSH)
    out["gres"] = (G, torch.zeros_like(G))
    return out


def gated_mlp_ref(x, wg, wu, wd, gy, residual=None):
    """``(silu(x @ wg^T) * (x @ wu^T)) @ wd^T (+ residual)`` of the gated MLP: y, gx, gwg, gwu, gwd, gres.  The gate and
    up projections are stored in bf16, the SwiGLU reads them and stores h and its two gradients in bf16."""
    X, Wg, Wu, Wd, G = x.double(), wg.double(), wu.double(), wd.double(), gy.double()
    M, K = X.shape
    Fh, N = Wg.shape[0], Wd.shape[0]
    gate, up = X @ Wg.t(), X @ Wu.t()
    s = torch.sigmoid(gate)
    silu, dsilu = gate * s, s * (1 + gate * (1 - s))
    rel = R.EXPF_APPROX * (1 + gate.abs())
    e_g = U8 * gate.abs() + K * R.ACC * (X.abs() @ Wg.abs().t())
    e_u = U8 * up.abs() + K * R.ACC * (X.abs() @ Wu.abs().t())
    h = silu * up
    e_h = U8 * h.abs() + R.ACT_LIPSCHITZ * up.abs() * e_g + silu.abs() * e_u + h.abs() * rel
    y = h @ Wd.t()
    e_y = Fh * R.ACC * (h.abs() @ Wd.abs().t()) + e_h @ Wd.abs().t()
    if residual is not None:
        y = y + residual.double()
        e_y = e_y + 2.0 ** -23 * y.abs()
    out = {"y": (y, U8 * y.abs() + e_y + R.FLUSH)}
    dh = G @ Wd
    e_dh = U8 * dh.abs() + N * R.ACC * (G.abs() @ Wd.abs())
    dgate, dup = dh * up * dsilu, dh * silu
    e_dgate = (U8 * dgate.abs() + (up * dsilu).abs() * e_dh + (dh * dsilu).abs() * e_u + 0.5 * (dh * up).abs() * e_g
               + (dh * up).abs() * s * (1 - s) * (1 + 2 * gate.abs()) * rel)
    e_dup = U8 * dup.abs() + silu.abs() * e_dh + R.ACT_LIPSCHITZ * dh.abs() * e_g + dup.abs() * rel
    gx = dgate @ Wg + dup @ Wu
    out["gx"] = (gx, U8 * gx.abs() + (2 * Fh * R.ACC * dgate.abs() + e_dgate) @ Wg.abs()
                 + (2 * Fh * R.ACC * dup.abs() + e_dup) @ Wu.abs() + R.FLUSH)
    out["gwg"] = (dgate.t() @ X, (M * R.ACC * dgate.abs() + e_dgate).t() @ X.abs() + R.FLUSH)
    out["gwu"] = (dup.t() @ X, (M * R.ACC * dup.abs() + e_dup).t() @ X.abs() + R.FLUSH)
    out["gwd"] = (G.t() @ h, G.abs().t() @ (M * R.ACC * h.abs() + e_h) + R.FLUSH)
    out["gres"] = (G, torch.zeros_like(G))
    return out
