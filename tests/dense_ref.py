"""Element-by-element comparison of the dense kernels (GEMM and its epilogues, norms, cross-entropy, SwiGLU, column sums)
with fp64 references computed from the exact bf16 / fp32 inputs the kernel saw.

Every check is ``|out - ref| <= bound`` per element, with the bound written down here rather than tuned:

* one rounding of the output dtype at ``|ref|`` (``ROUND``);
* for a sum of ``n`` products (GEMM over K, a norm's row statistics over H, column sums over rows, the softmax
  denominator over V): ``n * 2^-23 * sum |terms|``, the worst case of fp32 accumulation with a factor 2 to spare;
* for an approximated function, its approximation error (``GELU_ERF_ABS``, ``TANH_APPROX_ABS``, ``EXPF_APPROX``);
* ``FLUSH``: results smaller than 2^-118 may come out as zero.  The kernels are built with --use_fast_math, so
  subnormal inputs and intermediates are flushed, and x / y is 0 for |y| > 2^126: x / (1 + e^-x) becomes 0 for
  x < -87.3, where the true value is below 1.1e-36.

A failing check reports the worst element: its index, value, reference and bound.
"""
import math

import torch

ROUND = {torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -23}
ACC = 2.0 ** -23            # per-term bound of an fp32 sum
FLUSH = 2.0 ** -118
# gelu_terms (common.cuh): Abramowitz-Stegun 7.1.26, |erf error| < 1.5e-7
GELU_ERF_ABS = 1.5e-7
# tanh.approx.f32: max |tanh_fast(u) - tanh(u)| over every fp32 u in [-16, 16] was 2^-16.93, measured once on an
# H100 80GB HBM3 (400 W power limit) with a kernel sweeping all fp32 bit patterns against the fp64 tanh; the constant
# rounds it up to the next power of two.
TANH_APPROX_ABS = 2.0 ** -16
# __expf(z) = ex2.approx(z * log2 e): max |__expf(z) / e^z - 1| / (1 + |z|) over every fp32 z in [-87, 88] was 2^-22.75
# in the same sweep (the |z| part is the rounding of z * log2 e); the constant rounds it up to the next power of two.
EXPF_APPROX = 2.0 ** -22
# max |act'(x)| over the reals is below 1.13 for gelu, gelu_tanh, silu and quick_gelu (1 for relu): an error in the
# pre-activation grows by at most this factor
ACT_LIPSCHITZ = 1.13

ACTS = {0: "none", 1: "gelu", 2: "gelu_tanh", 3: "relu", 4: "silu", 5: "quick_gelu"}
_SQRT_2_OVER_PI = math.sqrt(2.0 / math.pi)


class Mismatch(AssertionError):
    pass


def check(out, ref, bound, what=""):
    """Raise ``Mismatch`` unless ``|out - ref| <= bound`` at every element (a NaN anywhere fails)."""
    out64 = out.detach().double()
    ref = ref.to(out64.device, torch.float64)
    bound = torch.as_tensor(bound, dtype=torch.float64, device=out64.device).expand_as(ref)
    err = (out64 - ref).abs()
    ok = err <= bound
    if bool(ok.all()):
        return
    # worst element: any NaN first, otherwise the largest excess over the bound relative to the bound
    score = torch.where(ok, torch.zeros_like(err), (err - bound) / (bound + FLUSH))
    score = torch.where(torch.isnan(score), torch.full_like(score, math.inf), score)
    flat = int(torch.argmax(score))
    idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(flat), ref.shape)) if ref.dim() else ()
    raise Mismatch(f"{what}: {int((~ok).sum())} of {ok.numel()} elements outside the bound; worst at {idx}: "
                   f"out={float(out64[idx])!r} ref={float(ref[idx])!r} bound={float(bound[idx]):.3e}")


# ---------------------------------------------------------------------------------------------------------- activations
def act_ref(v, act):
    """fp64 activation and its derivative."""
    if act == 0:
        return v, torch.ones_like(v)
    if act == 1:
        cdf = 0.5 * torch.erfc(-v / math.sqrt(2.0))
        return v * cdf, cdf + v * torch.exp(-0.5 * v * v) / math.sqrt(2.0 * math.pi)
    if act == 2:
        u = _SQRT_2_OVER_PI * (v + 0.044715 * v ** 3)
        t = torch.tanh(u)
        du = _SQRT_2_OVER_PI * (1.0 + 3.0 * 0.044715 * v * v)
        return 0.5 * v * (1.0 + t), 0.5 * (1.0 + t) + 0.5 * v * (1.0 - t * t) * du
    if act == 3:
        return torch.relu(v), (v > 0).double()
    k = 1.0 if act == 4 else 1.702
    s = torch.sigmoid(k * v)
    return v * s, s * (1.0 + k * v * (1.0 - s))


def act_approx(v, act):
    """Bounds of the approximation errors of act(v) and act'(v) (fp64 ``v``): the fast erf, tanh and exp of common.cuh."""
    a = v.abs()
    if act == 1:
        return 0.5 * a * GELU_ERF_ABS, 0.5 * GELU_ERF_ABS + a * torch.exp(-0.5 * v * v) * 2.0 ** -21
    if act == 2:
        du = _SQRT_2_OVER_PI * (1.0 + 3.0 * 0.044715 * v * v)
        return 0.5 * a * TANH_APPROX_ABS, TANH_APPROX_ABS * (0.5 + a * du)
    if act in (4, 5):
        k = 1.0 if act == 4 else 1.702
        y, _ = act_ref(v, act)
        s = torch.sigmoid(k * v)
        rel = EXPF_APPROX * (1.0 + k * a)      # relative error of e^{-kv}, hence of the sigmoid
        return y.abs() * rel, s * (1.0 - s) * (1.0 + 2.0 * k * a) * rel
    return torch.zeros_like(v), torch.zeros_like(v)


# ---------------------------------------------------------------------------------------------------------------- GEMM
def gemm_operands(a, b, layout):
    """(A [M, K], B [N, K]) of ``ext.gemm``'s layouts 0: a[M,K] b[N,K]; 1: a[M,K] b[K,N]; 2: a[K,M] b[K,N]."""
    if layout == 0:
        return a, b
    if layout == 1:
        return a, b.t()
    return a.t(), b.t()


def check_gemm(out, A, B, what, *, bias=None, act=0, pre=None, residual=None, base=None, dpre=None, chunk=1024,
               acc_bound=None):
    """``out`` against ``A @ B^T`` in fp64, in row chunks of ``chunk``.

    ``bias`` [N] and ``act`` apply the epilogue act(acc + bias); ``pre`` is then the bf16 copy of acc + bias.
    ``residual`` [M, N]: out = acc + bias + residual.  ``base`` [M, N]: out = base + acc (fp32 accumulation; base is the
    content of the buffer before the call).  ``dpre`` [M, N]: out = acc * act'(dpre).  ``acc_bound``: a function of the
    row slice giving the accumulation error bound of those rows, for accumulators that are not fp32."""
    M, K = A.shape
    for r0 in range(0, M, chunk):
        a = A[r0:r0 + chunk].double()
        acc = a @ B.double().t()
        rows = slice(r0, r0 + chunk)
        kterm = K * ACC * (a.abs() @ B.double().abs().t()) if acc_bound is None else acc_bound(rows)
        v, vbound = acc, kterm
        if bias is not None:
            v = v + bias.double()
            vbound = vbound + 2.0 ** -24 * v.abs()
        if residual is not None:
            v = v + residual[rows].double()
            vbound = vbound + 2.0 ** -24 * v.abs()
        if base is not None:
            v = v + base[rows].double()
            vbound = vbound + 2.0 ** -24 * v.abs()
        if dpre is not None:
            d = dpre[rows].double()
            _, grad = act_ref(d, act)
            _, gapprox = act_approx(d, act)
            ref = acc * grad
            bound = grad.abs() * kterm + acc.abs() * gapprox
        else:
            ref, _ = act_ref(v, act)
            fapprox, _ = act_approx(v, act)
            lip = 1.0 if act in (0, 3) else ACT_LIPSCHITZ
            bound = lip * vbound + fapprox
            if pre is not None:
                check(pre[rows], v, ROUND[pre.dtype] * v.abs() + vbound + FLUSH, what + " (pre-activation)")
        check(out[rows], ref, ROUND[out.dtype] * ref.abs() + bound + FLUSH, what)


# --------------------------------------------------------------------------------------------------------------- norms
def norm_stats(x, rms, eps):
    xd = x.double()
    mean = torch.zeros(x.shape[0], 1, dtype=torch.float64, device=x.device) if rms else xd.mean(1, keepdim=True)
    var = ((xd - mean) ** 2).mean(1, keepdim=True)
    return mean, torch.rsqrt(var + eps)


def check_norm_fwd(y, mean_k, rstd_k, x, gamma, beta, rms, eps, what):
    H = x.shape[1]
    c = (H + 8) * ACC                                       # row sums over H, rsqrt.approx, the few fp32 roundings
    xd = x.double()
    mean, rstd = norm_stats(x, rms, eps)
    xh = (xd - mean) * rstd
    g = gamma.double()
    ref = xh * g + (0.0 if beta is None else beta.double())
    dmean = 0.0 if rms else c * xd.abs().mean(1, keepdim=True)
    dxh = rstd * dmean + c * xh.abs()
    check(y, ref, ROUND[y.dtype] * ref.abs() + g.abs() * dxh + c * ref.abs() + FLUSH, what + " y")
    check(rstd_k.double()[:, None], rstd, c * rstd, what + " rstd")
    if not rms:
        check(mean_k.double()[:, None], mean, dmean, what + " mean")


def norm_bwd_ref(gy, x, gamma, rms, eps):
    """fp64 (gx, dγ, dβ) and their bounds."""
    H, R = x.shape[1], x.shape[0]
    c = (H + 8) * ACC
    xd, gd, g = x.double(), gy.double(), gamma.double()
    mean, rstd = norm_stats(x, rms, eps)
    xh = (xd - mean) * rstd
    gw = gd * g
    s1 = torch.zeros_like(mean) if rms else gw.mean(1, keepdim=True)
    s2 = (gw * xh).mean(1, keepdim=True)
    gx = rstd * (gw - s1 - xh * s2)
    dmean = 0.0 if rms else c * xd.abs().mean(1, keepdim=True)
    dxh = rstd * dmean + c * xh.abs()                       # error of the kernel's x̂ (its mean / rstd are fp32)
    s1e = 0.0 if rms else c * gw.abs().mean(1, keepdim=True)
    s2e = c * (gw * xh).abs().mean(1, keepdim=True) + (gw.abs() * dxh).mean(1, keepdim=True)
    gx_b = rstd * (c * (gw.abs() + xh.abs() * s2.abs()) + s1e + dxh * s2.abs() + xh.abs() * s2e) + c * gx.abs()
    dg = (gd * xh).sum(0)
    dg_b = (R + 8) * ACC * (gd * xh).abs().sum(0) + (gd.abs() * dxh).sum(0)
    db = gd.sum(0)
    db_b = (R + 8) * ACC * gd.abs().sum(0)
    return (gx, gx_b), (dg, dg_b), (db, db_b)


# ------------------------------------------------------------------------------------------------------ cross-entropy
def ce_ref(logits, labels, vocab_start):
    """fp64 (loss, lse) of one vocabulary shard as the native op computes it (a label outside the shard contributes a
    target logit of 0), and the bound of the kernel's lse."""
    V = logits.shape[1]
    ld = logits.double()
    lse = torch.logsumexp(ld, 1)
    local = labels - vocab_start
    inside = (local >= 0) & (local < V)
    tgt = torch.where(inside, ld.gather(1, local.clamp(0, V - 1)[:, None])[:, 0], torch.zeros_like(lse))
    m = ld.max(1).values
    span = torch.where(torch.isfinite(ld), (ld - m[:, None]).abs(), torch.zeros_like(ld)).max(1).values
    # each of the kernel's 256 threads sums V / 256 terms and rescales its sum at most once per term; then two
    # shuffle trees, each with one rescale
    lse_b = (V / 256 + 16) * ACC + EXPF_APPROX * (V / 256 + 3 + 2 * span) + 2.0 ** -22 * (lse.abs() + m.abs())
    return lse - tgt, lse, lse_b, local, inside


def check_ce(loss, dlogits, logits, labels, vocab_start, gloss, what):
    ref_loss, lse, lse_b, local, inside = ce_ref(logits, labels, vocab_start)
    check(loss, ref_loss, ROUND[torch.float32] * ref_loss.abs() + lse_b + 2.0 ** -23 * tgt_abs(logits, local, inside)
          + FLUSH, what + " loss")
    z = logits.double() - lse[:, None]
    p = torch.exp(z)
    ref = p.clone()
    rows = torch.nonzero(inside)[:, 0]
    ref[rows, local[rows]] -= 1.0
    g = gloss.double()[:, None]
    ref = ref * g
    zabs = torch.where(torch.isfinite(z), z.abs(), torch.zeros_like(z))
    bound = g.abs() * p * (lse_b[:, None] + EXPF_APPROX * (1.0 + zabs) + 2.0 ** -22 * zabs)
    check(dlogits, ref, ROUND[dlogits.dtype] * ref.abs() + bound + FLUSH, what + " dlogits")


def tgt_abs(logits, local, inside):
    V = logits.shape[1]
    t = logits.double().gather(1, local.clamp(0, V - 1)[:, None])[:, 0].abs()
    return torch.where(inside, t, torch.zeros_like(t))


# -------------------------------------------------------------------------------------------------------------- SwiGLU
def swiglu_ref(gate, up, gy=None):
    """fp64 silu(gate) * up and its bound; with ``gy`` also (d gate, d up) and their bounds."""
    g, u = gate.double(), up.double()
    s = torch.sigmoid(g)
    y = g * s * u
    rel = EXPF_APPROX * (1.0 + g.abs())
    y_b = y.abs() * (rel + 4 * ACC)
    if gy is None:
        return y, y_b
    d = gy.double()
    du = d * g * s
    dg = d * u * s * (1.0 + g * (1.0 - s))
    du_b = du.abs() * (rel + 4 * ACC)
    dg_b = (d * u).abs() * s * (1.0 - s) * (1.0 + 2.0 * g.abs()) * rel + dg.abs() * 6 * ACC
    return y, y_b, dg, dg_b, du, du_b
