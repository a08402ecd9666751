"""Element-by-element references for the kernels of a training step that tests/dense_ref.py and tests/attention_ref.py
leave out: the fused Adam / AdamW update, the embedding gather and its scatter-add backward, the E4M3 quantiser and the
fp8 forward GEMM.  Each reference takes the exact fp32 / bf16 / E4M3 inputs the kernel saw; the checks reuse
``dense_ref.check``, which reports the worst element with its index, value, reference and bound.

The kernels are built with --use_fast_math, so:

* ``x / y`` is div.approx.ftz.f32: within 2 ulp (``DIV_APPROX``) for |y| in [2^-126, 2^126];
* ``sqrtf`` is sqrt.approx.ftz.f32 (MUFU.SQRT), ``SQRT_APPROX``;
* subnormal inputs and results are flushed to zero: every flushed value is below 2^-126 (``TINY`` covers a few).

Additions and multiplications stay correctly rounded (``F32_RN`` each); a multiply-add may be fused, which only removes
a rounding.  The embedding kernels are exact: the forward is a bit copy, the backward a fixed-order fp32 sum that an
fp32 emulation reproduces bit for bit.
"""
import torch

from tests.dense_ref import ACC, check, check_gemm

F32_RN = 2.0 ** -24                 # one round-to-nearest fp32 operation, relative
DIV_APPROX = 2.0 ** -22             # div.approx.f32: 2 ulp = 2 * 2^-23 relative (PTX ISA, |y| in [2^-126, 2^126])
# sqrt.approx.ftz.f32: max |sqrt.approx(x) / sqrt(x) - 1| over every positive normal fp32 x was 2^-23.25 (1.0001e-7),
# measured once by dev/measure_sqrt_approx.py on an H100 80GB HBM3 (400 W power limit); the constant rounds it up to the
# next power of two.
SQRT_APPROX = 2.0 ** -23
TINY = 2.0 ** -124                  # a few flushed subnormals
E4M3_MAX = 448.0
# accumulation of the fp8 GEMM: see FP8_ACC and fp8_acc_bound
FP8_KSTEP = 32                      # E4M3 elements per wgmma (one k-step)


def f32(x):
    """The fp32 value of a Python float, as the bindings' ``(float)`` casts give it."""
    return float(torch.tensor(x, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------------------ Adam
def adam_hparams(lr, b1, b2, eps, wd, step, bias_correction=True):
    """Hyperparameters of one step as the kernel receives them: the optimizer computes the bias corrections in double,
    the binding casts every value to fp32."""
    bc1, bc2 = (1.0 - b1 ** step, 1.0 - b2 ** step) if bias_correction else (1.0, 1.0)
    return dict(lr=f32(lr), b1=f32(b1), b2=f32(b2), eps=f32(eps), wd=f32(wd), bc1=f32(bc1), bc2=f32(bc2))


def adam_moments_ref(master, grad, m, v, scale, hp, decoupled):
    """fp64 new (m, v) from the fp32 state, with their bounds."""
    P, G, M, V = (t.double() for t in (master, grad, m, v))
    c1, c2 = f32(1.0 - hp["b1"]), f32(1.0 - hp["b2"])     # the kernel's fp32 1 - b (exact in double, then RNE)
    gs = G * scale
    wdp = hp["wd"] * P
    g = gs if decoupled else gs + wdp
    # g: the product (and with coupled decay, wd * p and the sum), one rounding each
    g_err = ACC * (gs.abs() + (0.0 if decoupled else wdp.abs())) + TINY
    t1, t2 = hp["b1"] * M, c1 * g
    m_ref = t1 + t2
    m_err = c1 * g_err + ACC * (t1.abs() + t2.abs()) + TINY
    u1, u2 = hp["b2"] * V, c2 * g * g
    v_ref = u1 + u2
    v_err = c2 * (2.0 * g.abs() * g_err + g_err * g_err) + 2 * ACC * (u1.abs() + u2.abs()) + TINY
    return (m_ref, m_err), (v_ref, v_err)


def adam_master_ref(master, m_new, v_new, hp, decoupled):
    """fp64 new master from the old master and the kernel's OWN new moments (the kernel divides the fp32 values it
    stores), with its bound: the divisions m / bc1, v / bc2 and m̂ / (√v̂ + ε), the square root, then the fp32 roundings
    of + ε, + wd·p, lr·u and p − lr·u."""
    P, M, V = master.double(), m_new.double(), v_new.double()
    den = torch.sqrt(V / hp["bc2"]) + hp["eps"]
    r = (M / hp["bc1"]) / den
    # first-order relative errors: m / bc1, v / bc2 (halved by the root), the root, + eps, the last division; the
    # factor covers their products
    r_rel = (3 * DIV_APPROX + DIV_APPROX / 2 + SQRT_APPROX + F32_RN) * (1 + 2.0 ** -20)
    wdp = hp["wd"] * P if decoupled else torch.zeros_like(P)
    u = r + wdp
    u_err = r.abs() * r_rel + ACC * (wdp.abs() + u.abs()) + TINY
    p_ref = P - hp["lr"] * u
    p_err = hp["lr"] * u_err + ACC * hp["lr"] * u.abs() + F32_RN * p_ref.abs() + TINY
    return p_ref, p_err


def check_adam(new, old, scale, hp, decoupled, what, lp=None):
    """``new`` = (master, m, v) after one kernel step from ``old`` = (master, grad, m, v); ``scale`` the fp32 value of the
    device multiplier.  ``lp``: the low-precision copy, which must be the round-to-nearest-even of the new master."""
    master, grad, m, v = old
    (m_ref, m_err), (v_ref, v_err) = adam_moments_ref(master, grad, m, v, scale, hp, decoupled)
    check(new[1], m_ref, m_err, what + " m")
    check(new[2], v_ref, v_err, what + " v")
    p_ref, p_err = adam_master_ref(master, new[1], new[2], hp, decoupled)
    check(new[0], p_ref, p_err, what + " master")
    if lp is not None:
        check_lp(lp, new[0], what)


def check_lp(lp, master, what):
    """Exactly the round-to-nearest-even of ``master`` in lp's dtype (bf16 or fp16), bit for bit."""
    want = master.to(lp.dtype)
    bits = torch.int16
    same = lp.view(bits) == want.view(bits)
    if not bool(same.all()):
        i = int(torch.nonzero(~same)[0, 0])
        raise AssertionError(f"{what} lp_out: {int((~same).sum())} of {same.numel()} elements are not the RNE of the "
                             f"master; first at {i}: out={float(lp[i])!r} want={float(want[i])!r} "
                             f"master={float(master[i])!r}")


# ------------------------------------------------------------------------------------------------------- embedding
def embedding_fwd_ref(ids, table, vocab_start):
    """The rows of ``ids - vocab_start`` with a zero row (+0.0) for every id outside the shard, negative ids included."""
    rows = table.shape[0]
    local = ids.reshape(-1) - vocab_start
    inside = (local >= 0) & (local < rows)
    out = table[local.clamp(0, rows - 1)]
    return torch.where(inside[:, None], out, torch.zeros_like(out))


def assert_no_subnormal_sums(*ts):
    """The backward's fp32 adds flush subnormal results.  With every nonzero |gy| and |grad| >= 2^-100, each partial sum
    is 0 or a multiple of 2^-123, hence normal, so no flush can act and the plain fp32 emulation below is exact."""
    for t in ts:
        a = t.float().abs()
        assert bool(((a == 0) | (a >= 2.0 ** -100)).all()), "inputs would make subnormal partial sums"


def embedding_bwd_ref(ids, gy, grad, vocab_start):
    """fp32 emulation of embedding_bwd_kernel: the ids sorted stably, every run of equal ids summed in token order into
    acc = 0, then grad[row] += acc.  Returns the new grad (a copy)."""
    assert_no_subnormal_sums(gy, grad)
    rows, H = grad.shape
    flat = ids.reshape(-1)
    T = flat.numel()
    out = grad.clone()
    if T == 0:
        return out
    sorted_ids, order = torch.sort(flat, stable=True)
    first = torch.ones(T, dtype=torch.bool, device=flat.device)
    first[1:] = sorted_ids[1:] != sorted_ids[:-1]
    run = torch.cumsum(first.long(), 0) - 1
    start = torch.nonzero(first)[:, 0]
    rank = torch.arange(T, device=flat.device) - start[run]
    acc = torch.zeros(start.numel(), H, dtype=torch.float32, device=grad.device)
    g = gy.float()
    for k in range(int(rank.max()) + 1):
        sel = torch.nonzero(rank == k)[:, 0]
        r = run[sel]                     # distinct runs: one fp32 add per element
        acc[r] = acc[r] + g[order[sel]]
    local = sorted_ids[start] - vocab_start
    inside = (local >= 0) & (local < rows)
    dst = local[inside]
    out[dst] = out[dst] + acc[inside]
    return out


def check_bits(out, want, what):
    """Bitwise equality (so -0.0 and +0.0 differ), reporting the first differing element."""
    ib = {torch.bfloat16: torch.int16, torch.float16: torch.int16, torch.float32: torch.int32}[out.dtype]
    assert out.dtype == want.dtype and out.shape == want.shape, (what, out.dtype, want.dtype, out.shape, want.shape)
    same = out.view(ib) == want.view(ib)
    if not bool(same.all()):
        idx = tuple(int(i) for i in torch.nonzero(~same)[0])
        raise AssertionError(f"{what}: {int((~same).sum())} of {same.numel()} elements differ; first at {idx}: "
                             f"out={float(out[idx])!r} want={float(want[idx])!r}")


# ------------------------------------------------------------------------------------------------------ quantiser
def e4m3(x):
    """Round-to-nearest-even E4M3 of fp64 values already inside [-448, 448] (torch casts through fp32; the callers'
    brackets are wide enough that this does not matter), as fp64."""
    return x.float().to(torch.float8_e4m3fn).double()


def quant_ref(x):
    """(amax, deq, deq bound, q_lo, q_hi): q must lie in [q_lo, q_hi] element by element.

    The kernel reads subnormal bf16 inputs as zero (FTZ); ``fmaxf`` ignores NaN; amax is floored at 1e-12, so an
    all-zero tensor gives q = 0 and a finite deq.  scale = 448 / amax is correctly rounded (``__fdiv_rn``), the product
    x * scale is one fp32 rounding, and the cast saturates to ±448.  The bracket widens x * 448 / amax by 2^-22
    relative, which covers both roundings, and is cast after clamping (PyTorch's cast is not relied on to saturate)."""
    xf = x.float().reshape(-1)
    xf = torch.where(xf.abs() < 2.0 ** -126, torch.zeros_like(xf), xf)
    a = torch.nan_to_num(xf.abs(), nan=0.0)
    amax = float(a.max()) if a.numel() else 0.0
    amax_eff = max(amax, f32(1e-12))
    deq = amax_eff / E4M3_MAX
    xs = xf.double() * (E4M3_MAX / amax_eff)
    lo = torch.minimum(xs * (1 - 2.0 ** -22), xs * (1 + 2.0 ** -22)).clamp(-E4M3_MAX, E4M3_MAX)
    hi = torch.maximum(xs * (1 - 2.0 ** -22), xs * (1 + 2.0 ** -22)).clamp(-E4M3_MAX, E4M3_MAX)
    return amax, deq, DIV_APPROX * deq, e4m3(lo), e4m3(hi)


def check_quant(q, deq, x, what):
    amax, deq_ref, deq_b, q_lo, q_hi = quant_ref(x)
    check(deq.reshape(1), torch.tensor([deq_ref]), deq_b, what + " deq")
    qd = q.reshape(-1).double()
    check(qd, (q_lo + q_hi) / 2, (q_hi - q_lo) / 2, what + " q")
    xf = x.float().reshape(-1)
    at_max = (xf.abs() == amax) & (amax >= 2.0 ** -126)
    if bool(at_max.any()):
        check(qd[at_max], torch.sign(xf[at_max].double()) * E4M3_MAX, 0.0, what + " q at ±amax")
    return amax


# ------------------------------------------------------------------------------------------------------- fp8 GEMM
# The fp8 wgmma does not accumulate in full fp32.  dev/measure_fp8_acc.py, on an H100 80GB HBM3 (400 W power limit):
# a product 2^-12 of the large ones it is summed with was lost in some probes and one 2^-14 in all, whether the
# products met inside one 32-wide k-step, across k-steps or across k-blocks; lost values came out as 0 (truncation).
# So every addition may drop what lies below 2^-11 of the largest magnitude involved.  For comparison, with random
# E4M3 operands 13.6 % (K = 1024) and 27.4 % (K = 4096) of the outputs differ from the correctly rounded bf16 result,
# against 0.00 % and 0.01 % for the bf16 GEMM (fp32 accumulator) on the same values.
FP8_ACC = 2.0 ** -11


def fp8_acc_bound(A, B, rows):
    """Accumulation error bound of rows ``rows`` of A @ B^T (fp64, E4M3 values times the dequantisation scale).

    Model: each 32-wide k-step adds its products to the accumulator and loses at most 2 * FP8_ACC * (|partial sum
    before it| + sum of |its products|).  This follows the measurement above but is not a worst case: a step of many
    products, each just above the truncation point of the largest, could lose more."""
    a = A[rows].double()
    b = B.double()
    K = a.shape[1]
    s = torch.zeros(a.shape[0], b.shape[0], dtype=torch.float64, device=a.device)
    bound = torch.zeros_like(s)
    for k0 in range(0, K, FP8_KSTEP):
        ak, bk = a[:, k0:k0 + FP8_KSTEP], b[:, k0:k0 + FP8_KSTEP]
        bound += 2 * FP8_ACC * (s.abs() + ak.abs() @ bk.abs().t())
        s += ak @ bk.t()
    return bound + F32_RN * s.abs()          # and the fp32 product by deq_x * deq_w


def fp8_alpha(deq_x, deq_w):
    """The kernel's fp32 product deq_x * deq_w (correctly rounded, as fp32 multiplication is)."""
    return float(deq_x.float().cpu() * deq_w.float().cpu())


def check_fp8_gemm(out, xq, wq, deq_x, deq_w, what, **epilogue):
    """``out`` of linear_fp8_fwd against Σ qx·qw in fp64 (each E4M3 product is exact) times fp32(deq_x·deq_w), then
    the epilogues of ``dense_ref.check_gemm`` (bias, act with its pre-activation copy, residual)."""
    A = xq.double() * fp8_alpha(deq_x, deq_w)
    B = wq.double()
    check_gemm(out, A, B, what, acc_bound=lambda rows: fp8_acc_bound(A, B, rows), **epilogue)


# ----------------------------------------------------------------------------------------------------- GEMM tiles
# mirror of the tile-width heuristic of gemm_impl (gemm_sm90.cu) for the forward GEMMs (bf16 epilogue, no comm)
TILE_CANDS = (256, 192, 128, 64)
TILE_PER_COL = {256: 0.00286, 192: 0.00272, 128: 0.00332, 64: 0.00414}
TILE_EPILOGUE_BF16 = {256: 54.0, 192: 24.4, 128: 11.6, 64: 4.2}
BLOCK_M, BLOCK_K = 128, 64


def pick_bn(M, N, K, sms=132, fp8=False):
    """Tile width the heuristic picks; ``K`` in elements of the operands (E4M3 when ``fp8``: the kernel sees K / 2
    bf16 columns)."""
    if fp8:
        K //= 2
    m_blocks = (M + BLOCK_M - 1) // BLOCK_M
    k_blocks = (K + BLOCK_K - 1) // BLOCK_K
    best, bn = 1e30, 0
    for c in TILE_CANDS:
        if c > 64 and N <= c // 2:
            continue
        tiles = m_blocks * ((N + c - 1) // c)
        waves = (tiles + sms - 1) // sms
        cost = waves * (c * k_blocks * TILE_PER_COL[c] + TILE_EPILOGUE_BF16[c])
        if cost < best - 1e-9:
            best, bn = cost, c
    return bn

