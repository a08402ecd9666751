"""Functional front-end of the hot operators (autograd wrappers).

Each function dispatches to the native sm_90a kernels for CUDA tensors and to the PyTorch
reference otherwise (see :mod:`libai_b200.ops`).  The reference call sites these replace are the
OneFlow fused ops: ``flow._C.layer_norm_affine`` / ``rms_norm``
(libai/layers/layer_norm.py:78-131), ``fused_bias_add_gelu`` (libai/layers/mlp.py:95),
``fused_bias_add_dropout`` (libai/layers/mlp.py:104, attention.py:265),
``fused_scale_mask_softmax_dropout`` / ``fused_scale_tril_softmax_mask_scale``
(libai/layers/attention.py:220-246), ``sparse_softmax_cross_entropy``
(libai/layers/cross_entropy.py:44) and the matmuls in libai/layers/linear.py:123-157.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn.functional as F

from . import count_launch, load_ext, use_native
from .. import ops

# --------------------------------------------------------------------------------------
# activations (reference math)
# --------------------------------------------------------------------------------------
_SQRT_2_OVER_PI = 0.7978845608028654


def gelu_ref(x, approximate: str = "none"):
    return F.gelu(x, approximate=approximate)


ACT_NONE, ACT_GELU, ACT_GELU_TANH, ACT_RELU, ACT_SILU, ACT_QUICK_GELU = 0, 1, 2, 3, 4, 5
_ACT_IDS = {
    None: ACT_NONE,
    "none": ACT_NONE,
    "gelu": ACT_GELU,
    "gelu_tanh": ACT_GELU_TANH,
    "relu": ACT_RELU,
    "silu": ACT_SILU,
    "quick_gelu": ACT_QUICK_GELU,
}


def _act_ref(x, act):
    if act in (None, "none"):
        return x
    if act == "gelu":
        return F.gelu(x)
    if act == "gelu_tanh":
        return F.gelu(x, approximate="tanh")
    if act == "relu":
        return F.relu(x)
    if act == "silu":
        return F.silu(x)
    if act == "quick_gelu":
        return x * torch.sigmoid(1.702 * x)
    raise ValueError(act)


# --------------------------------------------------------------------------------------
# GEMM: y = x @ w^T (+ bias) (+ activation)
# --------------------------------------------------------------------------------------
def _gemm_ok(x: torch.Tensor, w: torch.Tensor) -> bool:
    """Shapes/dtypes the wgmma kernel accepts (TMA needs 16-byte aligned rows)."""
    return (
        x.dtype == torch.bfloat16
        and w.dtype == torch.bfloat16
        and x.shape[-1] % 8 == 0
        and w.shape[0] % 8 == 0
        and x.numel() > 0
    )



_FP8_WEIGHTS: dict = {}


def _fp8_ok(x2: torch.Tensor, w: torch.Tensor) -> bool:
    return ops.fp8_enabled() and x2.shape[-1] % 16 == 0 and w.is_contiguous()


def _fp8_weight(ext, w):
    """E4M3 copy of a weight + its dequantisation scale, cached until the optimizer rewrites the parameters
    (``ops.bump_fp8_weight_epoch``) or the tensor is modified through PyTorch (``_version``).  Inside a CUDA-graph
    capture the quantisation is always issued (and captured): a cached tensor would pin stale addresses."""
    if torch.cuda.is_current_stream_capturing():
        count_launch(2)
        return ext.quantize_e4m3(w.detach())
    key = (ops.fp8_weight_epoch(), w._version, w.data_ptr())
    hit = _FP8_WEIGHTS.get(id(w))
    if hit is not None and hit[0] == key:
        return hit[1], hit[2]
    wq, dw = ext.quantize_e4m3(w.detach())
    count_launch(2)
    _FP8_WEIGHTS[id(w)] = (key, wq, dw)
    return wq, dw


def _linear_fwd_any(ext, x2, w, bias, act_id, need_pre, residual=None):
    """Forward GEMM of a linear layer: E4M3 operands when the fp8 path is on, bf16 otherwise."""
    if _fp8_ok(x2, w):
        xq, dx = ext.quantize_e4m3(x2)
        wq, dw = _fp8_weight(ext, w)
        count_launch(3)
        return ext.linear_fp8_fwd(xq, wq, dx, dw, bias, act_id, need_pre, residual)
    count_launch()
    if residual is not None:
        return ext.linear_bias_residual(x2, w, bias, residual), None
    return ext.linear_fwd(x2, w, bias, act_id, need_pre)


def _main_grad(p):
    """``p.main_grad`` when it is an fp32 contiguous tensor (the optimizers' slice of their flat gradient buffer), else
    None.  A native backward accumulates a parameter's gradient into this tensor and sets
    ``p.grad_added_to_main_grad``, or, without it, returns the gradient to autograd in ``p``'s dtype; CUDA-graph
    capture and ``sync_gradients`` rely on that choice."""
    mg = getattr(p, "main_grad", None)
    return mg if mg is not None and mg.dtype == torch.float32 and mg.is_contiguous() else None


def _fused_bias_grad_target(bias):
    """Where a dgrad GEMM epilogue may add the column sums of its result as ``bias``' gradient: ``_main_grad(bias)``
    when ``ops.fused_bias_grad()`` is on and that slice is 16-byte aligned (the tensor-parallel epilogue adds into it
    with vector reductions), else None."""
    if not ops.fused_bias_grad():
        return None
    mg = _main_grad(bias)
    return mg if mg is not None and mg.data_ptr() % 16 == 0 else None


def _bias_grad(ext, g2, bias):
    """Column sums of ``g2`` as the gradient of ``bias``: accumulated straight into ``bias.main_grad`` (fp32 slice of
    the optimizer's flat gradient buffer) when the parameter owns one – no temporary, no bf16 round trip, no
    per-parameter add kernel later – otherwise returned as a tensor for autograd."""
    count_launch()
    main_grad = _main_grad(bias)
    if main_grad is not None:
        ext.colsum(g2, main_grad)
        bias.grad_added_to_main_grad = True
        return None
    return ext.colsum(g2).to(bias.dtype)


def _weight_grad(ext, g, x, w):
    """``gᵀ · x`` as the gradient of ``w``: a ``TN`` split-K GEMM accumulating in fp32 straight into ``w.main_grad``
    when the parameter owns one (gradient-accumulation fusion), otherwise returned to autograd in ``w``'s dtype."""
    count_launch()
    main_grad = _main_grad(w)
    if main_grad is not None:
        ext.gemm(g, x, 2, None, main_grad, True, torch.float32)
        w.grad_added_to_main_grad = True
        return None
    return ext.gemm(g, x, 2, None, None, False, torch.float32).to(w.dtype)


class _LinearFn(torch.autograd.Function):
    """Native linear: fwd ``NT`` GEMM with fused bias/activation epilogue, dgrad ``NN`` GEMM, wgrad through
    :func:`_weight_grad`.  With ``residual`` (no activation) the epilogue also adds it, and its gradient is ``gy``."""

    @staticmethod
    def forward(ctx, x, w, bias, act, residual=None):
        ext = load_ext()
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        # the backward runs whenever any input needs a gradient, and every gradient (the bias' alone included) goes
        # through the activation backward, which reads the pre-activation
        need_pre = act not in (None, "none") and any(ctx.needs_input_grad[:3])
        res2 = None if residual is None else residual.reshape(-1, w.shape[0]).contiguous()
        y, pre = _linear_fwd_any(ext, x2, w, bias, _ACT_IDS[act], need_pre, res2)
        ctx.act = act
        ctx.bias_param = bias
        ctx.has_res = residual is not None
        ctx.save_for_backward(x2, w, pre if need_pre else None)
        ctx.x_shape = x.shape
        return y.view(*x.shape[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, gy):
        ext = load_ext()
        x2, w, pre = ctx.saved_tensors
        g2 = gy.reshape(-1, gy.shape[-1]).contiguous()
        if ctx.act not in (None, "none"):
            g2 = ext.act_bwd(g2, pre, _ACT_IDS[ctx.act])
            count_launch()
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            gx = ext.gemm(g2, w, 1, None, None, False, torch.bfloat16)  # NN: [M,N]x[N,K]
            count_launch()
            gx = gx.view(ctx.x_shape)
        if ctx.needs_input_grad[1]:
            gw = _weight_grad(ext, g2, x2, w)
        if ctx.needs_input_grad[2]:
            gb = _bias_grad(ext, g2, ctx.bias_param)
        return gx, gw, gb, None, (gy if ctx.has_res else None)


def reject_quantized_weight(what: str, *weights) -> None:
    """FP8 (E4M3) weights read back only with their row scales, and packed INT4 weights (uint8) only with their group
    scales and zeros, which the bf16 GEMM entries do not take: they raise instead of multiplying the bytes
    (:func:`linear_fp8w` and :func:`linear_int4w` are the entries for such weights)."""
    for w in weights:
        if w is not None and w.dtype == torch.float8_e4m3fn:
            raise TypeError(f"{what}: float8_e4m3fn weight; FP8 weights take OF.linear_fp8w with their row scales")
        if w is not None and w.dtype == torch.uint8:
            raise TypeError(f"{what}: packed INT4 (uint8) weight; INT4 weights take OF.linear_int4w with their group "
                            "scales and zeros")


def linear(x, w, bias=None, act: Optional[str] = None):
    """``act(x @ w.T + bias)``; ``w`` is ``[out, in]``."""
    reject_quantized_weight("linear", w)
    if use_native(x, w) and _gemm_ok(x, w):
        return _LinearFn.apply(x, w, bias, act)
    y = F.linear(x, w.to(x.dtype) if w.dtype != x.dtype else w, None if bias is None else bias.to(x.dtype))
    return _act_ref(y, act)



class _MLPFn(torch.autograd.Function):
    """``act(x @ w1ᵀ + b1) @ w2ᵀ`` as one autograd node so the backward can fuse across the two GEMMs:
    ``dpre = (dy @ w2) ⊙ act'(pre)`` is a single kernel (activation backward in the dgrad epilogue) – the
    separate bias+activation backward pass over the ``[tokens, ffn]`` tensor disappears."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, act, b2=None, residual=None):
        ext = load_ext()
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        h, pre = _linear_fwd_any(ext, x2, w1, b1, _ACT_IDS[act], True)
        # with a residual, the second bias and the block's residual add ride in the epilogue of the second GEMM
        res2 = residual.reshape(-1, w2.shape[0]).contiguous() if residual is not None else None
        y, _ = _linear_fwd_any(ext, h, w2, b2, 0, False, res2)
        ctx.act = act
        ctx.save_for_backward(x2, w1, w2, pre, h)
        ctx.x_shape = x.shape
        ctx.bias_param = b1
        ctx.bias2_param = b2
        ctx.has_res = residual is not None
        return y.view(*x.shape[:-1], w2.shape[0])

    @staticmethod
    def backward(ctx, gy):
        ext = load_ext()
        x2, w1, w2, pre, h = ctx.saved_tensors
        g2 = gy.reshape(-1, gy.shape[-1]).contiguous()
        # bias gradient of the first linear = column sums of dpre, accumulated into b1.main_grad by the dgrad call (a
        # column-sum pass with a fixed summation order, launched right behind the GEMM)
        b1 = ctx.bias_param
        fused_gb1 = _fused_bias_grad_target(b1) if ctx.needs_input_grad[2] else None
        dpre = ext.dgrad_actgrad(g2, w2, pre, _ACT_IDS[ctx.act], fused_gb1)
        count_launch()
        gw2 = _weight_grad(ext, g2, h, w2) if ctx.needs_input_grad[3] else None
        gw1 = _weight_grad(ext, dpre, x2, w1) if ctx.needs_input_grad[1] else None
        gb1 = None
        if fused_gb1 is not None:
            b1.grad_added_to_main_grad = True
        elif ctx.needs_input_grad[2]:
            gb1 = _bias_grad(ext, dpre, b1)
        gx = None
        if ctx.needs_input_grad[0]:
            gx = ext.gemm(dpre, w1, 1, None, None, False, torch.bfloat16).view(ctx.x_shape)
            count_launch()
        gb2 = None
        if ctx.bias2_param is not None and ctx.needs_input_grad[5]:
            gb2 = _bias_grad(ext, g2, ctx.bias2_param)
        return gx, gw1, gb1, gw2, None, gb2, (gy if ctx.has_res else None)


def mlp(x, w1, b1, w2, act: str = "gelu", b2=None, residual=None):
    """``act(x @ w1ᵀ + b1) @ w2ᵀ``; with ``residual`` also ``+ b2 + residual`` in the second GEMM's epilogue
    (without it the second bias is left to the fused bias+dropout+residual op)."""
    reject_quantized_weight("mlp", w1, w2)
    if use_native(x, w1) and _gemm_ok(x, w1) and _gemm_ok(x.new_empty(1, w1.shape[0]), w2):
        if residual is not None:
            return _MLPFn.apply(x, w1, b1, w2, act, b2, residual)
        return _MLPFn.apply(x, w1, b1, w2, act)
    y = linear(linear(x, w1, b1, act), w2, b2)
    return y if residual is None else y + residual


def linear_bias_residual(x, w, bias, residual):
    """``x @ wᵀ + bias + residual`` (output projection of a block, dropout-free)."""
    reject_quantized_weight("linear_bias_residual", w)
    if use_native(x, w) and _gemm_ok(x, w) and residual is not None and residual.dtype == torch.bfloat16:
        return _LinearFn.apply(x, w, bias, None, residual)
    y = linear(x, w, bias)
    return y if residual is None else y + residual


# --------------------------------------------------------------------------------------
# FP8 (E4M3) weights for inference: ``w`` [N, K] float8_e4m3fn with one fp32 scale per output channel, ``w_scale``
# [N] (:func:`kv_cache_quantize_ref` per row, see ``Linear1D.quantize_fp8_``); the weight reads back as float(e)·s
# --------------------------------------------------------------------------------------
# Up to this many rows (tokens) run the weight-streaming kernel; more dequantize the weight to bf16 and run the bf16 GEMM.
# 64 is the most the kernel takes: it was faster than dequantize + GEMM at every M of the sweep up to 64
# (dev/fp8_weights_bench.py, Kernels.md "FP8 weights")
FP8W_KERNEL_MAX_M = 64


def linear_fp8w_ref(x, w, w_scale, bias=None, act: Optional[str] = None):
    """``act(x @ (float(w)·w_scale[:, None])ᵀ + bias)`` in fp32, rounded to x's dtype."""
    y = F.linear(x.float(), w.float() * w_scale.float()[:, None], None if bias is None else bias.float())
    return _act_ref(y, act).to(x.dtype)


def linear_fp8w(x, w, w_scale, bias=None, act: Optional[str] = None):
    """``act(x @ (float(w)·w_scale[:, None])ᵀ + bias)`` for FP8 weights ``w`` [N, K] (float8_e4m3fn) with fp32 row
    scales ``w_scale`` [N]; returns x's dtype.  On the GPU with bf16 x (K % 16 == 0): up to ``FP8W_KERNEL_MAX_M``
    rows run the weight-streaming kernel (fp32 accumulation, scale, bias and activation on the fp32 sum), more rows
    dequantize the weight to bf16 (``bf16_rn(float(e)·s)``, a temporary of the caching allocator) and run the bf16 GEMM
    with its bias/activation epilogue.  Other inputs (CPU, fp32 or fp16 x, other shapes) run :func:`linear_fp8w_ref`.
    Inference only: a call that would need a gradient raises."""
    if torch.is_grad_enabled() and (x.requires_grad or (bias is not None and bias.requires_grad)):
        raise RuntimeError("FP8 weights are for inference: run the model under torch.no_grad() (and without inputs "
                           "that require a gradient)")
    N, K = w.shape
    x2 = x.reshape(-1, K)
    M = x2.shape[0]
    if (use_native(x) and x.dtype == torch.bfloat16 and w.is_cuda and w.is_contiguous() and K % 16 == 0 and M >= 1
            and (bias is None or bias.dtype == torch.bfloat16)):
        ext = load_ext()
        x2 = x2.contiguous()
        b = None if bias is None else bias.contiguous()
        if x2.data_ptr() % 16 == 0 and w.data_ptr() % 16 == 0:
            if M <= FP8W_KERNEL_MAX_M:
                y = ext.linear_fp8w(x2, w, w_scale, b, _ACT_IDS[act])
                count_launch(2)   # the kernel, and the sum over its K ranges
                return y.view(*x.shape[:-1], N)
            if N % 8 == 0:
                wb = ext.dequant_e4m3_rows(w, w_scale)
                y, _ = ext.linear_fwd(x2, wb, b, _ACT_IDS[act], False)
                count_launch(2)
                return y.view(*x.shape[:-1], N)
    return linear_fp8w_ref(x, w, w_scale, bias, act)


# --------------------------------------------------------------------------------------
# Group-wise INT4 weights for inference: ``w`` [N, K/2] uint8 holds the 4-bit values q two per byte (column 2j in the low
# nibble of byte j), ``w_scale`` [N, K/128] bf16 and ``w_zero`` [N, K/128] uint8 one scale s and zero point z per row and
# group of 128 columns (:func:`int4_quantize_ref`, see ``Linear1D.quantize_int4_``).  The weight reads back as
# Ŵ[n, k] = bf16_rn((q[n, k] − z[n, k/128]) · s[n, k/128]): q − z is an integer in [−15, 15] and s has an 8-bit
# significand, so the product is exact in fp32 and Ŵ is one rounding, the same bits in the kernel, the dequantize kernel
# and :func:`int4_dequant_ref`.
# --------------------------------------------------------------------------------------
INT4_GROUP = 128
# Up to this many rows (tokens) run the weight-streaming kernel; more dequantize the weight to bf16 and run the bf16 GEMM.
# 64 is the most the kernel takes: it was faster than dequantize + GEMM at every M of the sweep up to 64
# (dev/int4_weights_bench.py, Kernels.md "INT4 weights")
INT4W_KERNEL_MAX_M = 64


def int4_quantize_ref(w):
    """``(weight, weight_scale, weight_zero)`` of ``w`` [N, K] (K % 128 == 0, finite): round to nearest per row and
    group of 128 columns, in fp32 on ``w``'s device.  With ``lo = min(0, min w)`` and ``hi = max(0, max w)`` of a group,
    ``s = bf16_rn((hi − lo) / 15)`` (1 if that is zero or subnormal), ``z = clamp(round(−lo / s), 0, 15)`` and
    ``q = clamp(round(w / s) + z, 0, 15)``, rounding half to even.  Returns q packed two per byte (uint8 [N, K/2]),
    s (bf16 [N, K/128]) and z (uint8 [N, K/128])."""
    if w.dim() != 2 or w.shape[1] % INT4_GROUP != 0:
        raise ValueError(f"int4_quantize_ref: a [N, K] weight with K % {INT4_GROUP} == 0, got {tuple(w.shape)}")
    if not bool(torch.isfinite(w).all()):
        raise ValueError("int4_quantize_ref: the weight has a non-finite value")
    N, K = w.shape
    g = w.float().view(N, K // INT4_GROUP, INT4_GROUP)
    lo = g.amin(-1).clamp(max=0.0)
    hi = g.amax(-1).clamp(min=0.0)
    s = ((hi - lo) / 15).to(torch.bfloat16).float()
    s = torch.where(s < torch.finfo(torch.float32).tiny, torch.ones_like(s), s)   # zero or subnormal
    z = torch.clamp(torch.round(-lo / s), 0, 15)
    q = torch.clamp(torch.round(g / s[..., None]) + z[..., None], 0, 15).to(torch.uint8).view(N, K)
    return q[:, 0::2] | (q[:, 1::2] << 4), s.to(torch.bfloat16), z.to(torch.uint8)


def int4_dequant_ref(w, w_scale, w_zero):
    """Ŵ = bf16_rn((q − z) · s) as bf16 [N, K] of a packed INT4 weight (:func:`int4_quantize_ref`)."""
    N = w.shape[0]
    q = torch.stack([w & 15, w >> 4], dim=-1).view(N, -1, INT4_GROUP).float()
    wf = (q - w_zero.float()[..., None]) * w_scale.float()[..., None]
    return wf.view(N, -1).to(torch.bfloat16)


def linear_int4w_ref(x, w, w_scale, w_zero, bias=None, act: Optional[str] = None):
    """``act(x @ Ŵᵀ + bias)`` in fp32, rounded to x's dtype."""
    wf = int4_dequant_ref(w, w_scale, w_zero).float()
    y = F.linear(x.float(), wf, None if bias is None else bias.float())
    return _act_ref(y, act).to(x.dtype)


def linear_int4w(x, w, w_scale, w_zero, bias=None, act: Optional[str] = None):
    """``act(x @ Ŵᵀ + bias)`` for a packed INT4 weight ``w`` [N, K/2] (uint8) with bf16 group scales ``w_scale`` and uint8
    zero points ``w_zero`` [N, K/128]; returns x's dtype.  On the GPU with bf16 x: up to ``INT4W_KERNEL_MAX_M`` rows run
    the weight-streaming kernel (fp32 accumulation, bias and activation on the fp32 sum), more rows dequantize the
    weight to bf16 Ŵ (a temporary of the caching allocator) and run the bf16 GEMM with its bias/activation epilogue.
    Other inputs (CPU, fp32 or fp16 x) run :func:`linear_int4w_ref`.  Inference only: a call that would need a gradient
    raises."""
    if torch.is_grad_enabled() and (x.requires_grad or (bias is not None and bias.requires_grad)):
        raise RuntimeError("INT4 weights are for inference: run the model under torch.no_grad() (and without inputs "
                           "that require a gradient)")
    N, K = w.shape[0], 2 * w.shape[1]
    x2 = x.reshape(-1, K)
    M = x2.shape[0]
    if (use_native(x) and x.dtype == torch.bfloat16 and w.is_cuda and K % INT4_GROUP == 0 and M >= 1
            and all(t.is_contiguous() for t in (w, w_scale, w_zero)) and (bias is None or bias.dtype == torch.bfloat16)):
        ext = load_ext()
        x2 = x2.contiguous()
        b = None if bias is None else bias.contiguous()
        if x2.data_ptr() % 16 == 0 and w.data_ptr() % 16 == 0:
            if M <= INT4W_KERNEL_MAX_M:
                y = ext.linear_int4w(x2, w, w_scale, w_zero, b, _ACT_IDS[act])
                count_launch(2)   # the kernel, and the sum over its K ranges
                return y.view(*x.shape[:-1], N)
            if N % 8 == 0:
                wb = ext.dequant_int4_rows(w, w_scale, w_zero)
                y, _ = ext.linear_fwd(x2, wb, b, _ACT_IDS[act], False)
                count_launch(2)
                return y.view(*x.shape[:-1], N)
    return linear_int4w_ref(x, w, w_scale, w_zero, bias, act)


# --------------------------------------------------------------------------------------
# speculative decoding: greedy acceptance of one iteration (Generator.speculative_search)
# --------------------------------------------------------------------------------------
def spec_accept_ref(logits, draft, unfinished, eos: Optional[int] = None, pad: Optional[int] = None):
    """The PyTorch mirror of :func:`spec_accept` (same outputs, ``unfinished`` updated in place)."""
    b, R, _ = logits.shape
    k = R - 1
    t = logits.argmax(dim=-1)   # the first of equal maxima
    match = (draft == t[:, :k]).long()
    a = match.cumprod(dim=1).sum(dim=1) if k > 0 else torch.zeros(b, dtype=torch.long, device=logits.device)
    return _spec_emit(t, a, unfinished, eos, pad)


def _spec_emit(t, a, unfinished, eos, pad):
    """n and the emitted tokens e of one speculative iteration from its tokens t [b, R] and a_b (``unfinished``
    updated in place): the ``[b, 2R + 3]`` output of :func:`spec_accept` and :func:`spec_accept_sample`."""
    b, R = t.shape
    k = R - 1
    live = unfinished != 0
    if eos is not None:
        upto = torch.arange(R, device=t.device)[None, :] <= a[:, None]
        live_a = torch.where(((t == eos) & upto).any(dim=1), k, a)
    else:
        live_a = a
    n = int(live_a[live].min()) if bool(live.any()) else k
    e = t.clone()
    u = unfinished.clone()
    for j in range(R):
        if j > n:
            e[:, j] = -1
        elif eos is not None:
            e[:, j] = torch.where(u != 0, t[:, j], pad)
            u = u * (e[:, j] != eos).long()
    unfinished.copy_(u)
    nn_ = torch.full((b, 1), n, dtype=torch.long, device=t.device)
    return torch.cat([t, e, a[:, None], nn_, u[:, None]], dim=1)


def spec_accept(logits, draft, unfinished, eos: Optional[int] = None, pad: Optional[int] = None):
    """Greedy acceptance of one speculative-decoding iteration, in one launch of the sm_90a kernel on the GPU.

    ``logits`` ``[b, k + 1, V]`` (bf16 or fp32, read in place): the verify step's rows after ``x, d_1 .. d_k``;
    ``draft`` int64 ``[b, k]``: the proposals; ``unfinished`` int64 ``[b]``, updated in place.  With ``t_j`` the argmax
    of row j (the lowest index among equal maxima, for finite or −inf logits):

    - ``a_b``: the length of the longest prefix with ``draft[b, j] == t_j``;
    - ``n``: the minimum of ``a_b`` over the samples unfinished on entry, a sample that emits ``eos`` among
      ``t_0 .. t_{a_b}`` counting as k; k when none is unfinished;
    - ``e_j``: ``t_j`` for ``j <= n`` while the sample is unfinished, ``pad`` once it is (emitting ``eos`` finishes it),
      −1 for ``j > n``.  ``eos=None``: no EOS (``pad`` unused).

    Returns int64 ``[b, 2(k + 1) + 3]``: columns ``[0, k + 1)`` t, ``[k + 1, 2(k + 1))`` e, then ``a_b``, ``n`` and the
    updated ``unfinished``: everything the host needs, in one readback.  CPU tensors run :func:`spec_accept_ref`."""
    if eos is not None and pad is None:
        raise ValueError("spec_accept: eos needs a pad token")
    if not use_native(logits):
        return spec_accept_ref(logits, draft, unfinished, eos, pad)
    out = load_ext().spec_accept(logits, draft, unfinished, -1 if eos is None else int(eos),
                                 0 if pad is None else int(pad))
    count_launch(1)
    return out


# --------------------------------------------------------------------------------------
# speculative sampling: the warp rule, the draft's draws and the acceptance of one iteration
# --------------------------------------------------------------------------------------
# the fp32 margin within which the mirrors flag a decision as a boundary case: the kernels compute the masses from
# fp32 exponentials and 2^-40 fixed-point sums, the mirrors in fp64, so a decision this close may go either way
SPEC_SAMPLE_MARGIN = 1e-5


def _f32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


def _warp64(logits, temperature: float, top_k: int, top_p: float):
    """The warp rule on rows ``logits [..., V]``: ``(z, keep, p, gap)``.  z: the fp32 ``logits / T``; keep: the final
    kept set; p: fp64 probabilities on it (0 elsewhere); gap: per row, the distance of the nearest top-p mass above a
    token to ``top_p`` (inf when top-p is off)."""
    x = logits.float()
    T = torch.tensor(_f32(temperature), dtype=torch.float64, device=x.device)
    z = (x.double() / T).float()   # fp32 division, correctly rounded (fp64 quotient of fp32 operands, rounded once)
    V = z.shape[-1]
    keep = torch.ones_like(z, dtype=torch.bool)
    if 0 < top_k < V:
        kth = z.topk(top_k, dim=-1).values[..., -1:]
        keep = z >= kth
    zmax = z.amax(dim=-1, keepdim=True)
    z64 = z.double()
    e = torch.where(z == zmax, torch.ones_like(z64), torch.exp(z64 - zmax.double())) * keep
    gap = torch.full(z.shape[:-1], float("inf"), dtype=torch.float64, device=z.device)
    tp = _f32(top_p)
    if tp < 1.0:
        pi = e / e.sum(dim=-1, keepdim=True)
        zs, idx = z.masked_fill(~keep, float("-inf")).sort(dim=-1, descending=True)
        ps = pi.gather(-1, idx)
        excl = ps.cumsum(dim=-1) - ps
        # the mass strictly above a token: the exclusive sum at the first token of its tie group
        first = torch.searchsorted((-zs).contiguous(), (-zs).contiguous(), right=False).clamp(max=V - 1)
        above = torch.empty_like(excl).scatter_(-1, idx, excl.gather(-1, first))
        gap = (above - tp).abs().masked_fill(~keep, float("inf")).amin(dim=-1)
        keep = keep & (above <= tp)
        e = e * keep
    return z, keep, e / e.sum(dim=-1, keepdim=True), gap


def spec_warp_ref(logits, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0):
    """The warp rule of speculative sampling on rows ``logits [..., V]`` (bf16 or fp32), as fp32 warped logits: z on
    the kept set, −inf elsewhere.

    - ``z = logit / T``, an fp32 division (``TemperatureLogitsWarper``);
    - top-k (``k' = min(top_k, V)``, off when 0): keep ``z >=`` the k'-th largest z, counting duplicates
      (``TopKLogitsWarper``);
    - top-p (off when >= 1): with π the softmax of the kept z, keep token i iff the mass of kept tokens with z strictly
      greater than ``z_i`` is ``<= top_p``.  This is ``TopPLogitsWarper`` except on ties at the boundary: there
      ``TopPLogitsWarper`` keeps those of the tied tokens its (unstable) sort puts first, this rule keeps every one.

    p is the softmax over the final kept set.  ``temperature`` and ``top_p`` are taken as fp32, as the kernels take
    them."""
    z, keep, _, _ = _warp64(logits, temperature, top_k, top_p)
    return z.masked_fill(~keep, float("-inf"))


def _pick64(w, u):
    """Inverse CDF in index order on fp64 weights ``w [n, V]`` with uniforms ``u [n]``: the smallest i whose inclusive
    prefix sum exceeds ``u · Σw``; and whether ``u · Σw`` lies within the margin of a step of the CDF."""
    total = w.sum(dim=-1)
    target = u.double() * total
    cum = w.cumsum(dim=-1)
    idx = torch.searchsorted(cum, target[:, None], right=True).clamp(max=w.shape[-1] - 1)[:, 0]
    upper = cum.gather(-1, idx[:, None])[:, 0]
    lower = torch.where(idx > 0, cum.gather(-1, (idx - 1).clamp(min=0)[:, None])[:, 0], torch.zeros_like(total))
    near = torch.minimum(target - lower, upper - target) <= SPEC_SAMPLE_MARGIN * total
    return idx, near


def spec_sample_ref(logits, q, j: int, u, proposals, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0,
                    flags: bool = False):
    """The fp64 PyTorch mirror of :func:`spec_sample`; ``flags=True`` also returns, per sample, whether the draw lies
    within :data:`SPEC_SAMPLE_MARGIN` of a boundary (a step of the CDF, or a top-p mass)."""
    q[:, j].copy_(logits)
    _, _, p, gap = _warp64(logits, temperature, top_k, top_p)
    d, near = _pick64(p, u[:, j])
    proposals[:, j] = d
    if flags:
        return near | (gap <= SPEC_SAMPLE_MARGIN)


def spec_sample(logits, q, j: int, u, proposals, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0):
    """One draft step of speculative sampling, in one launch of the sm_90a kernel on the GPU: keeps the draft's logits
    row ``logits [b, V]`` (bf16 or fp32) in ``q[:, j]`` (``q [b, K, V]``, the same dtype; q itself is never
    materialised) and draws ``proposals[:, j]`` (int64 ``[b, J]``) from its warped distribution (:func:`spec_warp_ref`)
    by inverse CDF in index order with the uniforms ``u[:, j]`` (fp32 ``[b, J]``), without a host sync.  CPU tensors
    run :func:`spec_sample_ref`."""
    if not use_native(logits):
        spec_sample_ref(logits, q, j, u, proposals, temperature, top_k, top_p)
        return
    load_ext().spec_sample(logits, q, int(j), u, proposals, float(temperature), int(top_k), float(top_p))
    count_launch(1)


def spec_accept_sample_ref(logits, q, draft, u, unfinished, temperature: float = 1.0, top_k: int = 0,
                           top_p: float = 1.0, eos: Optional[int] = None, pad: Optional[int] = None, scores=None,
                           flags: bool = False):
    """The fp64 PyTorch mirror of :func:`spec_accept_sample` (same outputs, ``unfinished`` and ``scores`` written in
    place).  ``flags=True`` also returns a bool ``[b, k + 1]``: the decisions of row j (its acceptance and its
    candidate) lie within :data:`SPEC_SAMPLE_MARGIN` of a boundary: a top-p mass of p_j or q_j, ``u · q`` against p, a
    step of the CDF, or a residual mass near 0."""
    b, R, V = logits.shape
    k = R - 1
    z, keep, p, gap = _warp64(logits, temperature, top_k, top_p)
    near = gap <= SPEC_SAMPLE_MARGIN
    if scores is not None:
        scores.copy_(z.masked_fill(~keep, float("-inf")))
    u0, u1 = u[..., 0].double(), u[..., 1]
    cand_w = p.clone()
    a = torch.zeros(b, dtype=torch.long, device=logits.device)
    if k > 0:
        _, _, qq, gap_q = _warp64(q[:, :k], temperature, top_k, top_p)
        d = draft.clamp(0, V - 1)[..., None]
        pd, qd = p[:, :k].gather(-1, d)[..., 0], qq.gather(-1, d)[..., 0]
        acc = (u0[:, :k] * qd < pd) & (draft >= 0) & (draft < V)
        near[:, :k] |= (gap_q <= SPEC_SAMPLE_MARGIN) | ((u0[:, :k] * qd - pd).abs() <= SPEC_SAMPLE_MARGIN * (pd + qd))
        r = (p[:, :k] - qq).clamp(min=0)
        rs = r.sum(dim=-1, keepdim=True)
        near[:, :k] |= (rs[..., 0] > 0) & (rs[..., 0] <= SPEC_SAMPLE_MARGIN)
        cand_w[:, :k] = torch.where(rs > 0, r, p[:, :k])
        a = acc.long().cumprod(dim=1).sum(dim=1)
    cand, near_pick = _pick64(cand_w.reshape(b * R, V), u1.reshape(b * R))
    cand = cand.view(b, R)
    near |= near_pick.view(b, R)
    t = cand.clone()
    if k > 0:
        t[:, :k] = torch.where(torch.arange(k, device=t.device)[None, :] < a[:, None], draft, cand[:, :k])
    out = _spec_emit(t, a, unfinished, eos, pad)
    return (out, near) if flags else out


def spec_accept_sample(logits, q, draft, u, unfinished, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0,
                       eos: Optional[int] = None, pad: Optional[int] = None, scores=None):
    """The acceptance of one speculative-sampling iteration, in one launch of the sm_90a kernel on the GPU.

    ``logits [b, k + 1, V]``: the verify step's rows after ``x, d_1 .. d_k`` (p_j warped from row j); ``q [b, K, V]``
    (K >= k): the draft's rows, q_j warped from ``q[:, j]`` by the same rule (:func:`spec_warp_ref`), so the q that
    accepts a proposal is the q it was drawn from, bit for bit; ``draft`` int64 ``[b, k]``: d_1 .. d_k; ``u`` fp32
    ``[b, k + 1, 2]``: uniforms; ``unfinished`` int64 ``[b]``, updated in place.  Per sample and row j:

    - accept_j: ``u[b, j, 0] · q_j(d_{j+1}) < p_j(d_{j+1})`` (j < k);
    - the candidate c_j, drawn with ``u[b, j, 1]`` by inverse CDF in index order from norm(max(0, p_j − q_j)) for
      j < k (from p_j when that mass is 0), from p_k for j = k (the bonus token);
    - ``a_b``: the first rejected j (k if none); ``t_j = d_{j+1}`` for ``j < a_b``, else c_j;
    - n, e and ``unfinished`` from t as :func:`spec_accept` defines them.

    Returns int64 ``[b, 2(k + 1) + 3]`` laid out as :func:`spec_accept`'s.  ``scores`` (optional, fp32 ``[b, k + 1,
    V]``): written with the target's warped logits (z on the kept set, −inf elsewhere).

    Why the batch rule is unbiased.  A sample's token at position j is emitted iff j <= n, and whether it reaches j
    depends only on its own acceptances before j and on the other samples, never on its own token at j.  Given its
    prefix, that token is d_{j+1} ~ q_j accepted with probability min(1, p_j/q_j), or on the first rejection a draw
    from norm(max(0, p_j − q_j)): together distributed as p_j (Leviathan et al. 2023, appendix A.1); at j = a_b with no
    rejection it is the bonus draw from p_j.  So every emitted token is distributed as p given its prefix, whatever
    the draft is.  CPU tensors run :func:`spec_accept_sample_ref`."""
    if eos is not None and pad is None:
        raise ValueError("spec_accept_sample: eos needs a pad token")
    if not use_native(logits):
        return spec_accept_sample_ref(logits, q, draft, u, unfinished, temperature, top_k, top_p, eos, pad, scores)
    out = load_ext().spec_accept_sample(logits, q, draft, u, unfinished, float(temperature), int(top_k), float(top_p),
                                        -1 if eos is None else int(eos), 0 if pad is None else int(pad), scores)
    count_launch(1)
    return out


def matmul_nt(a, b):
    """``a @ b.T`` without autograd bookkeeping beyond PyTorch's (used by LM head on ref path)."""
    return linear(a, b)


# --------------------------------------------------------------------------------------
# LayerNorm / RMSNorm (optionally fused with the preceding residual add)
# --------------------------------------------------------------------------------------
class _LayerNormFn(torch.autograd.Function):
    """``with_skip``: additionally return the input itself as a second output.  A pre-LN block uses the same tensor for
    the norm and for the skip connection; autograd would sum the two gradients with a separate kernel — here both
    arrive in one ``backward`` call and the skip gradient is added inside the LayerNorm backward kernel."""

    @staticmethod
    def forward(ctx, x, weight, bias, eps, rms, with_skip=False):
        ext = load_ext()
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        y, mean, rstd = ext.norm_fwd(x2, weight, bias, eps, rms)
        count_launch()
        ctx.save_for_backward(x2, weight, mean, rstd)
        ctx.rms = rms
        ctx.has_bias = bias is not None
        ctx.bias_param = bias
        ctx.with_skip = with_skip
        if with_skip:
            return y.view(x.shape), x.view_as(x)
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, gy, gskip=None):
        ext = load_ext()
        x2, weight, mean, rstd = ctx.saved_tensors
        if gy is None:          # only the skip output was used
            return gskip, None, None, None, None, None
        g2 = gy.reshape(-1, gy.shape[-1]).contiguous()
        gadd = None if gskip is None else gskip.reshape(-1, gskip.shape[-1]).contiguous()
        count_launch(2)
        wg = _main_grad(weight)
        bg = _main_grad(ctx.bias_param) if ctx.has_bias else None
        if wg is not None and (not ctx.has_bias or bg is not None):
            # dγ / dβ are reduced straight into the fp32 main-grad slices (one kernel for both)
            gx, _, _ = ext.norm_bwd(g2, x2, weight, mean, rstd, ctx.rms, ctx.has_bias, wg, bg, gadd)
            weight.grad_added_to_main_grad = True
            if ctx.has_bias:
                ctx.bias_param.grad_added_to_main_grad = True
            return gx.view(gy.shape), None, None, None, None, None
        gx, gw, gb = ext.norm_bwd(g2, x2, weight, mean, rstd, ctx.rms, ctx.has_bias, None, None, gadd)
        return (gx.view(gy.shape), gw.to(weight.dtype), (gb.to(weight.dtype) if ctx.has_bias else None), None, None,
                None)


_NORM_DTYPES = {(torch.bfloat16, torch.bfloat16), (torch.bfloat16, torch.float32), (torch.float32, torch.float32)}


def _norm_native(x, weight, bias=None) -> bool:
    """The native norm kernels take these (activation, γ) dtype pairs, with β of γ's dtype."""
    return (use_native(x) and weight is not None and (x.dtype, weight.dtype) in _NORM_DTYPES
            and (bias is None or bias.dtype == weight.dtype))


def layer_norm_with_skip(x, weight, bias, eps: float = 1e-5):
    """``(layer_norm(x), x)`` where the second output carries the skip connection (see ``_LayerNormFn``)."""
    if _norm_native(x, weight, bias) and x.requires_grad:
        return _LayerNormFn.apply(x, weight, bias, eps, False, True)
    return layer_norm(x, weight, bias, eps), x


def layer_norm(x, weight, bias, eps: float = 1e-5):
    if _norm_native(x, weight, bias):
        return _LayerNormFn.apply(x, weight, bias, eps, False)
    w = None if weight is None else weight.float()
    b = None if bias is None else bias.float()
    return F.layer_norm(x.float(), (x.shape[-1],), w, b, eps).to(x.dtype)


def rms_norm(x, weight, eps: float = 1e-6):
    if _norm_native(x, weight):
        return _LayerNormFn.apply(x, weight, None, eps, True)
    xf = x.float()
    y = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    return (y * weight.float()).to(x.dtype)


# --------------------------------------------------------------------------------------
# bias + gelu, bias + dropout + residual
# --------------------------------------------------------------------------------------
class _BiasActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, bias, act):
        ext = load_ext()
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        y = ext.bias_act_fwd(x2, bias, _ACT_IDS[act])
        count_launch()
        ctx.save_for_backward(x2, bias)
        ctx.act = act
        ctx.bias_param = bias
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, gy):
        ext = load_ext()
        x2, bias = ctx.saved_tensors
        g2 = gy.reshape(-1, gy.shape[-1]).contiguous()
        gx = ext.bias_act_bwd(g2, x2, bias, _ACT_IDS[ctx.act])
        count_launch()
        gb = None
        if bias is not None and ctx.needs_input_grad[1]:
            gb = _bias_grad(ext, gx, ctx.bias_param)
        return gx.view(gy.shape), gb, None


def bias_act(x, bias, act: str = "gelu"):
    """``act(x + bias)`` (replaces ``fused_bias_add_gelu``)."""
    if use_native(x) and x.dtype == torch.bfloat16:
        return _BiasActFn.apply(x, bias, act)
    y = x if bias is None else x + bias.to(x.dtype)
    return _act_ref(y, act)


def bias_gelu(x, bias):
    return bias_act(x, bias, "gelu")


def tp_rng_salt(sharded: bool) -> int:
    """Salt of the dropout RNG stream (TP-aware RNG).  All tensor-parallel ranks of a model replica share
    one (seed, offset) sequence (``dutil.model_parallel_seed``); activations that are *sharded* over the TP group
    (attention heads, token shards under sequence parallelism) must see different masks on different ranks → the TP
    rank is mixed into the Philox key; *replicated* activations (salt 0) get identical masks everywhere."""
    if not sharded:
        return 0
    from libai_b200.utils import distributed as dutil

    topo = dutil.get_dist_util()
    return topo.tp_rank + 1 if topo.tensor_parallel_size > 1 else 0


def _activations_token_sharded() -> bool:
    from libai_b200.utils import distributed as dutil

    return bool(dutil.get_dist_util().sequence_parallel)


class _BiasDropoutAddFn(torch.autograd.Function):
    """``residual + dropout(x + bias)`` in one native kernel; the mask is a pure function of the Philox
    ``(seed, offset)`` pair stored by the forward and the element index, so nothing but 16 bytes is kept for backward."""

    @staticmethod
    def forward(ctx, x, bias, residual, p, salt):
        ext = load_ext()
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        r2 = None if residual is None else residual.reshape(-1, x.shape[-1]).contiguous()
        y, rng_state = ext.bias_dropout_residual(x2, bias, r2, p, salt, None)
        count_launch()
        ctx.save_for_backward(rng_state)
        ctx.p, ctx.bias_param, ctx.has_res = p, bias, residual is not None
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, gy):
        ext = load_ext()
        (rng_state,) = ctx.saved_tensors
        g2 = gy.reshape(-1, gy.shape[-1]).contiguous()
        gx, _ = ext.bias_dropout_residual(g2, None, None, ctx.p, 0, rng_state)
        count_launch()
        gb = None
        if ctx.bias_param is not None and ctx.needs_input_grad[1]:
            gb = _bias_grad(ext, gx, ctx.bias_param)
        return gx.view(gy.shape), gb, (gy if ctx.has_res else None), None, None


def bias_dropout_add(x, bias, residual, p: float, training: bool, sharded=None):
    """``residual + dropout(x + bias)`` (replaces ``fused_bias_add_dropout`` + the add).  ``sharded``: whether ``x`` is
    sharded over the tensor-parallel group (default: yes iff sequence parallelism is on), see :func:`tp_rng_salt`."""
    if use_native(x) and x.dtype == torch.bfloat16 and x.shape[-1] % 8 == 0:
        if p == 0.0 or not training:
            return _BiasAddFn.apply(x, bias, residual)
        if sharded is None:
            sharded = _activations_token_sharded()
        return _BiasDropoutAddFn.apply(x, bias, residual, float(p), tp_rng_salt(sharded))
    y = x if bias is None else x + bias.to(x.dtype)
    y = F.dropout(y, p=p, training=training)
    return y if residual is None else residual + y


def dropout(x, p: float, training: bool, sharded: bool = False):
    """Native Philox dropout (same kernel as :func:`bias_dropout_add` without bias / residual)."""
    if p == 0.0 or not training:
        return x
    if use_native(x) and x.dtype == torch.bfloat16 and x.shape[-1] % 8 == 0:
        return _BiasDropoutAddFn.apply(x, None, None, float(p), tp_rng_salt(sharded))
    return F.dropout(x, p=p, training=training)


class _BiasAddFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, bias, residual):
        ext = load_ext()
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        r2 = None if residual is None else residual.reshape(-1, x.shape[-1]).contiguous()
        y = ext.bias_residual_fwd(x2, bias, r2)
        count_launch()
        ctx.has_bias = bias is not None
        ctx.bias_param = bias
        ctx.has_res = residual is not None
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, gy):
        gb = None
        if ctx.has_bias and ctx.needs_input_grad[1]:
            gb = _bias_grad(load_ext(), gy.reshape(-1, gy.shape[-1]).contiguous(), ctx.bias_param)
        return gy, gb, (gy if ctx.has_res else None)


# --------------------------------------------------------------------------------------
# attention
#
# Grouped-query attention (GQA): ``a`` query heads share ``g`` key/value heads (``a % g == 0``), query head ``h`` reading
# K/V head ``h // (a // g)``.  The packed projection of a grouped model is ``[b, s, g, r + 2, d]`` with ``q_0 .. q_{r-1},
# k, v`` per group (``r = a // g``); the 4-D ``[b, s, a, 3d]`` (per-head ``[q|k|v]``) keeps meaning MHA and is the
# same memory as the grouped view with ``r = 1``.
# --------------------------------------------------------------------------------------
def _expand_kv(x, heads: int):
    """K/V ``[.., g, s, d]`` repeated to ``heads`` query heads (reference math only: the kernels read the g heads)."""
    g = x.shape[-3]
    if g == heads:
        return x
    if heads % g:
        raise ValueError(f"{heads} query heads cannot share {g} key/value heads")
    return x.repeat_interleave(heads // g, dim=-3)


def split_qkv(qkv):
    """q ``[b, s, a, d]`` and k, v ``[b, s, g, d]`` of a packed projection ``[b, s, a, 3d]`` or ``[b, s, g, r + 2, d]``."""
    if qkv.dim() == 4:
        d = qkv.shape[-1] // 3
        return qkv[..., :d], qkv[..., d : 2 * d], qkv[..., 2 * d :]
    b, s, g, r2, d = qkv.shape
    return qkv[..., : r2 - 2, :].reshape(b, s, g * (r2 - 2), d), qkv[..., r2 - 2, :], qkv[..., r2 - 1, :]


def _packed_views(qkv):
    """The attention kernels' operands, read in place: q ``[b, a, s, d]`` (from ``[b, s, a, 3d]``) or ``[b, g, r, s, d]``
    (from ``[b, s, g, r + 2, d]``), k and v ``[b, g, s, d]``."""
    if qkv.dim() == 4:
        d = qkv.shape[-1] // 3
        v4 = qkv.permute(0, 2, 1, 3)
        return v4[..., :d], v4[..., d : 2 * d], v4[..., 2 * d :]
    r = qkv.shape[3] - 2
    return (qkv[:, :, :, :r].permute(0, 2, 3, 1, 4), qkv[:, :, :, r].permute(0, 2, 1, 3),
            qkv[:, :, :, r + 1].permute(0, 2, 1, 3))


def packed_head_dim(qkv) -> int:
    return qkv.shape[-1] // 3 if qkv.dim() == 4 else qkv.shape[-1]


def attention_ref(q, k, v, *, causal: bool, scale: float, mask=None, bias=None, dropout_p: float = 0.0,
                  training: bool = False, fill: float = -10000.0):
    """Unfused attention on ``[b, a, s, d]`` queries and ``[b, g, s, d]`` keys / values (``g`` divides ``a``; the K/V
    heads are repeated here). ``mask``: 1 = keep, 0 = masked
    (filled with ``fill`` like the reference: libai/layers/attention.py:223-245)."""
    k, v = _expand_kv(k, q.shape[-3]), _expand_kv(v, q.shape[-3])
    scores = torch.matmul(q.float(), k.float().transpose(-1, -2)) * scale
    if bias is not None:
        scores = scores + bias.float()
    sq, sk = scores.shape[-2], scores.shape[-1]
    if causal:
        tril = torch.ones(sq, sk, dtype=torch.bool, device=q.device).tril(diagonal=sk - sq)
        scores = torch.where(tril, scores, torch.full_like(scores, fill))
    if mask is not None:
        scores = torch.where(mask.bool(), scores, torch.full_like(scores, fill))
    probs = torch.softmax(scores, dim=-1)
    probs = F.dropout(probs, p=dropout_p, training=training)
    return torch.matmul(probs, v.float()).to(q.dtype)


def visible_keys(sq: int, sk: int, *, causal: bool, kv_start=None, kv_lens=None, doc_start=None, prefix_lens=None,
                 device=None):
    """Boolean ``[b|1, 1, sq, sk]`` visibility of the flash kernels: key ``j`` is visible to query ``i`` of sample ``b``
    iff ``kv_start[b] <= j < max(1, kv_lens[b])`` (defaults ``0`` and ``sk``) and, when ``causal``,
    ``j <= i + sk - sq`` (bottom-right alignment) or ``j < prefix_lens[b]`` (int ``[b]``, causal only: a prefix LM's
    bidirectional context, counted in key coordinates).  ``doc_start`` (int ``[b, sq]``, packed sequences) adds
    ``j >= doc_start[b, i]``, with ``doc_start`` clamped to ``[0, i]`` so that every query sees itself."""
    if prefix_lens is not None and not causal:
        raise ValueError("prefix_lens needs causal=True")
    j = torch.arange(sk, device=device)
    vis = torch.ones(1, sq, sk, dtype=torch.bool, device=device)
    if causal:
        c = (j[None, :] <= torch.arange(sq, device=device)[:, None] + (sk - sq))[None]
        if prefix_lens is not None:
            c = c | (j[None, None, :] < prefix_lens.to(device=device, dtype=torch.long)[:, None, None])
        vis = vis & c
    if doc_start is not None:
        i = torch.arange(sq, device=device)
        beg = torch.minimum(doc_start.to(device=device, dtype=torch.long).clamp(min=0), i[None, :])
        vis = vis & (j[None, None, :] >= beg[:, :, None])
    if kv_start is not None:
        vis = vis & (j[None, None, :] >= kv_start.to(device=device, dtype=torch.long)[:, None, None])
    if kv_lens is not None:
        end = kv_lens.to(device=device, dtype=torch.long).clamp(min=1)
        vis = vis & (j[None, None, :] < end[:, None, None])
    return vis[:, None]


def _prep_bias(bias, q):
    """Additive score bias for the flash kernel: bf16 ``[B|1, A|1, Sq, Sk]`` with contiguous keys and rows whose stride
    is a multiple of 8 elements (a key length that is not gets its rows padded)."""
    if bias is None:
        return None
    b = bias
    while b.dim() < 4:
        b = b.unsqueeze(0)
    if b.dtype != torch.bfloat16:
        b = b.to(torch.bfloat16)
    if b.stride(-1) != 1 or b.stride(-2) % 8 or b.stride(0) % 8 or b.stride(1) % 8 or b.data_ptr() % 16:
        sk = b.shape[-1]
        if sk % 8 == 0:
            b = b.contiguous()
        else:
            padded = b.new_zeros(*b.shape[:-1], sk + (-sk % 8))
            padded[..., :sk] = b
            b = padded[..., :sk]
    return b


class _FlashAttnFn(torch.autograd.Function):
    """Flash attention on ``[b, a, sq, d]`` / ``[b, g, sk, d]`` views with optional additive bias (dense or ALiBi
    slopes), per-sample key windows (``kv_start`` / ``kv_lens``), a prefix-LM prefix (``prefix_lens``) and Philox
    dropout on the probabilities — all inside the wgmma kernels."""

    @staticmethod
    def forward(ctx, q, k, v, causal, scale, bias, alibi_slopes, p_drop, kv_lens, kv_start=None, prefix_lens=None):
        ext = load_ext()
        b = _prep_bias(bias, q)
        ctx.prefix = {} if prefix_lens is None else {"prefix_lens": prefix_lens}
        o, lse, rng_state = ext.attn_fwd(q, k, v, causal, scale, kv_lens, b, alibi_slopes, p_drop,
                                         tp_rng_salt(True) if p_drop > 0 else 0, kv_start, **ctx.prefix)
        count_launch()
        ctx.save_for_backward(q, k, v, o, lse, b, alibi_slopes, rng_state, kv_lens, kv_start, prefix_lens)
        ctx.causal, ctx.scale, ctx.p_drop = causal, scale, p_drop
        ctx.bias_shape = None if bias is None else (bias.shape, bias.dtype)
        return o

    @staticmethod
    def backward(ctx, go):
        ext = load_ext()
        q, k, v, o, lse, b, slopes, rng_state, kv_lens, kv_start, prefix_lens = ctx.saved_tensors
        prefix = {} if prefix_lens is None else {"prefix_lens": prefix_lens}
        dbias = None
        if b is not None and ctx.needs_input_grad[5]:
            dbias = torch.zeros(b.shape, dtype=torch.float32, device=b.device)
            if dbias.stride() != b.stride():
                dbias = torch.empty_strided(b.shape, b.stride(), dtype=torch.float32, device=b.device).zero_()
        dq, dk, dv, _ = ext.attn_bwd(go, q, k, v, o, lse, ctx.causal, ctx.scale, kv_lens, b, slopes, dbias, ctx.p_drop,
                                     rng_state if ctx.p_drop > 0 else None, kv_start, **prefix)
        count_launch(3)
        gb = None
        if dbias is not None:
            shape, dtype = ctx.bias_shape
            gb = dbias.to(dtype).reshape(shape)
        return dq, dk, dv, None, None, gb, None, None, None, None, None


class _FlashAttnPackedFn(torch.autograd.Function):
    """Self-attention straight from the packed QKV projection ``[b, s, a, 3d]`` (per-head ``[q|k|v]``) or
    ``[b, s, g, r + 2, d]`` (grouped): the kernels read q/k/v through strided TMA maps and the backward writes one packed
    ``dqkv`` of the same layout – no slicing, no expanded K/V, no gradient accumulation kernels around the attention."""

    @staticmethod
    def forward(ctx, qkv, causal, scale, kv_lens, p_drop=0.0, alibi_slopes=None, doc_start=None):
        ext = load_ext()
        q, k, v = _packed_views(qkv)
        o, lse, rng_state = ext.attn_fwd(q, k, v, causal, scale, kv_lens, None, alibi_slopes, p_drop,
                                         tp_rng_salt(True) if p_drop > 0 else 0, None, doc_start)
        count_launch()
        ctx.save_for_backward(qkv, o, lse, kv_lens, rng_state, alibi_slopes, doc_start)
        ctx.causal, ctx.scale, ctx.p_drop = causal, scale, p_drop
        return o.permute(0, 2, 1, 3)  # [b, s, a, d] contiguous

    @staticmethod
    def backward(ctx, go):
        ext = load_ext()
        qkv, o, lse, kv_lens, rng_state, slopes, doc_start = ctx.saved_tensors
        q, k, v = _packed_views(qkv)
        _, _, _, dqkv = ext.attn_bwd(go.permute(0, 2, 1, 3), q, k, v, o, lse, ctx.causal, ctx.scale, kv_lens, None, slopes,
                                     None, ctx.p_drop, rng_state if ctx.p_drop > 0 else None, None, doc_start)
        count_launch(3)
        return dqkv.view(qkv.shape), None, None, None, None, None, None


def flash_head_dim_supported(d: int) -> bool:
    """True for the head dims the flash kernels take: multiples of 8 from 8 to 128 (a head dim up to 64 runs on the
    64-wide tile, a larger one on the 128-wide tile, with the columns past ``d`` zero-filled)."""
    return d % 8 == 0 and 8 <= d <= 128


def attention_qkvpacked_supported(qkv, mask, dropout_p, training, doc_start=None) -> bool:
    """True when :func:`attention_qkvpacked` runs the native flash kernels: a contiguous bf16 projection on the GPU
    whose head dim :func:`flash_head_dim_supported` accepts, and no dense ``mask``; packed sequences (``doc_start``)
    also need no attention dropout in training."""
    return (
        use_native(qkv)
        and qkv.dtype == torch.bfloat16
        and mask is None
        and flash_head_dim_supported(packed_head_dim(qkv))
        and qkv.is_contiguous()
        and (doc_start is None or not (training and dropout_p > 0))
    )


def attention_qkvpacked(qkv, *, causal: bool, scale: float, kv_lens=None, dropout_p: float = 0.0, training: bool = False,
                        alibi_slopes=None, doc_start=None):
    """qkv ``[b, s, a, 3d]`` or grouped ``[b, s, g, r + 2, d]`` → context ``[b, s, a, d]``; ``kv_lens`` (int32 ``[b]``): valid keys per sample
    of a right-padded batch (keys beyond it are masked inside the kernel); ``dropout_p`` > 0 in training drops
    attention probabilities inside the kernel (Philox, TP-rank salted).  ``doc_start`` (int32 ``[b, s]``, causal
    only): packed sequences, query ``i`` sees the keys ``doc_start[b, i] <= j <= i`` (see :func:`visible_keys`)."""
    p = float(dropout_p) if training else 0.0
    return _FlashAttnPackedFn.apply(qkv, causal, float(scale), kv_lens, p, alibi_slopes, doc_start)


def attention_supported(q, k, mask=None, bias=None) -> bool:
    """True when :func:`attention` of ``q`` over ``k`` runs the native flash kernels: bf16 on the GPU, a head dim
    :func:`flash_head_dim_supported` accepts (a multiple of 8 from 8 to 128), no dense 0/1 ``mask`` and a dense
    ``bias`` (if any) of shape ``[.., sq, sk]``.  Query and key lengths are free.  Otherwise :func:`attention` runs the
    reference math."""
    return (
        use_native(q)
        and q.dtype == torch.bfloat16
        and mask is None
        and flash_head_dim_supported(q.shape[-1])
        and (bias is None or (bias.shape[-1] == k.shape[-2] and bias.shape[-2] == q.shape[-2]))
    )


def attention(q, k, v, *, causal: bool = False, scale: Optional[float] = None, mask=None, bias=None,
              dropout_p: float = 0.0, training: bool = False, alibi_slopes=None, kv_lens=None, kv_start=None,
              prefix_lens=None):
    """Softmax attention of q ``[b, a, sq, d]`` over k, v ``[b, g, sk, d]`` (``g = a`` or, grouped-query, a divisor of
    ``a``; ``sq`` and ``sk`` independent).  Key ``j`` is visible to query ``i`` of sample ``b`` iff
    ``kv_start[b] <= j < kv_lens[b]`` (int32 ``[b]`` device tensors, defaults ``0`` and ``sk``; ``kv_lens`` is clamped to
    at least 1) and, when ``causal``, ``j <= i + sk - sq`` (bottom-right alignment).  A query without a visible key
    gets zeros.  The native flash kernels (see :func:`attention_supported`) handle this masking, an additive score bias
    (dense ``[b|1, a|1, sq, sk]`` — T5 relative positions — or ``alibi_slopes`` ``[a]``, ``slope·(j − i − (sk − sq))``)
    and dropout on the probabilities; arbitrary dense 0/1 masks use the reference math.  The reference applies
    ``kv_lens`` only together with ``kv_start`` or ``prefix_lens``.

    ``prefix_lens`` (int32 ``[b]`` device tensor, ``causal`` only, without ``bias`` or ``alibi_slopes``): a prefix LM,
    key ``j`` is also visible to every query when ``j < prefix_lens[b]`` (GLM's bidirectional context, counted in key
    coordinates).  The reference math builds the same rule densely (:func:`visible_keys`)."""
    if scale is None:
        scale = 1.0 / math.sqrt(q.shape[-1])
    if prefix_lens is not None and (not causal or bias is not None or alibi_slopes is not None):
        raise ValueError("prefix_lens needs causal=True and combines with neither bias nor alibi_slopes")
    if attention_supported(q, k, mask, bias):
        # strided [b, a, s, d] views of the packed QKV projection are consumed directly (TMA strides)
        return _FlashAttnFn.apply(q, k, v, causal, float(scale), bias, alibi_slopes,
                                  float(dropout_p) if training else 0.0, kv_lens, kv_start, prefix_lens)
    if kv_start is not None or prefix_lens is not None:
        vis = visible_keys(q.shape[-2], k.shape[-2], causal=causal, kv_start=kv_start, kv_lens=kv_lens,
                           prefix_lens=prefix_lens, device=q.device)
        if mask is not None:
            vis = vis & mask.bool()
        o = attention(q, k, v, causal=False, scale=scale, mask=vis, bias=bias, dropout_p=dropout_p, training=training,
                      alibi_slopes=alibi_slopes)
        return o.masked_fill(~vis.any(-1, keepdim=True), 0)
    if alibi_slopes is not None:
        sq, sk = q.shape[-2], k.shape[-2]
        rel = torch.arange(sk, device=q.device)[None, :] - torch.arange(sk - sq, sk, device=q.device)[:, None]
        ab = alibi_slopes.float()[None, :, None, None] * rel[None, None].float()
        bias = ab if bias is None else bias.float() + ab
    return attention_ref(q, k, v, causal=causal, scale=scale, mask=mask, bias=bias,
                         dropout_p=dropout_p, training=training)


# --------------------------------------------------------------------------------------
# shifted-window attention (Swin, SwinV2)
# --------------------------------------------------------------------------------------
def window_attention_supported(x, *, H: int, W: int, window: int, shift: int, head_dim: int, attn_drop: float = 0.0,
                               training: bool = False) -> bool:
    """True when a Swin block on the tokens ``x`` ``[B, H·W, C]`` runs :func:`window_attention`: bf16 on the GPU, a head
    dim that is a multiple of 8 from 8 to 64, a window of 1 to 16 that tiles the ``H × W`` map, ``0 <= shift < window``,
    and no attention dropout in training (the kernel has none).  Otherwise the block keeps its PyTorch window path."""
    return (
        use_native(x)
        and x.dtype == torch.bfloat16
        and head_dim % 8 == 0
        and 8 <= head_dim <= 64
        and 1 <= window <= 16
        and H % window == 0
        and W % window == 0
        and 0 <= shift < window
        and not (training and attn_drop > 0.0)
    )


class _WindowAttnFn(torch.autograd.Function):
    """Shifted-window attention read straight from the image-ordered qkv projection; the backward writes one ``dqkv`` of
    the same layout and the table (and ``tau``) gradients, reduced in a fixed order."""

    @staticmethod
    def forward(ctx, qkv, table, tau, H, W, window, shift, heads, scale):
        ext = load_ext()
        qkv = qkv.contiguous()
        o, lse = ext.window_attn_fwd(qkv, H, W, window, shift, heads, scale, table, tau)
        count_launch()
        ctx.save_for_backward(qkv, lse, table, tau)
        ctx.geom = (H, W, window, shift, heads, scale)
        return o

    @staticmethod
    def backward(ctx, go):
        ext = load_ext()
        qkv, lse, table, tau = ctx.saved_tensors
        dqkv, dtable, dtau = ext.window_attn_bwd(go.contiguous(), qkv, lse, *ctx.geom, table, tau)
        count_launch(3)
        return dqkv, dtable, (dtau if tau is not None else None), None, None, None, None, None, None


def window_attention(qkv, *, H: int, W: int, window: int, shift: int, heads: int, scale: float, table, tau=None):
    """Attention inside the ``window × window`` windows of an ``H × W`` map cyclically shifted by ``shift`` (Swin).

    ``qkv`` ``[B, H·W, 3C]`` is the qkv projection of the tokens in image order (per token ``[3, heads, d]``); returns
    the attention output ``[B, H·W, C]`` in image order.  Exactly ``roll(-shift)`` → window partition → attention →
    window reverse → ``roll(+shift)``, with the score ``scale·q·k + table[relative_position_index, h]`` plus ``-100``
    between tokens of different shifted regions (``shifted_window_mask``).  With ``tau`` (fp32 ``[heads]``) the scores
    are cosine ones, ``tau_h·q̂·k̂`` (SwinV2; ``scale`` is unused).  ``table`` is fp32 ``[(2·window − 1)², heads]``.
    Gradients flow to ``qkv``, ``table`` and ``tau``.  Needs :func:`window_attention_supported`."""
    return _WindowAttnFn.apply(qkv, table, tau, int(H), int(W), int(window), int(shift), int(heads), float(scale))


# --------------------------------------------------------------------------------------
# KV-cache decoding: caches are [b, g, C, d] buffers (g = the key/value heads) (libai_b200.inference.kv_cache.StaticKVCache); ``cache_seqlens``
# (int32 [b]) is the number of rows already held, ``kv_start`` (int32 [b]) the left padding of each sample
# --------------------------------------------------------------------------------------
def _decode_native(x, k_cache) -> bool:
    """The decode kernels take bf16 projections and bf16 or FP8 (E4M3, with row scales) caches with head dim 64 or
    128; other dtypes and head dims run the reference math (as :func:`attention` does)."""
    return (
        use_native(x)
        and x.dtype == torch.bfloat16
        and k_cache.dtype in (torch.bfloat16, torch.float8_e4m3fn)
        and k_cache.shape[-1] in (64, 128)
    )


# FP8 (E4M3) caches hold each row x (the bf16 row a bf16 cache would hold) as the bytes e4m3_rn_satfinite(x / s) and
# the fp32 scale s = amax|x| / 448 (1 for a zero row), ``k_scale`` / ``v_scale`` [b, g, C]; a row reads back as
# float(e)·s.  The decode kernel folds the scales into its scores and probabilities; every other path attends over the
# window dequantized to the projection's dtype.
E4M3_MAX = 448.0


def kv_cache_quantize_ref(x):
    """``(e, s)``: the E4M3 bytes (``float8_e4m3fn``, ``x``'s shape) and fp32 row scales (``x.shape[:-1]``) of the rows
    of ``x`` by the rule above — bit for bit what the append kernel stores for the same bf16 rows."""
    xf = x.float()
    amax = xf.abs().amax(dim=-1)
    # (a tensor divisor: PyTorch's CUDA division by a Python scalar multiplies by its rounded reciprocal)
    s = torch.where(amax == 0, torch.ones_like(amax), amax / torch.full_like(amax, E4M3_MAX))
    return (xf / s[..., None]).to(torch.float8_e4m3fn), s


def kv_cache_dequant(e, s, dtype=torch.bfloat16):
    """The rows ``float(e)·s`` of FP8 bytes ``e`` and their scales ``s``, rounded to ``dtype``."""
    return (e.float() * s[..., None]).to(dtype)


def _check_scales(k_cache, k_scale, v_scale):
    if k_cache.dtype == torch.float8_e4m3fn:
        if k_scale is None or v_scale is None:
            raise ValueError("an FP8 cache needs k_scale and v_scale")
    elif k_scale is not None or v_scale is not None:
        raise ValueError(f"k_scale and v_scale belong to an FP8 cache, not a {k_cache.dtype} one")


def kv_cache_append(qkv, k_cache, v_cache, cache_seqlens, cos=None, sin=None, return_q: bool = True, k_scale=None,
                    v_scale=None, block_table=None):
    """Write k, v of the packed projection ``qkv`` (``[b, s, a, 3d]``, or grouped ``[b, s, g, r + 2, d]``) into rows
    ``cache_seqlens[b] + i`` of the caches ``[b, g, C, d]``.  With
    ``cos/sin`` (fp32 ``[positions, d]``) q and k are first rotated at those positions, exactly as
    :func:`apply_rotary_qkv` with ``pos_offset = cache_seqlens[b]`` does.  Returns q ``[b, s, a, d]`` (rotated when the
    tables are given) when ``return_q``, else None.  FP8 caches (``float8_e4m3fn``) take their row scales ``k_scale``,
    ``v_scale`` (fp32 ``[b, g, C]``) and store each row quantized (:func:`kv_cache_quantize_ref`).
    ``block_table`` (int32 ``[b, max_pages]``): the caches are paged, pools ``[P, g, 64, d]`` (scales ``[P, g, 64]``)
    whose logical row ``j`` of sample ``b`` is row ``j % 64`` of page ``block_table[b, j // 64]``
    (:class:`~libai_b200.inference.kv_cache.PagedKVCache`); the bytes and scales written are those of a contiguous
    cache.  Page ids in ``[0, P)`` for the rows written are the caller's guarantee (the reference path checks them)."""
    _check_scales(k_cache, k_scale, v_scale)
    if _decode_native(qkv, k_cache) and (cos is None or cos.dtype == torch.float32):
        ext = load_ext()
        qkv = qkv if qkv.is_contiguous() else qkv.contiguous()
        if block_table is not None and k_scale is not None:
            q = ext.kv_append_fp8_paged(qkv, k_cache, v_cache, k_scale, v_scale, block_table, cache_seqlens, cos, sin,
                                        bool(return_q))
        elif block_table is not None:
            q = ext.kv_append_paged(qkv, k_cache, v_cache, block_table, cache_seqlens, cos, sin, bool(return_q))
        elif k_scale is not None:
            q = ext.kv_append_fp8(qkv, k_cache, v_cache, k_scale, v_scale, cache_seqlens, cos, sin, bool(return_q))
        else:
            q = ext.kv_append(qkv, k_cache, v_cache, cache_seqlens, cos, sin, bool(return_q))
        count_launch()
        return q if return_q else None
    pages = {} if block_table is None else {"block_table": block_table}
    q = kv_cache_append_ref(qkv, k_cache, v_cache, cache_seqlens, cos, sin, k_scale, v_scale, **pages)
    return q if return_q else None


PAGE_ROWS = 64   # the rows of a page of a paged cache: one key tile of the decode kernel


def _page_ids(block_table, rows, num_pages):
    """The page ids ``[b, n]`` of the logical rows ``rows`` (long ``[b, n]``), checked to be in ``[0, num_pages)``."""
    ids = block_table.long().gather(1, rows // PAGE_ROWS)
    if bool(((ids < 0) | (ids >= num_pages)).any()):
        raise ValueError(f"block_table: a row in use maps to a page outside [0, {num_pages})")
    return ids


def kv_pages_gather(pool, block_table, L: int):
    """The logical rows ``[:L]`` of a paged cache's pool ``[P, g, 64, ...]`` (bytes, or scales ``[P, g, 64]``) through
    ``block_table`` ``[b, max_pages]``, contiguous: ``[b, g, L, ...]``.  Every row below ``L`` must be mapped."""
    rows = torch.arange(L, device=block_table.device)[None].expand(block_table.shape[0], L)
    ids = _page_ids(block_table, rows, pool.shape[0]).to(pool.device)
    off = (rows % PAGE_ROWS).to(pool.device)
    return pool[ids, :, off].transpose(1, 2)   # [b, L, g, ...] -> [b, g, L, ...]


def kv_page_copy(arrays, pairs):
    """Copy page ``src`` to page ``dst`` of every array in ``arrays`` (pools ``[P, ...]``: the K and V pools, and the
    FP8 scales, of every layer of a paged cache) for each ``(src, dst)`` of ``pairs`` (a list, or int32 ``[n, 2]``).
    One launch on the GPU."""
    pairs = torch.as_tensor(pairs, dtype=torch.int32).reshape(-1, 2).cpu()
    if pairs.shape[0] == 0:
        return
    P = arrays[0].shape[0]
    if bool(((pairs < 0) | (pairs >= P)).any()):
        raise ValueError(f"kv_page_copy: page ids must be in [0, {P})")
    if use_native(arrays[0]):
        load_ext().kv_page_copy(list(arrays), pairs)
        count_launch()
        return
    src, dst = pairs[:, 0].long(), pairs[:, 1].long()
    for t in arrays:
        t[dst.to(t.device)] = t[src.to(t.device)]


def kv_cache_append_ref(qkv, k_cache, v_cache, cache_seqlens, cos=None, sin=None, k_scale=None, v_scale=None,
                        block_table=None):
    s_len = qkv.shape[1]
    starts = [int(x) for x in cache_seqlens.tolist()]
    if cos is not None:
        pos = torch.tensor(starts, device=cos.device)[:, None] + torch.arange(s_len, device=cos.device)[None]
        qkv = _rotary_qkv_ref(qkv, cos, sin, position_ids=pos)
    q, k, v = split_qkv(qkv)
    if block_table is not None:   # [b, s, g, d] rows scattered to their pages
        rows = torch.tensor(starts, device=block_table.device)[:, None] + torch.arange(s_len, device=block_table.device)
        ids = _page_ids(block_table, rows, k_cache.shape[0]).to(k_cache.device)
        off = (rows % PAGE_ROWS).to(k_cache.device)
        for cache, scale, x in ((k_cache, k_scale, k), (v_cache, v_scale, v)):
            if scale is None:
                cache[ids, :, off] = x.to(cache.dtype)
            else:
                cache[ids, :, off], scale[ids, :, off] = kv_cache_quantize_ref(x)
        return q
    for b, st in enumerate(starts):
        for cache, scale, x in ((k_cache, k_scale, k[b]), (v_cache, v_scale, v[b])):
            if scale is None:
                cache[b, :, st : st + s_len] = x.transpose(0, 1)
            else:
                cache[b, :, st : st + s_len], scale[b, :, st : st + s_len] = kv_cache_quantize_ref(x.transpose(0, 1))
    return q


def decode_attention(q, k_cache, v_cache, cache_seqlens, kv_start, *, scale: float, splits: int = 0,
                     past: Optional[int] = None, alibi_slopes=None, rel_bias=None, causal: bool = True, k_scale=None,
                     v_scale=None, block_table=None):
    """Attention of ``q [b, s, a, d]`` (new tokens, already appended to the caches; any strides with d contiguous) over
    the caches ``[b, g, C, d]`` (query head ``h`` reads cache head ``h // (a // g)``): query ``i`` of sample ``b`` sees exactly the keys ``kv_start[b] <= j <= cache_seqlens[b] + i``.  Returns
    ``[b, s, a, d]`` contiguous; a query without a visible key gets zeros.  The native kernel takes up to 16 new tokens
    and reads lengths on the device (no host sync; one CUDA-graph capture replays after the lengths change); ``splits``
    > 0 fixes its number of key-range splits.  ``past`` (host int): the rows every sample held before these tokens
    (``cache_seqlens`` all equal to it, as in a :class:`~libai_b200.inference.kv_cache.StaticKVCache`); with it, more
    than 16 new tokens run the causal flash kernel over the cache window ``[:past + s]`` (chunked prefill); over a paged
    bf16 cache (``block_table``) that kernel reads the pages in place (:func:`attention_paged`).
    ``alibi_slopes`` (fp32 ``[a]``, on q's device): ALiBi, every visible score gets ``slope_h·(j − cache_seqlens[b] − i)``
    — the flash kernel's ``slope·(j − i − (sk − sq))`` over the cache window, so both paths score alike.
    ``rel_bias`` (fp32 ``[a, R]``, contiguous, on q's device): T5's relative-position bias, every visible score gets
    ``rel_bias[h, min(cache_seqlens[b] + i − j, R − 1)]``; longer ``past=`` continuations run the flash kernel with the
    dense bias it expands to.
    ``causal=False`` (cross-attention, no bias): every query sees ``kv_start[b] <= j < cache_seqlens[b]`` — a cache the
    new tokens are not in; more than 16 tokens run the rectangular flash kernel over that window (whose end, like
    :func:`attention`'s ``kv_lens``, is at least 1).
    FP8 caches (``float8_e4m3fn``) take their row scales ``k_scale``, ``v_scale`` (fp32 ``[b, g, C]``); the attention is
    that over the dequantized rows.  The decode kernel reads the bytes; every other path dequantizes the window to
    q's dtype first (:func:`kv_cache_dequant`).
    Rows read: the decode kernel reads no row at or past a sample's window end (``cache_seqlens[b] + s``, or
    ``cache_seqlens[b]`` for cross-attention); the flash kernel reads the window ``[:past + s]`` (``[:past]`` for
    cross-attention; without ``past``, any row of the capacity); the reference math reads ``[:max(cache_seqlens) + s]``
    and zeroes the value rows a sample cannot see.  So rows past the window may hold anything, NaN included (an
    uninitialised cache), while invisible rows inside it (before ``kv_start[b]``, or in cross-attention from
    ``cache_seqlens[b]`` to ``past``) may be loaded with weight zero and must be finite, as the appends leave them."""
    _check_scales(k_cache, k_scale, v_scale)
    native = _decode_native(q, k_cache)
    if block_table is not None:
        if rel_bias is not None or not causal:
            raise ValueError("block_table: a paged cache takes no rel_bias and no causal=False")
        if native and q.shape[1] <= 16:
            o = load_ext().decode_attn_paged(q, k_cache, v_cache, block_table, cache_seqlens, kv_start, float(scale),
                                             int(splits), alibi_slopes, k_scale, v_scale)
            count_launch(2)
            return o
        if native and k_scale is None and past is not None:
            return attention_paged(q, k_cache, v_cache, block_table, past, kv_start, scale=scale,
                                   alibi_slopes=alibi_slopes)
        return decode_attention_paged_ref(q, k_cache, v_cache, block_table, cache_seqlens, kv_start, scale=scale,
                                          splits=splits, past=past, alibi_slopes=alibi_slopes, k_scale=k_scale,
                                          v_scale=v_scale)
    if native and q.shape[1] <= 16:
        ext = load_ext()
        extra = () if rel_bias is None and causal else (rel_bias, bool(causal))
        if k_scale is not None:
            extra = (rel_bias, bool(causal), k_scale, v_scale)
        o = ext.decode_attn(q, k_cache, v_cache, cache_seqlens, kv_start, float(scale), int(splits), alibi_slopes,
                            *extra)
        count_launch(2)
        return o
    if k_scale is not None:
        if past is not None:
            L = past + q.shape[1] if causal else past
        else:
            L = k_cache.shape[2] if native else int(cache_seqlens.max()) + (q.shape[1] if causal else 0)
        k_cache = kv_cache_dequant(k_cache[:, :, :L], k_scale[:, :, :L], q.dtype)
        v_cache = kv_cache_dequant(v_cache[:, :, :L], v_scale[:, :, :L], q.dtype)
    if native:
        if not causal:
            if past is not None:   # the kernel loads whole key tiles: rows past the window must not enter P·V
                k_cache, v_cache = k_cache[:, :, :past], v_cache[:, :, :past]
            o = attention(q.permute(0, 2, 1, 3), k_cache, v_cache, causal=False, scale=scale, kv_start=kv_start,
                          kv_lens=cache_seqlens)
            return o.transpose(1, 2)
        if past is not None:
            L = past + q.shape[1]
            bias = None
            if rel_bias is not None:   # [1, a, s, L]: query past + i, key j
                dist = torch.arange(past, L, device=q.device)[:, None] - torch.arange(L, device=q.device)[None, :]
                bias = rel_bias[:, dist.clamp(0, rel_bias.shape[1] - 1)].to(torch.bfloat16)[None]
            o = attention(q.permute(0, 2, 1, 3), k_cache[:, :, :L], v_cache[:, :, :L], causal=True, scale=scale,
                          kv_start=kv_start, alibi_slopes=alibi_slopes, bias=bias)
            return o.transpose(1, 2)   # the kernel's [b, s, a, d] output
    return decode_attention_ref(q, k_cache, v_cache, cache_seqlens, kv_start, scale=scale, alibi_slopes=alibi_slopes,
                                rel_bias=rel_bias, causal=causal)


def attention_paged_supported(q, k_pool) -> bool:
    """True when :func:`attention_paged` runs: bf16 projections on the GPU over a bf16 pool of head dim 64 or 128 (the
    decode kernels' caches, FP8 excepted)."""
    return _decode_native(q, k_pool) and k_pool.dtype == torch.bfloat16


def attention_paged(q, k_pool, v_pool, block_table, past: int, kv_start=None, *, scale: float, alibi_slopes=None):
    """Causal flash attention of the new tokens ``q [b, s, a, d]`` (appended already; any strides with d contiguous)
    over the logical rows ``[:past + s]`` of a paged cache's bf16 pools ``[P, g, 64, d]``, read in place through
    ``block_table`` ``[b, max_pages]``; ``kv_start`` (int32 ``[b]``) and ``alibi_slopes`` as in :func:`attention`.
    Returns ``[b, s, a, d]`` contiguous, bit for bit the flash kernel over the gathered rows
    (``kv_pages_gather(pool, block_table, past + s)``).  Rows at or past ``past + s`` are never read, so they may hold
    anything.  One launch, no host sync; the sm_90a kernel only (see :func:`attention_paged_supported`)."""
    if not attention_paged_supported(q, k_pool):
        raise RuntimeError("attention_paged: needs bf16 q and pools with head dim 64 or 128 on the GPU, with the native "
                           "extension")
    o = load_ext().attn_fwd_paged(q, k_pool, v_pool, block_table, int(past), float(scale), kv_start, alibi_slopes)
    count_launch()
    return o


def varlen_tiles(q_lens, past=None) -> torch.Tensor:
    """The tile list of :func:`attention_paged_varlen` for sequences of ``q_lens`` new tokens after ``past`` rows each
    (default 0): int32 ``[n, 2]`` on the host, ``(sequence, 128-query block)`` for every block of every sequence, the
    blocks that see the most keys (``past`` plus the block's last query) first."""
    past = [0] * len(q_lens) if past is None else [int(p) for p in past]
    tiles = [(n, blk) for n, s in enumerate(q_lens) for blk in range(-(-int(s) // 128))]
    tiles.sort(key=lambda t: -(past[t[0]] + min(128 * (t[1] + 1), int(q_lens[t[0]]))))
    return torch.tensor(tiles, dtype=torch.int32).reshape(-1, 2)


def attention_paged_varlen(q, k_pool, v_pool, block_table, cu_q, past, tiles=None, *, scale: float,
                           alibi_slopes=None, k_scale=None, v_scale=None):
    """Causal attention of ``N`` ragged sequences packed in ``q [T, a, d]`` over their rows of a paged cache's pools
    ``[P, g, 64, d]``: sequence ``n`` owns rows ``cu_q[n] .. cu_q[n + 1]`` of q (int32 ``[N + 1]``, from 0 to T) and
    holds ``past[n]`` rows (int32 ``[N]``) before them in row ``n`` of ``block_table`` ``[N, max_pages]``; its query
    ``i`` sees its logical rows ``[0, past[n] + i]``.  ``alibi_slopes`` as in :func:`attention`.  Returns ``[T, a, d]``.

    On the GPU (bf16, head dim 64 or 128) one launch of the ragged paged flash kernel, one CTA per (128-query tile of
    a sequence, query head) of ``tiles`` (int32 ``[n, 2]`` on q's device, :func:`varlen_tiles`; built here, with a host
    sync, when None); each sequence's rows are bit for bit those of :func:`attention_paged` on that sequence alone.
    Rows of a page past a sequence's window never reach P·V, whatever they hold.  Elsewhere the reference math per
    sequence (:func:`attention_paged_varlen_ref`).

    FP8 pools (``float8_e4m3fn``) take their row scales ``k_scale``, ``v_scale`` (fp32 ``[P, g, 64]``); the attention
    is that over the dequantized rows (:func:`kv_cache_dequant`).  On the GPU the FP8 instances of the same kernel
    dequantize the pages in shared memory, and each sequence's rows are bit for bit this op's over the bf16 pools
    ``kv_cache_dequant(pool, scale)``."""
    _check_scales(k_pool, k_scale, v_scale)
    fp8 = k_scale is not None
    if _decode_native(q, k_pool):
        if tiles is None:
            tiles = varlen_tiles(cu_q.diff().tolist(), past.tolist()).to(q.device)
        ext = load_ext()
        if fp8:
            o = ext.attn_fwd_paged_varlen_fp8(q, k_pool, v_pool, k_scale, v_scale, block_table, cu_q, past, tiles,
                                              float(scale), alibi_slopes)
        else:
            o = ext.attn_fwd_paged_varlen(q, k_pool, v_pool, block_table, cu_q, past, tiles, float(scale),
                                          alibi_slopes)
        count_launch()
        return o
    return attention_paged_varlen_ref(q, k_pool, v_pool, block_table, cu_q, past, scale=scale,
                                      alibi_slopes=alibi_slopes, k_scale=k_scale, v_scale=v_scale)


def attention_paged_varlen_ref(q, k_pool, v_pool, block_table, cu_q, past, *, scale: float, alibi_slopes=None,
                               k_scale=None, v_scale=None):
    """:func:`attention_paged_varlen` by the reference math: per sequence, its rows ``[:past[n] + s_n]`` gathered
    through its table row (and dequantized to q's dtype for FP8 pools), then :func:`attention_ref` (causal,
    bottom-right aligned, with the ALiBi bias ``slope_h·(j − past[n] − i)``)."""
    _check_scales(k_pool, k_scale, v_scale)
    cu, pa = [int(x) for x in cu_q.tolist()], [int(x) for x in past.tolist()]
    o = torch.zeros_like(q)
    for n in range(len(pa)):
        s = cu[n + 1] - cu[n]
        if s == 0:
            continue
        L = pa[n] + s
        k = kv_pages_gather(k_pool, block_table[n : n + 1], L)
        v = kv_pages_gather(v_pool, block_table[n : n + 1], L)
        if k_scale is not None:
            k = kv_cache_dequant(k, kv_pages_gather(k_scale, block_table[n : n + 1], L), q.dtype)
            v = kv_cache_dequant(v, kv_pages_gather(v_scale, block_table[n : n + 1], L), q.dtype)
        qn = q[cu[n] : cu[n + 1]].transpose(0, 1)[None]   # [1, a, s, d]
        bias = None
        if alibi_slopes is not None:
            dist = torch.arange(L, device=q.device)[None, :] - torch.arange(pa[n], L, device=q.device)[:, None]
            bias = (alibi_slopes.float().to(q.device)[:, None, None] * dist[None].float())[None]
        o[cu[n] : cu[n + 1]] = attention_ref(qn, k.to(q.dtype), v.to(q.dtype), causal=True, scale=scale,
                                             bias=bias)[0].transpose(0, 1)
    return o


def kv_cache_append_paged_varlen(qkv, k_pool, v_pool, block_table, cu_q, past, cos=None, sin=None, k_scale=None,
                                 v_scale=None):
    """Write k, v of the packed projection ``qkv`` (``[1, T, a, 3d]`` or ``[1, T, g, r + 2, d]``) of ``N`` ragged
    sequences into a paged cache's pools ``[P, g, 64, d]``: token ``t`` of sequence ``n`` (``cu_q[n] <= t < cu_q[n +
    1]``, int32 ``[N + 1]`` from 0 to T) at its logical row ``past[n] + t − cu_q[n]`` of row ``n`` of ``block_table``
    ``[N, max_pages]``, q and k rotated at that position by ``cos/sin`` when given.  Returns q ``[1, T, a, d]``.  On
    the GPU one launch of the ragged append, whose bytes are :func:`kv_cache_append`'s per sequence; elsewhere
    :func:`kv_cache_append_ref` per sequence.  FP8 pools (``float8_e4m3fn``) take their row scales ``k_scale``,
    ``v_scale`` (fp32 ``[P, g, 64]``) and store each row quantized, bytes and scales those of :func:`kv_cache_append`
    per sequence."""
    _check_scales(k_pool, k_scale, v_scale)
    if _decode_native(qkv, k_pool) and (cos is None or cos.dtype == torch.float32):
        qkv = qkv if qkv.is_contiguous() else qkv.contiguous()
        ext = load_ext()
        if k_scale is not None:
            q = ext.kv_append_fp8_paged_varlen(qkv, k_pool, v_pool, k_scale, v_scale, block_table, cu_q, past, cos,
                                               sin, True)
        else:
            q = ext.kv_append_paged_varlen(qkv, k_pool, v_pool, block_table, cu_q, past, cos, sin, True)
        count_launch()
        return q
    return kv_cache_append_paged_varlen_ref(qkv, k_pool, v_pool, block_table, cu_q, past, cos, sin, k_scale, v_scale)


def kv_cache_append_paged_varlen_ref(qkv, k_pool, v_pool, block_table, cu_q, past, cos=None, sin=None, k_scale=None,
                                     v_scale=None):
    cu, pa = [int(x) for x in cu_q.tolist()], past.to(torch.int32)
    qs = []
    for n in range(len(cu) - 1):
        if cu[n + 1] > cu[n]:
            qs.append(kv_cache_append_ref(qkv[:, cu[n] : cu[n + 1]], k_pool, v_pool, pa[n : n + 1], cos, sin,
                                          k_scale, v_scale, block_table=block_table[n : n + 1]))
    return torch.cat(qs, dim=1)


def decode_attention_paged_ref(q, k_pool, v_pool, block_table, cache_seqlens, kv_start, *, scale: float, splits=0,
                               past: Optional[int] = None, alibi_slopes=None, k_scale=None, v_scale=None):
    """:func:`decode_attention` over a paged cache by its logical rows: the rows ``[:L]`` gathered through the table
    (``L = past + s`` with ``past``, else ``max(cache_seqlens) + s``) into contiguous caches, then the contiguous call
    (the flash kernel beyond 16 new tokens on the GPU, the reference math on the CPU)."""
    L = past + q.shape[1] if past is not None else int(cache_seqlens.max()) + q.shape[1]
    k, v = kv_pages_gather(k_pool, block_table, L), kv_pages_gather(v_pool, block_table, L)
    scales = {}
    if k_scale is not None:
        scales = {"k_scale": kv_pages_gather(k_scale, block_table, L), "v_scale": kv_pages_gather(v_scale, block_table, L)}
    return decode_attention(q, k, v, cache_seqlens, kv_start, scale=scale, splits=splits, past=past,
                            alibi_slopes=alibi_slopes, **scales)


def decode_attention_ref(q, k_cache, v_cache, cache_seqlens, kv_start, *, scale: float, alibi_slopes=None,
                         rel_bias=None, causal: bool = True, k_scale=None, v_scale=None):
    """:func:`attention_ref` over the window ``[:L]`` of the caches (``L = max(cache_seqlens) + s``) with the mask built
    from ``kv_start`` and causality among the new tokens, and the ALiBi bias ``slope_h·(j − (cache_seqlens[b] + i))``
    when ``alibi_slopes`` is given, or T5's ``rel_bias[h, min(cache_seqlens[b] + i − j, R − 1)]`` when ``rel_bias`` is.
    ``causal=False``: every query sees ``kv_start[b] <= j < cache_seqlens[b]`` (``L = max(cache_seqlens)``).  FP8
    caches with ``k_scale`` / ``v_scale``: over the window dequantized to q's dtype."""
    _check_scales(k_cache, k_scale, v_scale)
    s_len = q.shape[1]
    lens = cache_seqlens.long()
    L = int(lens.max()) + (s_len if causal else 0)
    if k_scale is not None:
        k_cache = kv_cache_dequant(k_cache[:, :, :L], k_scale[:, :, :L], q.dtype)
        v_cache = kv_cache_dequant(v_cache[:, :, :L], v_scale[:, :, :L], q.dtype)
    j = torch.arange(L, device=q.device)[None, None, :]
    i = torch.arange(s_len, device=q.device)[None, :, None]
    end = lens[:, None, None] + i if causal else lens[:, None, None] - 1
    visible = (j >= kv_start.long()[:, None, None]) & (j <= end)                              # [b, s, L]
    # a masked score gets probability 0, but 0 · NaN is NaN: a shorter sample's rows past its own window end (never
    # written) must not reach P @ V
    v_cache = torch.where(visible.any(1)[:, None, :, None], v_cache[:, :, :L], 0)
    bias = None
    if alibi_slopes is not None:
        rel = (j - (lens[:, None, None] + i)).float()                                          # [b, s, L]
        bias = alibi_slopes.float()[None, :, None, None] * rel[:, None]                        # [b, a, s, L]
    if rel_bias is not None:
        dist = (lens[:, None, None] + i - j).clamp(0, rel_bias.shape[1] - 1)                   # [b, s, L]
        bias = rel_bias[:, dist].permute(1, 0, 2, 3)                                           # [b, a, s, L]
    o = attention_ref(q.permute(0, 2, 1, 3), k_cache[:, :, :L], v_cache[:, :, :L], causal=False, scale=scale,
                      mask=visible[:, None], bias=bias)
    o = o.masked_fill(~visible.any(-1)[:, None, :, None], 0)
    return o.permute(0, 2, 1, 3).contiguous()


# --------------------------------------------------------------------------------------
# vocab-parallel softmax cross entropy
# --------------------------------------------------------------------------------------
class _VocabParallelCE(torch.autograd.Function):
    """Per-token CE over logits whose last dim is split across ``group``.

    fwd: local (max, sum-exp, target-logit) → 3 tiny all-reduces → loss; bwd: softmax − onehot
    written in place of the saved logits (no extra ``[T, V/t]`` buffer)."""

    @staticmethod
    def forward(ctx, logits, labels, vocab_start, group):
        T, Vl = logits.shape
        world = 1 if group is None else dist.get_world_size(group)
        native = use_native(logits) and logits.dtype in (torch.bfloat16, torch.float32)
        if native:
            ext = load_ext()
            mx, se, tgt = ext.ce_stats(logits, labels, vocab_start)
            count_launch()
        else:
            lf = logits.float()
            mx = lf.max(dim=-1).values
            se = torch.exp(lf - mx[:, None]).sum(-1)
            local = labels - vocab_start
            inside = (local >= 0) & (local < Vl)
            idx = local.clamp(0, Vl - 1)
            tgt = torch.where(inside, lf.gather(1, idx[:, None]).squeeze(1), torch.zeros_like(mx))
        if world > 1:
            gmx = mx.clone()
            dist.all_reduce(gmx, op=dist.ReduceOp.MAX, group=group)
            se = se * torch.exp(mx - gmx)
            packed = torch.stack([se, tgt])
            dist.all_reduce(packed, group=group)
            se, tgt = packed[0], packed[1]
            mx = gmx
        lse = mx + torch.log(se)
        loss = lse - tgt
        ctx.save_for_backward(logits, labels, lse)
        ctx.vocab_start = vocab_start
        ctx.native = native
        return loss

    @staticmethod
    def backward(ctx, gloss):
        logits, labels, lse = ctx.saved_tensors
        if ctx.native:
            ext = load_ext()
            g = ext.ce_bwd(logits, labels, lse, gloss.contiguous().float(), ctx.vocab_start)
            count_launch()
            return g, None, None, None
        Vl = logits.shape[1]
        p = torch.exp(logits.float() - lse[:, None])
        local = labels - ctx.vocab_start
        inside = (local >= 0) & (local < Vl)
        idx = local.clamp(0, Vl - 1)
        p.scatter_add_(1, idx[:, None], -inside.to(p.dtype)[:, None])
        return (p * gloss.float()[:, None]).to(logits.dtype), None, None, None


def vocab_parallel_cross_entropy(logits, labels, vocab_start: int = 0, group=None):
    """logits ``[..., V/t]``, labels ``[...]`` (global ids) → per-token loss ``[...]`` (fp32)."""
    shp = labels.shape
    out = _VocabParallelCE.apply(logits.reshape(-1, logits.shape[-1]), labels.reshape(-1), vocab_start, group)
    return out.view(shp)


# --------------------------------------------------------------------------------------
# embedding
# --------------------------------------------------------------------------------------
class _EmbeddingFn(torch.autograd.Function):
    """Row gather; the backward scatters ``gy`` straight into the table's fp32 ``main_grad`` with vector reductions
    (no sort / segment-reduce / temporary gradient the size of the table, and no later fold of ``p.grad``)."""

    @staticmethod
    def forward(ctx, ids, table, vocab_start):
        ext = load_ext()
        flat = ids.reshape(-1).contiguous()
        out = ext.embedding_fwd(flat, table, vocab_start)
        count_launch()
        ctx.save_for_backward(flat)
        ctx.table = table
        ctx.vocab_start = vocab_start
        return out.view(*ids.shape, table.shape[1])

    @staticmethod
    def backward(ctx, gy):
        (flat,) = ctx.saved_tensors
        table = ctx.table
        g2 = gy.reshape(-1, gy.shape[-1]).contiguous()
        ext = load_ext()
        count_launch()
        main_grad = _main_grad(table)
        if main_grad is not None:
            ext.embedding_bwd(flat, g2, main_grad, ctx.vocab_start)
            table.grad_added_to_main_grad = True
            return None, None, None
        grad = torch.zeros(table.shape, dtype=torch.float32, device=table.device)
        ext.embedding_bwd(flat, g2, grad, ctx.vocab_start)
        return None, grad.to(table.dtype), None


def embedding(ids, table, vocab_start: int = 0):
    """Row gather with zero rows for ids outside ``[vocab_start, vocab_start + rows)``."""
    rows = table.shape[0]
    if (use_native(table) and table.dtype == torch.bfloat16 and table.dim() == 2 and table.shape[1] % 8 == 0
            and table.is_contiguous() and ids.dtype == torch.long):
        return _EmbeddingFn.apply(ids, table, int(vocab_start))
    local = ids - vocab_start
    inside = (local >= 0) & (local < rows)
    out = F.embedding(local.clamp(0, rows - 1), table)
    return out * inside.unsqueeze(-1).to(out.dtype)


# --------------------------------------------------------------------------------------
# rotary position embedding
# --------------------------------------------------------------------------------------
def rotate_half(x):
    x1, x2 = x[..., : x.shape[-1] // 2], x[..., x.shape[-1] // 2 :]
    return torch.cat((-x2, x1), dim=-1)


class _RopeQKVFn(torch.autograd.Function):
    """Rotary embedding on every q and k of the packed projection (``[b, s, a, 3d]`` or ``[b, s, g, r + 2, d]``) in one
    pass (v copied);
    the backward applies the inverse rotation to the packed ``dqkv`` into a new tensor: the incoming gradient may be
    the caller's own tensor or one autograd also hands to another branch, so it is never overwritten."""

    @staticmethod
    def forward(ctx, qkv, cos, sin, pos_offset, positions=None):
        ext = load_ext()
        ctx.save_for_backward(cos, sin, positions)
        ctx.pos_offset = pos_offset
        count_launch()
        return ext.rope_qkv(qkv, cos, sin, pos_offset, False, False, positions)

    @staticmethod
    def backward(ctx, g):
        ext = load_ext()
        cos, sin, positions = ctx.saved_tensors
        count_launch()
        g = g if g.is_contiguous() else g.contiguous()
        return ext.rope_qkv(g, cos, sin, ctx.pos_offset, True, False, positions), None, None, None, None


def apply_rotary_qkv(qkv, cos, sin, pos_offset: int = 0, position_ids=None):
    """qkv ``[b, s, a, 3d]`` (per-head ``[q|k|v]``) or grouped ``[b, s, g, r + 2, d]`` (per group ``q_0 .. q_{r-1}, k,
    v``); cos/sin fp32 ``[max_pos, d]``; token ``i`` of the sequence uses position ``i + pos_offset``, or
    ``position_ids[b, i]`` (int32 ``[b, s]``, packed sequences; clamped to the tables) when given."""
    if use_native(qkv) and qkv.dtype == torch.bfloat16 and cos.dtype == torch.float32 and qkv.is_contiguous():
        return _RopeQKVFn.apply(qkv, cos, sin, int(pos_offset), position_ids)
    return _rotary_qkv_ref(qkv, cos, sin, pos_offset, position_ids)


def _rotary_qkv_ref(qkv, cos, sin, pos_offset=0, position_ids=None):
    """The reference math of :func:`apply_rotary_qkv` (reference projects/Llama/llama.py:31-43)."""
    s_len = qkv.shape[1]
    if position_ids is not None:   # [b, s, 1, d] (+ a group axis below)
        idx = position_ids.to(device=cos.device, dtype=torch.long).clamp(0, cos.shape[0] - 1)
        c, sn = cos[idx][:, :, None, :].to(qkv.dtype), sin[idx][:, :, None, :].to(qkv.dtype)
    else:
        c = cos[pos_offset : pos_offset + s_len, None, :].to(qkv.dtype)
        sn = sin[pos_offset : pos_offset + s_len, None, :].to(qkv.dtype)
    if qkv.dim() == 5:
        r = qkv.shape[3] - 2
        c, sn = c.unsqueeze(-2), sn.unsqueeze(-2)
        qk = qkv[..., : r + 1, :]
        return torch.cat([qk * c + rotate_half(qk) * sn, qkv[..., r + 1 :, :]], dim=3)
    d = qkv.shape[-1] // 3
    q, k, v = qkv[..., :d], qkv[..., d : 2 * d], qkv[..., 2 * d :]
    return torch.cat([q * c + rotate_half(q) * sn, k * c + rotate_half(k) * sn, v], dim=-1)


# ChatGLM2/3 ("GLM") rotary: the first half of every head rotates in interleaved pairs by an fp32 ``[positions, d/4, 2]``
# (cos, sin) table (reference projects/ChatGLM/chatglm.py ``RotaryEmbedding`` / ``apply_rotary_pos_emb``)
def glm_rope_table(seq_len: int, rotary_dim: int, base: float = 10000.0, device=None):
    """``[seq_len, rotary_dim/2, 2]`` (cos, sin) table; ``rotary_dim`` = half of the head dimension."""
    theta = 1.0 / (base ** (torch.arange(0, rotary_dim, 2, dtype=torch.float32, device=device) / rotary_dim))
    idx = torch.outer(torch.arange(seq_len, dtype=torch.float32, device=device), theta)
    return torch.stack([idx.cos(), idx.sin()], dim=-1)


def apply_glm_rotary(x: torch.Tensor, table: torch.Tensor) -> torch.Tensor:
    """x ``[b, s, heads, d]``; rotates interleaved pairs of the first ``2·table.shape[-2]`` channels by the first ``s``
    rows of ``table``, in fp32."""
    b, s, h, d = x.shape
    rot = table.shape[-2] * 2
    xr, xp = x[..., :rot], x[..., rot:]
    xr = xr.float().reshape(b, s, h, rot // 2, 2)
    c = table[:s].view(1, s, 1, rot // 2, 2)
    out = torch.stack([xr[..., 0] * c[..., 0] - xr[..., 1] * c[..., 1], xr[..., 1] * c[..., 0] + xr[..., 0] * c[..., 1]], -1)
    return torch.cat([out.flatten(3).to(x.dtype), xp], dim=-1)


def apply_glm_rotary_qkv_ref(mixed, *, heads: int, kv_heads: int, table, pos_offset: int = 0, position_ids=None,
                             grouped: bool = False, pos_base=None):
    """:func:`apply_glm_rotary_qkv` in PyTorch: :func:`apply_glm_rotary` on q and k, then stacked (and, per-head,
    repeated) into the packed layout."""
    b, s, _ = mixed.shape
    a, g = heads, kv_heads
    d = mixed.shape[-1] // (a + 2 * g)
    if pos_base is not None:
        rope = table[pos_base[0].long() + pos_offset + torch.arange(s, device=table.device)]
    else:
        rope = table[position_ids[0].long()] if position_ids is not None else table[pos_offset : pos_offset + s]
    q, k, v = mixed.split([a * d, g * d, g * d], dim=-1)
    q = apply_glm_rotary(q.view(b, s, a, d), rope)
    k = apply_glm_rotary(k.view(b, s, g, d), rope)
    v = v.view(b, s, g, d)
    if grouped:
        return torch.cat([q.view(b, s, g, a // g, d), k.unsqueeze(3), v.unsqueeze(3)], dim=3)
    return torch.cat([q, k.repeat_interleave(a // g, dim=2), v.repeat_interleave(a // g, dim=2)], dim=-1)


class _GlmRotaryQKVFn(torch.autograd.Function):
    """The GLM rotary pass from the fused projection to a packed layout; the backward sums the per-head K/V copies and
    rotates back in one pass."""

    @staticmethod
    def forward(ctx, mixed, heads, kv_heads, table, pos_offset, position_ids, grouped, pos_base):
        ext = load_ext()
        ctx.save_for_backward(table, position_ids, pos_base)
        ctx.geom = (heads, kv_heads, pos_offset)
        count_launch()
        return ext.glm_rotary_qkv(mixed, heads, kv_heads, table, pos_offset, position_ids, grouped, pos_base)

    @staticmethod
    def backward(ctx, g):
        ext = load_ext()
        table, position_ids, pos_base = ctx.saved_tensors
        heads, kv_heads, pos_offset = ctx.geom
        count_launch()
        dmixed = ext.glm_rotary_qkv_bwd(g.contiguous(), heads, kv_heads, table, pos_offset, position_ids, pos_base)
        return dmixed, None, None, None, None, None, None, None


def apply_glm_rotary_qkv(mixed, *, heads: int, kv_heads: int, table, pos_offset: int = 0, position_ids=None,
                         grouped: bool = False, pos_base=None):
    """ChatGLM's fused projection ``mixed`` ``[b, s, (a + 2g)·d]`` (all ``a`` q heads, then the ``g`` k heads, then the
    ``g`` v heads) → the packed layout the attention kernels read, q and k rotated by the GLM rotary (:func:`apply_glm_rotary`
    with the fp32 ``table`` ``[P, d/4, 2]`` of :func:`glm_rope_table`): per-head ``[b, s, a, 3d]`` (query head ``h``
    with copies of K/V group ``h // (a // g)``, for :func:`attention_qkvpacked`), or with ``grouped`` ``[b, s, g, a/g + 2,
    d]`` (for :func:`kv_cache_append`).  Token ``i`` sits at position ``pos_offset + i``, or ``position_ids[0, i]``
    (``[b, s]``; the first row serves the whole batch) when given.  The native kernel's forward is bit-identical to
    :func:`apply_glm_rotary_qkv_ref`; its backward sums the K/V copies in fp32 and rounds once.
    ``pos_base`` (int32 ``[>= 1]``, not with ``position_ids``): token ``i`` sits at ``pos_base[0] + pos_offset + i``,
    read on the device, forward and backward.  A cached step passes its cache's lengths, so that the step holds no
    host-side position and a CUDA graph of it replays at the cache's current length."""
    if pos_base is not None and position_ids is not None:
        raise ValueError("position_ids and pos_base exclude each other")
    if use_native(mixed) and mixed.dtype == torch.bfloat16 and table.dtype == torch.float32:
        if position_ids is not None:
            position_ids = position_ids.to(device=mixed.device, dtype=torch.int32).contiguous()
        return _GlmRotaryQKVFn.apply(mixed.contiguous(), int(heads), int(kv_heads), table.contiguous(), int(pos_offset),
                                     position_ids, bool(grouped), pos_base)
    return apply_glm_rotary_qkv_ref(mixed, heads=heads, kv_heads=kv_heads, table=table, pos_offset=pos_offset,
                                    position_ids=position_ids, grouped=grouped, pos_base=pos_base)


# --------------------------------------------------------------------------------------
# fused softmax variants kept for exact-parity tests
# --------------------------------------------------------------------------------------
def fused_scale_mask_softmax(scores, mask=None, scale: float = 1.0, causal: bool = False, fill: float = -10000.0):
    s = scores.float() * scale
    if causal:
        sq, sk = s.shape[-2:]
        tril = torch.ones(sq, sk, dtype=torch.bool, device=s.device).tril(diagonal=sk - sq)
        s = torch.where(tril, s, torch.full_like(s, fill))
    if mask is not None:
        s = torch.where(mask.bool(), s, torch.full_like(s, fill))
    return torch.softmax(s, dim=-1).to(scores.dtype)


def swiglu(gate, up):
    """``silu(gate) * up`` (reference projects/Llama/llama.py:111-113)."""
    if use_native(gate) and gate.dtype == torch.bfloat16:
        return _SwigluFn.apply(gate, up)
    return F.silu(gate) * up


class _SwigluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gate, up):
        ext = load_ext()
        g, u = gate.contiguous(), up.contiguous()
        ctx.save_for_backward(g, u)
        count_launch()
        return ext.swiglu_fwd(g, u)

    @staticmethod
    def backward(ctx, gy):
        ext = load_ext()
        g, u = ctx.saved_tensors
        count_launch()
        dg, du = ext.swiglu_bwd(gy.contiguous(), g, u)
        return dg, du
