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


def _bias_grad(ext, g2, bias):
    """Column sums of ``g2`` as the gradient of ``bias``: accumulated straight into ``bias.main_grad`` (fp32 slice of
    the optimizer's flat gradient buffer) when the parameter owns one – no temporary, no bf16 round trip, no
    per-parameter add kernel later – otherwise returned as a tensor for autograd."""
    count_launch()
    main_grad = getattr(bias, "main_grad", None)
    if main_grad is not None and main_grad.dtype == torch.float32:
        ext.colsum(g2, main_grad)
        bias.grad_added_to_main_grad = True
        return None
    return ext.colsum(g2).to(bias.dtype)


class _LinearFn(torch.autograd.Function):
    """Native linear: fwd ``NT`` GEMM with fused bias/activation epilogue, dgrad ``NN`` GEMM,
    wgrad ``TN`` split-K GEMM accumulating in fp32 straight into ``weight.main_grad`` when the
    parameter owns one (gradient-accumulation fusion)."""

    @staticmethod
    def forward(ctx, x, w, bias, act):
        ext = load_ext()
        x2 = x.reshape(-1, x.shape[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        need_pre = act not in (None, "none") and (x.requires_grad or w.requires_grad)
        y, pre = _linear_fwd_any(ext, x2, w, bias, _ACT_IDS[act], need_pre)
        ctx.act = act
        ctx.has_bias = bias is not None
        ctx.bias_param = bias
        ctx.save_for_backward(x2, w, pre if need_pre else None)
        ctx.x_shape = x.shape
        return y.view(*x.shape[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, gy):
        ext = load_ext()
        x2, w, pre = ctx.saved_tensors
        g2 = gy.reshape(-1, gy.shape[-1])
        if not g2.is_contiguous():
            g2 = g2.contiguous()
        if ctx.act not in (None, "none"):
            g2 = ext.act_bwd(g2, pre, _ACT_IDS[ctx.act])
            count_launch()
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            gx = ext.gemm(g2, w, 1, None, None, False, torch.bfloat16)  # NN: [M,N]x[N,K]
            count_launch()
            gx = gx.view(ctx.x_shape)
        if ctx.needs_input_grad[1]:
            main_grad = getattr(w, "main_grad", None)
            if main_grad is not None:
                ext.gemm(g2, x2, 2, None, main_grad, True, torch.float32)  # TN accumulate
                gw = None
                w.grad_added_to_main_grad = True
            else:
                gw = ext.gemm(g2, x2, 2, None, None, False, torch.float32).to(w.dtype)
            count_launch()
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = _bias_grad(ext, g2, ctx.bias_param)
        return gx, gw, gb, None


def linear(x, w, bias=None, act: Optional[str] = None):
    """``act(x @ w.T + bias)``; ``w`` is ``[out, in]``."""
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
        x2 = x.reshape(-1, x.shape[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        h, pre = _linear_fwd_any(ext, x2, w1, b1, _ACT_IDS[act], True)
        # with a residual, the second bias and the block's residual add ride in the epilogue of the second GEMM
        res2 = residual.reshape(-1, w2.shape[0]).contiguous() if residual is not None else None
        y, _ = _linear_fwd_any(ext, h, w2, b2, 0, False, res2)
        ctx.act = act
        ctx.save_for_backward(x2, w1, w2, pre, h)
        ctx.x_shape = x.shape
        ctx.has_bias = b1 is not None
        ctx.bias_param = b1
        ctx.bias2_param = b2
        ctx.has_res = residual is not None
        return y.view(*x.shape[:-1], w2.shape[0])

    @staticmethod
    def backward(ctx, gy):
        ext = load_ext()
        x2, w1, w2, pre, h = ctx.saved_tensors
        g2 = gy.reshape(-1, gy.shape[-1])
        if not g2.is_contiguous():
            g2 = g2.contiguous()
        # bias gradient of the first linear = column sums of dpre, accumulated into b1.main_grad by the dgrad call (a
        # column-sum pass with a fixed summation order, launched right behind the GEMM)
        b1 = ctx.bias_param
        fused_gb1 = None
        if ctx.has_bias and ctx.needs_input_grad[2] and ops.fused_bias_grad():
            mg = getattr(b1, "main_grad", None)
            if mg is not None and mg.dtype == torch.float32 and mg.is_contiguous():
                fused_gb1 = mg
        dpre = ext.dgrad_actgrad(g2, w2, pre, _ACT_IDS[ctx.act], fused_gb1)
        count_launch()

        def wgrad(g, inp, w):
            main_grad = getattr(w, "main_grad", None)
            count_launch()
            if main_grad is not None:
                ext.gemm(g, inp, 2, None, main_grad, True, torch.float32)
                w.grad_added_to_main_grad = True
                return None
            return ext.gemm(g, inp, 2, None, None, False, torch.float32).to(w.dtype)

        gw2 = wgrad(g2, h, w2) if ctx.needs_input_grad[3] else None
        gw1 = wgrad(dpre, x2, w1) if ctx.needs_input_grad[1] else None
        gb1 = None
        if fused_gb1 is not None:
            b1.grad_added_to_main_grad = True
        elif ctx.has_bias and ctx.needs_input_grad[2]:
            gb1 = _bias_grad(ext, dpre, ctx.bias_param)
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
    if use_native(x, w1) and _gemm_ok(x, w1) and _gemm_ok(x.new_empty(1, w1.shape[0]), w2):
        if residual is not None:
            return _MLPFn.apply(x, w1, b1, w2, act, b2, residual)
        return _MLPFn.apply(x, w1, b1, w2, act)
    y = linear(linear(x, w1, b1, act), w2, b2)
    return y if residual is None else y + residual


class _LinearResidualFn(torch.autograd.Function):
    """``x @ wᵀ + bias + residual`` with bias and residual added in the GEMM epilogue."""

    @staticmethod
    def forward(ctx, x, w, bias, residual):
        ext = load_ext()
        x2 = x.reshape(-1, x.shape[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        y, _ = _linear_fwd_any(ext, x2, w, bias, 0, False, residual.reshape(-1, w.shape[0]).contiguous())
        ctx.bias_param = bias
        ctx.save_for_backward(x2, w)
        ctx.x_shape = x.shape
        return y.view(*x.shape[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, gy):
        ext = load_ext()
        x2, w = ctx.saved_tensors
        g2 = gy.reshape(-1, gy.shape[-1])
        if not g2.is_contiguous():
            g2 = g2.contiguous()
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            gx = ext.gemm(g2, w, 1, None, None, False, torch.bfloat16).view(ctx.x_shape)
            count_launch()
        if ctx.needs_input_grad[1]:
            main_grad = getattr(w, "main_grad", None)
            if main_grad is not None:
                ext.gemm(g2, x2, 2, None, main_grad, True, torch.float32)
                w.grad_added_to_main_grad = True
            else:
                gw = ext.gemm(g2, x2, 2, None, None, False, torch.float32).to(w.dtype)
            count_launch()
        if ctx.bias_param is not None and ctx.needs_input_grad[2]:
            gb = _bias_grad(ext, g2, ctx.bias_param)
        return gx, gw, gb, gy


def linear_bias_residual(x, w, bias, residual):
    """``x @ wᵀ + bias + residual`` (output projection of a block, dropout-free)."""
    if use_native(x, w) and _gemm_ok(x, w) and residual is not None and residual.dtype == torch.bfloat16:
        return _LinearResidualFn.apply(x, w, bias, residual)
    y = linear(x, w, bias)
    return y if residual is None else y + residual


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
        wg = getattr(weight, "main_grad", None)
        bg = getattr(ctx.bias_param, "main_grad", None) if ctx.has_bias else None
        if wg is not None and wg.dtype == torch.float32 and (not ctx.has_bias or bg is not None):
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


def visible_keys(sq: int, sk: int, *, causal: bool, kv_start=None, kv_lens=None, device=None):
    """Boolean ``[b|1, 1, sq, sk]`` visibility of the flash kernels: key ``j`` is visible to query ``i`` of sample ``b``
    iff ``kv_start[b] <= j < max(1, kv_lens[b])`` (defaults ``0`` and ``sk``) and, when ``causal``,
    ``j <= i + sk - sq`` (bottom-right alignment)."""
    j = torch.arange(sk, device=device)
    vis = torch.ones(1, sq, sk, dtype=torch.bool, device=device)
    if causal:
        vis = vis & (j[None, :] <= torch.arange(sq, device=device)[:, None] + (sk - sq))[None]
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
    slopes), per-sample key windows (``kv_start`` / ``kv_lens``) and Philox dropout on the probabilities — all inside
    the wgmma kernels."""

    @staticmethod
    def forward(ctx, q, k, v, causal, scale, bias, alibi_slopes, p_drop, kv_lens, kv_start=None):
        ext = load_ext()
        b = _prep_bias(bias, q)
        o, lse, rng_state = ext.attn_fwd(q, k, v, causal, scale, kv_lens, b, alibi_slopes, p_drop,
                                         tp_rng_salt(True) if p_drop > 0 else 0, kv_start)
        count_launch()
        ctx.save_for_backward(q, k, v, o, lse, b, alibi_slopes, rng_state, kv_lens, kv_start)
        ctx.causal, ctx.scale, ctx.p_drop = causal, scale, p_drop
        ctx.bias_shape = None if bias is None else (bias.shape, bias.dtype)
        return o

    @staticmethod
    def backward(ctx, go):
        ext = load_ext()
        q, k, v, o, lse, b, slopes, rng_state, kv_lens, kv_start = ctx.saved_tensors
        dbias = None
        if b is not None and ctx.needs_input_grad[5]:
            dbias = torch.zeros(b.shape, dtype=torch.float32, device=b.device)
            if dbias.stride() != b.stride():
                dbias = torch.empty_strided(b.shape, b.stride(), dtype=torch.float32, device=b.device).zero_()
        dq, dk, dv, _ = ext.attn_bwd(go, q, k, v, o, lse, ctx.causal, ctx.scale, kv_lens, b, slopes, dbias, ctx.p_drop,
                                     rng_state if ctx.p_drop > 0 else None, kv_start)
        count_launch(3)
        gb = None
        if dbias is not None:
            shape, dtype = ctx.bias_shape
            gb = dbias.to(dtype).reshape(shape)
        return dq, dk, dv, None, None, gb, None, None, None, None


class _FlashAttnPackedFn(torch.autograd.Function):
    """Self-attention straight from the packed QKV projection ``[b, s, a, 3d]`` (per-head ``[q|k|v]``) or
    ``[b, s, g, r + 2, d]`` (grouped): the kernels read q/k/v through strided TMA maps and the backward writes one packed
    ``dqkv`` of the same layout – no slicing, no expanded K/V, no gradient accumulation kernels around the attention."""

    @staticmethod
    def forward(ctx, qkv, causal, scale, kv_lens, p_drop=0.0, alibi_slopes=None):
        ext = load_ext()
        q, k, v = _packed_views(qkv)
        o, lse, rng_state = ext.attn_fwd(q, k, v, causal, scale, kv_lens, None, alibi_slopes, p_drop,
                                         tp_rng_salt(True) if p_drop > 0 else 0)
        count_launch()
        ctx.save_for_backward(qkv, o, lse, kv_lens, rng_state, alibi_slopes)
        ctx.causal, ctx.scale, ctx.p_drop = causal, scale, p_drop
        return o.permute(0, 2, 1, 3)  # [b, s, a, d] contiguous

    @staticmethod
    def backward(ctx, go):
        ext = load_ext()
        qkv, o, lse, kv_lens, rng_state, slopes = ctx.saved_tensors
        q, k, v = _packed_views(qkv)
        _, _, _, dqkv = ext.attn_bwd(go.permute(0, 2, 1, 3), q, k, v, o, lse, ctx.causal, ctx.scale, kv_lens, None, slopes,
                                     None, ctx.p_drop, rng_state if ctx.p_drop > 0 else None)
        count_launch(3)
        return dqkv.view(qkv.shape), None, None, None, None, None


def flash_head_dim_supported(d: int) -> bool:
    """True for the head dims the flash kernels take: multiples of 8 from 8 to 128 (a head dim up to 64 runs on the
    64-wide tile, a larger one on the 128-wide tile, with the columns past ``d`` zero-filled)."""
    return d % 8 == 0 and 8 <= d <= 128


def attention_qkvpacked_supported(qkv, mask, dropout_p, training) -> bool:
    """True when :func:`attention_qkvpacked` runs the native flash kernels: a contiguous bf16 projection on the GPU
    whose head dim :func:`flash_head_dim_supported` accepts, and no dense ``mask``."""
    return (
        use_native(qkv)
        and qkv.dtype == torch.bfloat16
        and mask is None
        and flash_head_dim_supported(packed_head_dim(qkv))
        and qkv.is_contiguous()
    )


def attention_qkvpacked(qkv, *, causal: bool, scale: float, kv_lens=None, dropout_p: float = 0.0, training: bool = False,
                        alibi_slopes=None):
    """qkv ``[b, s, a, 3d]`` or grouped ``[b, s, g, r + 2, d]`` → context ``[b, s, a, d]``; ``kv_lens`` (int32 ``[b]``): valid keys per sample
    of a right-padded batch (keys beyond it are masked inside the kernel); ``dropout_p`` > 0 in training drops
    attention probabilities inside the kernel (Philox, TP-rank salted)."""
    p = float(dropout_p) if training else 0.0
    return _FlashAttnPackedFn.apply(qkv, causal, float(scale), kv_lens, p, alibi_slopes)


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
              dropout_p: float = 0.0, training: bool = False, alibi_slopes=None, kv_lens=None, kv_start=None):
    """Softmax attention of q ``[b, a, sq, d]`` over k, v ``[b, g, sk, d]`` (``g = a`` or, grouped-query, a divisor of
    ``a``; ``sq`` and ``sk`` independent).  Key ``j`` is visible to query ``i`` of sample ``b`` iff
    ``kv_start[b] <= j < kv_lens[b]`` (int32 ``[b]`` device tensors, defaults ``0`` and ``sk``; ``kv_lens`` is clamped to
    at least 1) and, when ``causal``, ``j <= i + sk - sq`` (bottom-right alignment).  A query without a visible key
    gets zeros.  The native flash kernels (see :func:`attention_supported`) handle this masking, an additive score bias
    (dense ``[b|1, a|1, sq, sk]`` — T5 relative positions — or ``alibi_slopes`` ``[a]``, ``slope·(j − i − (sk − sq))``)
    and dropout on the probabilities; arbitrary dense 0/1 masks use the reference math.  The reference applies
    ``kv_lens`` only together with ``kv_start``."""
    if scale is None:
        scale = 1.0 / math.sqrt(q.shape[-1])
    if attention_supported(q, k, mask, bias):
        # strided [b, a, s, d] views of the packed QKV projection are consumed directly (TMA strides)
        return _FlashAttnFn.apply(q, k, v, causal, float(scale), bias, alibi_slopes,
                                  float(dropout_p) if training else 0.0, kv_lens, kv_start)
    if kv_start is not None:
        vis = visible_keys(q.shape[-2], k.shape[-2], causal=causal, kv_start=kv_start, kv_lens=kv_lens, device=q.device)
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
    """The decode kernels take bf16 projections and caches with head dim 64 or 128; other dtypes and head dims run the
    reference math (as :func:`attention` does)."""
    return (
        use_native(x)
        and x.dtype == torch.bfloat16
        and k_cache.dtype == torch.bfloat16
        and k_cache.shape[-1] in (64, 128)
    )


def kv_cache_append(qkv, k_cache, v_cache, cache_seqlens, cos=None, sin=None, return_q: bool = True):
    """Write k, v of the packed projection ``qkv`` (``[b, s, a, 3d]``, or grouped ``[b, s, g, r + 2, d]``) into rows
    ``cache_seqlens[b] + i`` of the caches ``[b, g, C, d]``.  With
    ``cos/sin`` (fp32 ``[positions, d]``) q and k are first rotated at those positions, exactly as
    :func:`apply_rotary_qkv` with ``pos_offset = cache_seqlens[b]`` does.  Returns q ``[b, s, a, d]`` (rotated when the
    tables are given) when ``return_q``, else None."""
    if _decode_native(qkv, k_cache) and (cos is None or cos.dtype == torch.float32):
        ext = load_ext()
        q = ext.kv_append(qkv if qkv.is_contiguous() else qkv.contiguous(), k_cache, v_cache, cache_seqlens, cos, sin,
                          bool(return_q))
        count_launch()
        return q if return_q else None
    q = kv_cache_append_ref(qkv, k_cache, v_cache, cache_seqlens, cos, sin)
    return q if return_q else None


def kv_cache_append_ref(qkv, k_cache, v_cache, cache_seqlens, cos=None, sin=None):
    s_len = qkv.shape[1]
    q, k, v = split_qkv(qkv)
    starts = [int(x) for x in cache_seqlens.tolist()]
    if cos is not None:
        pos = torch.tensor(starts, device=cos.device)[:, None] + torch.arange(s_len, device=cos.device)[None]
        c = cos[pos][:, :, None, :].to(qkv.dtype)
        sn = sin[pos][:, :, None, :].to(qkv.dtype)
        q = q * c + rotate_half(q) * sn
        k = k * c + rotate_half(k) * sn
    for b, st in enumerate(starts):
        k_cache[b, :, st : st + s_len] = k[b].transpose(0, 1)
        v_cache[b, :, st : st + s_len] = v[b].transpose(0, 1)
    return q


def decode_attention(q, k_cache, v_cache, cache_seqlens, kv_start, *, scale: float, splits: int = 0,
                     past: Optional[int] = None):
    """Attention of ``q [b, s, a, d]`` (new tokens, already appended to the caches; any strides with d contiguous) over
    the caches ``[b, g, C, d]`` (query head ``h`` reads cache head ``h // (a // g)``): query ``i`` of sample ``b`` sees exactly the keys ``kv_start[b] <= j <= cache_seqlens[b] + i``.  Returns
    ``[b, s, a, d]`` contiguous; a query without a visible key gets zeros.  The native kernel takes up to 16 new tokens
    and reads lengths on the device (no host sync; one CUDA-graph capture replays after the lengths change); ``splits``
    > 0 fixes its number of key-range splits.  ``past`` (host int): the rows every sample held before these tokens
    (``cache_seqlens`` all equal to it, as in a :class:`~libai_b200.inference.kv_cache.StaticKVCache`); with it, more
    than 16 new tokens run the causal flash kernel over the cache window ``[:past + s]`` (chunked prefill)."""
    if _decode_native(q, k_cache):
        if q.shape[1] <= 16:
            ext = load_ext()
            o = ext.decode_attn(q, k_cache, v_cache, cache_seqlens, kv_start, float(scale), int(splits))
            count_launch(2)
            return o
        if past is not None:
            L = past + q.shape[1]
            o = attention(q.permute(0, 2, 1, 3), k_cache[:, :, :L], v_cache[:, :, :L], causal=True, scale=scale,
                          kv_start=kv_start)
            return o.transpose(1, 2)   # the kernel's [b, s, a, d] output
    return decode_attention_ref(q, k_cache, v_cache, cache_seqlens, kv_start, scale=scale)


def decode_attention_ref(q, k_cache, v_cache, cache_seqlens, kv_start, *, scale: float):
    """:func:`attention_ref` over the window ``[:L]`` of the caches (``L = max(cache_seqlens) + s``) with the mask built
    from ``kv_start`` and causality among the new tokens."""
    s_len = q.shape[1]
    lens = cache_seqlens.long()
    L = int(lens.max()) + s_len
    j = torch.arange(L, device=q.device)[None, None, :]
    i = torch.arange(s_len, device=q.device)[None, :, None]
    visible = (j >= kv_start.long()[:, None, None]) & (j <= lens[:, None, None] + i)          # [b, s, L]
    o = attention_ref(q.permute(0, 2, 1, 3), k_cache[:, :, :L], v_cache[:, :, :L], causal=False, scale=scale,
                      mask=visible[:, None])
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
        main_grad = getattr(table, "main_grad", None)
        if main_grad is not None and main_grad.dtype == torch.float32:
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


class _RopeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, cos, sin):
        ext = load_ext()
        ctx.save_for_backward(cos, sin)
        count_launch()
        return ext.rope(x.contiguous(), cos, sin, False)

    @staticmethod
    def backward(ctx, g):
        ext = load_ext()
        cos, sin = ctx.saved_tensors
        count_launch()
        return ext.rope(g.contiguous(), cos, sin, True), None, None


def apply_rotary(x, cos, sin):
    """x ``[b, a, s, d]``; cos/sin ``[s, d]`` (HF "rotate_half" convention; reference
    projects/Llama/llama.py:31-43)."""
    if use_native(x) and x.dtype == torch.bfloat16 and cos.dtype == torch.float32:
        return _RopeFn.apply(x, cos, sin)
    c = cos[None, None].to(x.dtype)
    s = sin[None, None].to(x.dtype)
    return x * c + rotate_half(x) * s



class _RopeQKVFn(torch.autograd.Function):
    """Rotary embedding on every q and k of the packed projection (``[b, s, a, 3d]`` or ``[b, s, g, r + 2, d]``) in one
    pass (v copied);
    the backward rotates the packed ``dqkv`` of the attention kernel in place with the inverse rotation."""

    @staticmethod
    def forward(ctx, qkv, cos, sin, pos_offset):
        ext = load_ext()
        ctx.save_for_backward(cos, sin)
        ctx.pos_offset = pos_offset
        count_launch()
        return ext.rope_qkv(qkv, cos, sin, pos_offset, False, False)

    @staticmethod
    def backward(ctx, g):
        ext = load_ext()
        cos, sin = ctx.saved_tensors
        count_launch()
        g = g if g.is_contiguous() else g.contiguous()
        return ext.rope_qkv(g, cos, sin, ctx.pos_offset, True, True), None, None, None


def apply_rotary_qkv(qkv, cos, sin, pos_offset: int = 0):
    """qkv ``[b, s, a, 3d]`` (per-head ``[q|k|v]``) or grouped ``[b, s, g, r + 2, d]`` (per group ``q_0 .. q_{r-1}, k,
    v``); cos/sin fp32 ``[max_pos, d]``; token ``i`` of the sequence uses position ``i + pos_offset``."""
    if use_native(qkv) and qkv.dtype == torch.bfloat16 and cos.dtype == torch.float32 and qkv.is_contiguous():
        return _RopeQKVFn.apply(qkv, cos, sin, int(pos_offset))
    s_len = qkv.shape[1]
    if qkv.dim() == 5:
        r = qkv.shape[3] - 2
        c = cos[pos_offset : pos_offset + s_len, None, None, :].to(qkv.dtype)
        sn = sin[pos_offset : pos_offset + s_len, None, None, :].to(qkv.dtype)
        qk = qkv[..., : r + 1, :]
        return torch.cat([qk * c + rotate_half(qk) * sn, qkv[..., r + 1 :, :]], dim=3)
    d = qkv.shape[-1] // 3
    c = cos[pos_offset : pos_offset + s_len, None, :].to(qkv.dtype)
    sn = sin[pos_offset : pos_offset + s_len, None, :].to(qkv.dtype)
    q, k, v = qkv[..., :d], qkv[..., d : 2 * d], qkv[..., 2 * d :]
    return torch.cat([q * c + rotate_half(q) * sn, k * c + rotate_half(k) * sn, v], dim=-1)


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
