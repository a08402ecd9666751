"""Multi-head attention (self / cross) with tensor-parallel heads.

Spec: reference libai/layers/attention.py:31-281 — fused QKV column-parallel projection whose
output features are laid out per head as ``[a, 3, d]`` (``view(b, s, a, 3d)`` then chunk,
:195-200; loaders depend on this layout), KV cache for incremental decoding (:201-208), scores
scaled by ``1/√d`` — optionally additionally divided by ``layer_idx+1`` with the softmax
multiplying it back (``apply_query_key_layer_scaling``, :87-91, numerically the identity in
exact arithmetic) — masked positions filled with −10000 (:223-245), row-parallel output
projection, bias+dropout fused with the residual add.

The softmax(QKᵀ)V core runs in the sm_90a flash-attention kernel (no ``[b,a,s,s]`` tensor, no
materialised masks) whenever the mask is purely causal or absent; padding-mask / bias / dropout
variants fall back to the reference math in :func:`libai_b200.ops.functional.attention_ref`.
"""
from __future__ import annotations

import enum
import math
from typing import Tuple

import torch
from torch import nn

from libai_b200.inference.kv_cache import KVCacheLayer
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dutil

from ._param import xavier_normal_
from .embedding import get_sp_shape
from .linear import Linear


class AttnMaskType(enum.Enum):
    padding = 1
    causal = 2


class KeyPaddingMask:
    """Padding mask of a right-padded batch.

    Carries the per-sample number of valid keys (``lengths``, int32 ``[b]``) for the flash-attention
    kernel and builds the reference's dense ``[b, 1, s, s]`` mask (``m_i * m_j``, reference
    libai/models/bert_model.py:36-48) on demand for the reference math."""

    def __init__(self, mask_2d: torch.Tensor):
        self.mask_2d = mask_2d
        self.lengths = mask_2d.to(torch.int32).sum(dim=-1).to(torch.int32).contiguous()
        self._dense = None
        self._prefix = None

    @classmethod
    def from_lengths(cls, lengths: torch.Tensor) -> "KeyPaddingMask":
        """Right-padded mask given directly by its key lengths (int32 ``[b]``) — no host synchronisation, usable while a
        CUDA graph is being captured (engine/cuda_graphs.py)."""
        self = cls.__new__(cls)
        self.mask_2d = None
        self.lengths = lengths
        self._dense = None
        self._prefix = True
        return self

    def is_prefix(self) -> bool:
        """True when every row is a right-padded contiguous prefix (``1…10…0``) — the only shape ``lengths`` can
        express.  Left padding / holes must take the dense ``m_i·m_j`` path.  Checked once per mask (one small sync)."""
        if self._prefix is None:
            m = self.mask_2d.to(torch.int8)
            self._prefix = bool((m[:, 1:] <= m[:, :-1]).all()) if m.shape[1] > 1 else True
        return self._prefix

    def dense(self) -> torch.Tensor:
        if self._dense is None:
            m = self.mask_2d.to(torch.int8)
            self._dense = (m.unsqueeze(1) * m.unsqueeze(2)).unsqueeze(1)
        return self._dense


class MultiheadAttention(nn.Module):
    def __init__(
        self,
        hidden_size,
        num_attention_heads,
        is_cross_attention=False,
        attention_dropout_prob=0.0,
        output_dropout_prob=0.0,
        init_method=xavier_normal_,
        output_layer_init_method=None,
        bias_dropout_fusion=False,
        scale_mask_softmax_fusion=False,
        apply_query_key_layer_scaling=False,
        attn_mask_type=AttnMaskType.padding,
        *,
        layer_idx=0,
    ):
        super().__init__()
        self.hidden_size = hidden_size
        if output_layer_init_method is None:
            output_layer_init_method = init_method
        assert hidden_size % num_attention_heads == 0, "hidden_size must be divisible by num_attention_heads."
        tp = dutil.get_tensor_parallel_size()
        assert num_attention_heads % tp == 0, "num_attention_heads must be divisible by tensor_parallel_size."
        self.num_heads = num_attention_heads
        self.local_heads = num_attention_heads // tp
        self.head_size = hidden_size // num_attention_heads
        self.attn_mask_type = attn_mask_type
        self.attention_dropout_prob = attention_dropout_prob
        self.output_dropout_prob = output_dropout_prob
        self.bias_dropout_fusion = bias_dropout_fusion
        self.scale_mask_softmax_fusion = scale_mask_softmax_fusion
        self.is_cross_attention = is_cross_attention
        # 1/sqrt(d); with query-key layer scaling the pre-softmax scores are additionally divided
        # by (layer_idx + 1) and the softmax multiplies it back → the product is norm_factor.
        self.coeff = None
        self.norm_factor = 1.0 / math.sqrt(float(self.head_size))
        if apply_query_key_layer_scaling:
            self.coeff = layer_idx + 1
            self.norm_factor /= self.coeff
        self.softmax_scale = self.norm_factor * (self.coeff or 1.0)

        if is_cross_attention:
            self.query = Linear(hidden_size, hidden_size, parallel="col", init_method=init_method, layer_idx=layer_idx)
            self.key_value = Linear(hidden_size, hidden_size * 2, parallel="col", init_method=init_method, layer_idx=layer_idx)
        else:
            self.query_key_value = Linear(hidden_size, hidden_size * 3, parallel="col", init_method=init_method, layer_idx=layer_idx)
        self.dense = Linear(
            hidden_size, hidden_size, parallel="row", init_method=output_layer_init_method,
            skip_bias_add=True, layer_idx=layer_idx,
        )

    def forward(
        self,
        hidden_states: torch.Tensor,
        encoder_states: torch.Tensor = None,
        attention_mask: torch.Tensor = None,
        past_key_value: Tuple[torch.Tensor, torch.Tensor] = None,
        use_cache: bool = False,
        residual: torch.Tensor = None,
    ):
        """hidden_states ``[b, s, h]`` (or ``[b·s/t, h]`` token shards under sequence parallelism).

        Returns the output-projection result with bias and dropout applied (plus ``residual`` when
        given); ``(output, (key, value))`` when ``use_cache``."""
        sp = dutil.get_dist_util().sequence_parallel
        a, d = self.local_heads, self.head_size
        if sp and hidden_states.dim() == 2:
            bsz, tgt_len = get_sp_shape()
        else:
            bsz, tgt_len = hidden_states.shape[:2]

        if self.is_cross_attention:
            query = self.query(hidden_states).view(bsz, -1, a, d).permute(0, 2, 1, 3)
            if past_key_value is not None:
                key, value = past_key_value
            elif encoder_states is not None:
                kv = self.key_value(encoder_states).view(bsz, -1, a, 2 * d).permute(0, 2, 1, 3)
                key, value = kv[..., :d], kv[..., d:]
            else:
                raise ValueError("past_key_value and encoder_states cannot be None at the same time.")
        else:
            qkv_packed = self.query_key_value(hidden_states).view(bsz, -1, a, 3 * d)
            kv_lens = None
            if isinstance(attention_mask, KeyPaddingMask) and attention_mask.is_prefix():
                kv_lens = attention_mask.lengths
            if (
                past_key_value is None and not use_cache
                and (attention_mask is None or kv_lens is not None)
                and OF.attention_qkvpacked_supported(qkv_packed, None, self.attention_dropout_prob, self.training)
            ):
                # fast path: flash attention directly on the packed projection
                context = OF.attention_qkvpacked(
                    qkv_packed, causal=self.attn_mask_type == AttnMaskType.causal, scale=self.softmax_scale,
                    kv_lens=kv_lens, dropout_p=self.attention_dropout_prob, training=self.training,
                ).reshape(bsz, -1, a * d)
                if sp and hidden_states.dim() == 2:
                    context = context.reshape(-1, a * d)
                topo = dutil.get_dist_util()
                if (residual is not None and topo.tensor_parallel_size == 1 and context.dtype == torch.bfloat16
                        and not getattr(self.dense, "quantized", False) and (self.output_dropout_prob == 0.0 or not self.training)):
                    # bias + residual in the epilogue of the output projection
                    return OF.linear_bias_residual(context, self.dense.weight, self.dense.bias, residual)
                if residual is not None and (self.output_dropout_prob == 0.0 or not self.training):
                    fused = self.dense.fused_bias_residual(context, residual)   # GEMM→RS + bias + residual, one kernel
                    if fused is not None:
                        return fused
                output, bias = self.dense(context)
                return OF.bias_dropout_add(output, bias, residual, self.output_dropout_prob, self.training)
            if isinstance(past_key_value, KVCacheLayer):
                if self.attn_mask_type != AttnMaskType.causal:
                    raise ValueError("a KVCacheLayer decodes causal self-attention only")
                if isinstance(attention_mask, KeyPaddingMask):
                    attention_mask = attention_mask.dense()
                q = past_key_value.append(qkv_packed)
                context = past_key_value.attend(q, scale=self.softmax_scale, mask=attention_mask,
                                                dropout_p=self.attention_dropout_prob, training=self.training)
                context = context.reshape(bsz, -1, a * d)
                if sp and hidden_states.dim() == 2:
                    context = context.reshape(-1, a * d)
                output, bias = self.dense(context)
                output = OF.bias_dropout_add(output, bias, residual, self.output_dropout_prob, self.training)
                return (output, past_key_value) if use_cache else output
            qkv = qkv_packed.permute(0, 2, 1, 3)
            query, key, value = qkv[..., :d], qkv[..., d : 2 * d], qkv[..., 2 * d :]
            if past_key_value is not None:
                past_key, past_value = past_key_value
                key = torch.cat((past_key.type_as(key), key), dim=2)
                value = torch.cat((past_value.type_as(value), value), dim=2)
        if use_cache:
            past_key_value = (key, value)

        key_lens = None
        if isinstance(attention_mask, KeyPaddingMask):
            if self.is_cross_attention and attention_mask.is_prefix() and OF.attention_supported(query, key):
                key_lens, attention_mask = attention_mask.lengths, None   # right-padded encoder keys, in the kernel
            else:
                attention_mask = attention_mask.dense()
        causal = (
            self.attn_mask_type == AttnMaskType.causal
            and attention_mask is None
            and not self.is_cross_attention
        )
        context = OF.attention(
            query, key, value,
            causal=causal,
            scale=self.softmax_scale,
            mask=attention_mask,
            dropout_p=self.attention_dropout_prob,
            training=self.training,
            kv_lens=key_lens,
        )  # [b, a, s, d]
        context = context.transpose(1, 2).reshape(bsz, -1, a * d)
        if sp and hidden_states.dim() == 2:
            context = context.reshape(-1, a * d)
        output, bias = self.dense(context)
        output = OF.bias_dropout_add(output, bias, residual, self.output_dropout_prob, self.training)
        if use_cache:
            return output, past_key_value
        return output

    def extra_repr(self) -> str:
        return "hidden_size={}, num_heads={}, is_cross_attention={}".format(
            self.hidden_size, self.num_heads, self.is_cross_attention
        )
