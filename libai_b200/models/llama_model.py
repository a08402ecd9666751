"""Llama (RMSNorm + rotary attention + SwiGLU) causal LM.

Spec: reference projects/Llama/llama.py — ``rotate_half/apply_rotary_pos_emb`` (:31-43), ``MLP`` with
``gate_proj/up_proj`` (col) and ``down_proj`` (row), no biases (:66-114), ``MultiheadAttention`` with a packed
per-head ``[q|k|v]`` ``query_key_value`` (col) + ``o_proj`` (row) and a KV cache (:117-227), ``CasualMask``
(:230-271), ``LlamaDecoderLayer`` (:274-386), ``LlamaModel`` with cached cos/sin tables (:389-494),
``SFTLoss`` = CE ignoring label 0 / negative labels (:497-520), ``LlamaForCausalLM`` (:523-649).  Parameter names
follow the reference so its HF loader mapping (projects/Llama/utils/llama_loader.py) carries over.

H100 path: rotary runs as one pass over the packed QKV projection (``rope_qkv`` kernel, v copied) feeding the
flash-attention kernel; SwiGLU and RMSNorm are native kernels; the LM head is vocab-parallel with the fused
vocab-parallel cross entropy (the reference replicates ``lm_head``).
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import torch
from torch import nn

from libai_b200.config import configurable
from libai_b200.layers import Linear, RMSLayerNorm, VocabEmbedding
from libai_b200.layers._param import xavier_normal_
from libai_b200.layers.attention import AttnMaskType
from libai_b200.layers.embedding import get_sp_shape, set_sp_shape
from libai_b200.ops import functional as OF
from libai_b200.parallel import mappings
from libai_b200.utils import distributed as dutil

from libai_b200.inference.generator.generation_utils import Generator
from libai_b200.inference.kv_cache import KVCacheLayer, KVCacheOwner, StaticKVCache, left_padding

from .utils.pipeline_model import PipelineStageMixin
from .utils.weight_init import init_method_normal, scaled_init_method_normal


def rotary_tables(rotary_dim: int, seq_len: int, base: float = 10000.0, device=None):
    """fp32 ``cos/sin`` ``[seq_len, rotary_dim]`` in the "rotate_half" (two halves) convention."""
    inv_freq = 1.0 / (base ** (torch.arange(0, rotary_dim, 2, dtype=torch.float32, device=device) / rotary_dim))
    freqs = torch.outer(torch.arange(seq_len, dtype=torch.float32, device=device), inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    return emb.cos().contiguous(), emb.sin().contiguous()


class RotaryEmbedding(nn.Module):
    """``cos, sin = rope(x, seq_len)`` — fp32 tables ``[seq_len, dim]`` on ``x``'s device, cached up to the longest
    length requested (reference projects/Llama/llama.py:46-63 returns slices of tables the model owns; the attention
    layers here call :func:`rotary_tables` through the same cache)."""

    def __init__(self, dim, max_position_embeddings=2048, base: float = 10000.0):
        super().__init__()
        self.dim, self.max_position_embeddings, self.base = dim, max_position_embeddings, base
        self._cache = None

    def forward(self, x, seq_len=None, cos_cached=None, sin_cached=None):
        seq_len = x.shape[-2] if seq_len is None else seq_len
        if seq_len > self.max_position_embeddings:
            raise ValueError(f"The maximum supported length is {self.max_position_embeddings}, "
                             f"and the current length is {seq_len}.")
        if cos_cached is not None and sin_cached is not None:
            return cos_cached[:seq_len].to(x.device), sin_cached[:seq_len].to(x.device)
        if self._cache is None or self._cache[0].shape[0] < seq_len or self._cache[0].device != x.device:
            self._cache = rotary_tables(self.dim, max(seq_len, 1), self.base, device=x.device)
        return self._cache[0][:seq_len], self._cache[1][:seq_len]


class LlamaMLP(nn.Module):
    def __init__(self, hidden_size, intermediate_size, init_method=xavier_normal_, output_layer_init_method=None, *,
                 layer_idx=0):
        super().__init__()
        output_layer_init_method = output_layer_init_method or init_method
        self.gate_proj = Linear(hidden_size, intermediate_size, bias=False, parallel="col", init_method=init_method,
                                layer_idx=layer_idx)
        self.up_proj = Linear(hidden_size, intermediate_size, bias=False, parallel="col", init_method=init_method,
                              layer_idx=layer_idx)
        self.down_proj = Linear(intermediate_size, hidden_size, bias=False, parallel="row",
                                init_method=output_layer_init_method, layer_idx=layer_idx)

    def forward(self, hidden_states):
        y = self._forward_fused_gate_up(hidden_states)
        if y is not None:
            return y
        return self.down_proj(OF.swiglu(self.gate_proj(hidden_states), self.up_proj(hidden_states)))

    def _forward_fused_gate_up(self, x):
        """Gate and up projection as ONE GEMM against the ``[2F, K]`` view over both weights (they are adjacent once the
        optimizer owns the parameters) — ``ops/gated_mlp.py``; ``None`` = not applicable, take the two-GEMM path."""
        from libai_b200.ops import gated_mlp, use_native

        if not (gated_mlp.enabled() and x.is_cuda and x.dtype == torch.bfloat16 and use_native(x)):
            return None
        wg, wu, wd = self.gate_proj.weight, self.up_proj.weight, self.down_proj.weight
        if self.gate_proj.bias is not None or self.up_proj.bias is not None or self.down_proj.bias is not None:
            return None
        if wg.dtype != torch.bfloat16 or gated_mlp.fused_gate_up_views(wg, wu) is None:
            return None
        topo = dutil.get_dist_util()
        t = topo.tensor_parallel_size
        if t == 1:
            return gated_mlp.gated_mlp(x, wg, wu, wd)
        if not (topo.fused_tp_comm and topo.sequence_parallel and x.dim() == 2):
            return None
        from libai_b200.ops import comm_gemm

        M, K = x.shape[0] * t, x.shape[1]
        if not (comm_gemm.fused_supported(M, 2 * wg.shape[0], K, t) and comm_gemm.fused_supported(M, wd.shape[0], wg.shape[0], t)):
            return None
        return gated_mlp.tp_gated_mlp(x.contiguous(), wg, wu, wd, None, topo.tp_group)


class LlamaAttention(nn.Module):
    def __init__(self, hidden_size, num_attention_heads, max_position_embeddings, init_method=xavier_normal_,
                 output_layer_init_method=None, scale_mask_softmax_fusion=False, attn_mask_type=AttnMaskType.causal,
                 qkv_bias=False, *, layer_idx=0):
        super().__init__()
        output_layer_init_method = output_layer_init_method or init_method
        topo = dutil.get_dist_util()
        self.hidden_size, self.num_heads = hidden_size, num_attention_heads
        self.head_size = hidden_size // num_attention_heads
        assert num_attention_heads % topo.tensor_parallel_size == 0
        self.local_heads = num_attention_heads // topo.tensor_parallel_size
        self.norm_factor = 1.0 / math.sqrt(float(self.head_size))
        self.attn_mask_type = attn_mask_type
        self.query_key_value = Linear(hidden_size, hidden_size * 3, bias=qkv_bias, parallel="col",
                                      init_method=init_method, layer_idx=layer_idx)
        self.o_proj = Linear(hidden_size, hidden_size, bias=False, parallel="row",
                             init_method=output_layer_init_method, layer_idx=layer_idx)

    def forward(self, hidden_states, attention_mask=None, past_key_value=None, cos_cached=None, sin_cached=None,
                use_cache=False):
        sp = dutil.get_dist_util().sequence_parallel and hidden_states.dim() == 2
        a, d = self.local_heads, self.head_size
        bsz, tgt_len = get_sp_shape() if sp else hidden_states.shape[:2]
        qkv = self.query_key_value(hidden_states).view(bsz, -1, a, 3 * d)
        if isinstance(past_key_value, KVCacheLayer):
            context = self._cached_attention(qkv, attention_mask, past_key_value, cos_cached, sin_cached)
            context = context.reshape(-1, a * d) if sp else context.reshape(bsz, -1, a * d)
            output = self.o_proj(context)
            return (output, past_key_value) if use_cache else output
        past_len = 0 if past_key_value is None else past_key_value[0].shape[2]
        qkv = OF.apply_rotary_qkv(qkv, cos_cached, sin_cached, past_len)
        if (
            past_key_value is None and not use_cache and attention_mask is None
            and OF.attention_qkvpacked_supported(qkv, None, 0.0, self.training)
        ):
            context = OF.attention_qkvpacked(qkv, causal=True, scale=self.norm_factor).reshape(bsz, -1, a * d)
        else:
            q4 = qkv.permute(0, 2, 1, 3)
            query, key, value = q4[..., :d], q4[..., d : 2 * d], q4[..., 2 * d :]
            if past_key_value is not None:
                key = torch.cat((past_key_value[0].type_as(key), key), dim=2)
                value = torch.cat((past_key_value[1].type_as(value), value), dim=2)
            if use_cache:
                past_key_value = (key, value)
            causal = attention_mask is None and key.shape[2] == query.shape[2]
            mask = attention_mask
            if mask is None and not causal:  # decoding with a cache: every cached key is visible
                mask = None
            context = OF.attention(query, key, value, causal=causal, scale=self.norm_factor, mask=mask)
            context = context.transpose(1, 2).reshape(bsz, -1, a * d)
        if sp:
            context = context.reshape(-1, a * d)
        output = self.o_proj(context)
        return (output, past_key_value) if use_cache else output

    def _cached_attention(self, qkv, attention_mask, cache, cos, sin):
        """Rotary + append into the layer's cache, then attention over it → ``[b, s, a, d]``.  Steps after the prefill
        (padding carried by ``cache.kv_start``) go to :func:`OF.decode_attention`: the split-KV kernel for bf16 with head
        dim 64 / 128 and up to 16 new tokens, the reference math otherwise.  The prefill runs the usual dispatch (flash
        kernel for a causal prompt) on views of the cache, and a dense ``attention_mask`` keeps the reference math."""
        past, s_len = cache.length, qkv.shape[1]
        q = OF.kv_cache_append(qkv, cache.k, cache.v, cache.seqlens, cos, sin)
        if past > 0 and attention_mask is None:
            return OF.decode_attention(q, cache.k, cache.v, cache.seqlens, cache.kv_start, scale=self.norm_factor)
        L = past + s_len
        key, value = cache.k[:, :, :L], cache.v[:, :, :L]
        causal = attention_mask is None   # prefill of an unpadded prompt
        context = OF.attention(q.permute(0, 2, 1, 3), key, value, causal=causal, scale=self.norm_factor,
                               mask=attention_mask)
        return context.transpose(1, 2)


class CasualMask(nn.Module):
    """Boolean ``[b, 1, tgt, src]`` visibility mask (True = attend) from the causal structure and an optional
    ``[b, src]`` padding mask (reference :230-271 builds the additive float version)."""

    def __init__(self, max_positions=1024, *, layer_idx=0):
        super().__init__()
        self.max_positions = max_positions

    def forward(self, input_ids, past_length=0, attention_mask=None, input_dtype=None):
        bsz, tgt_len = input_ids.shape
        src_len = past_length + tgt_len
        mask = torch.ones(src_len, src_len, dtype=torch.bool, device=input_ids.device).tril()
        mask = mask[src_len - tgt_len :, :][None, None].expand(bsz, 1, tgt_len, src_len)
        if attention_mask is not None:
            pad = attention_mask[:, None, None, :src_len] > 0 if attention_mask.dim() == 2 else attention_mask > 0
            mask = mask & pad
        return mask


class LlamaDecoderLayer(nn.Module):
    def __init__(self, hidden_size, intermediate_size, num_attention_heads, is_decoder=False, rms_norm_eps=1e-5,
                 max_position_embeddings=None, init_method=xavier_normal_, output_layer_init_method=None,
                 scale_mask_softmax_fusion=False, attn_mask_type=AttnMaskType.causal, qkv_bias=False, *, layer_idx=0):
        super().__init__()
        self.layer_idx, self.is_decoder = layer_idx, is_decoder
        self.input_layernorm = RMSLayerNorm(hidden_size, eps=rms_norm_eps, layer_idx=layer_idx)
        self.self_attn = LlamaAttention(hidden_size, num_attention_heads, max_position_embeddings,
                                        init_method=init_method, output_layer_init_method=output_layer_init_method,
                                        scale_mask_softmax_fusion=scale_mask_softmax_fusion,
                                        attn_mask_type=attn_mask_type, qkv_bias=qkv_bias, layer_idx=layer_idx)
        self.post_attention_layernorm = RMSLayerNorm(hidden_size, eps=rms_norm_eps, layer_idx=layer_idx)
        self.mlp = LlamaMLP(hidden_size, intermediate_size, init_method, output_layer_init_method, layer_idx=layer_idx)

    def forward(self, hidden_states, attention_mask=None, past_key_value=None, cos_cached=None, sin_cached=None,
                use_cache=False):
        attn = self.self_attn(self.input_layernorm(hidden_states), attention_mask=attention_mask,
                              past_key_value=past_key_value, cos_cached=cos_cached, sin_cached=sin_cached,
                              use_cache=use_cache)
        presents = None
        if use_cache:
            attn, presents = attn
        hidden_states = hidden_states + attn
        output = hidden_states + self.mlp(self.post_attention_layernorm(hidden_states))
        return (output, presents) if use_cache else output


class LlamaModel(nn.Module):
    def __init__(self, hidden_layers, vocab_size, hidden_size, intermediate_size, num_attention_heads,
                 max_position_embeddings=1024, rms_norm_eps=1e-5, initializer_range=0.02,
                 use_scaled_init_for_output_weights=True, scale_mask_softmax_fusion=False, amp_enabled=False,
                 qkv_bias=False, rope_base=10000.0):
        super().__init__()
        init_method = init_method_normal(sigma=initializer_range)
        output_layer_init_method = (
            scaled_init_method_normal(initializer_range, hidden_layers) if use_scaled_init_for_output_weights
            else init_method
        )
        self.embed_tokens = VocabEmbedding(vocab_size, hidden_size, init_method=init_method, amp_enabled=amp_enabled)
        self.layers = nn.ModuleList(
            [
                LlamaDecoderLayer(hidden_size, intermediate_size, num_attention_heads, rms_norm_eps=rms_norm_eps,
                                  max_position_embeddings=max_position_embeddings, init_method=init_method,
                                  output_layer_init_method=output_layer_init_method,
                                  scale_mask_softmax_fusion=scale_mask_softmax_fusion,
                                  attn_mask_type=AttnMaskType.causal, qkv_bias=qkv_bias, layer_idx=i)
                for i in range(hidden_layers)
            ]
        )
        self.norm = RMSLayerNorm(hidden_size, eps=rms_norm_eps, layer_idx=-1)
        self.rope_base = rope_base
        self._set_cos_sin_cache(hidden_size // num_attention_heads, max_position_embeddings, base=rope_base)

    def _set_cos_sin_cache(self, rotary_dim, seq_len, base=10000, dtype=None, layer_idx=0):
        cos, sin = rotary_tables(rotary_dim, seq_len, base)
        self.register_buffer("cos_cached", cos, persistent=False)
        self.register_buffer("sin_cached", sin, persistent=False)

    def embed(self, input_ids):
        bsz, seq = input_ids.shape
        topo = dutil.get_dist_util()
        if topo.sequence_parallel:
            set_sp_shape(bsz, seq)
            return self.embed_tokens(input_ids, scatter_to_sequence_parallel=True)
        return self.embed_tokens(input_ids)

    def forward(self, input_ids, attention_mask=None, past_key_values=None, use_cache=False, set_cache=None):
        if isinstance(past_key_values, StaticKVCache):
            # the layers append in place; the lengths advance once every layer has seen this step's tokens
            cache = past_key_values
            if self.cos_cached.device != input_ids.device:   # tables built on the CPU for a model built on the GPU
                self.cos_cached, self.sin_cached = self.cos_cached.to(input_ids.device), self.sin_cached.to(input_ids.device)
            hidden_states = self.embed(input_ids)
            for i, layer in enumerate(self.layers):
                hidden_states = layer(hidden_states, attention_mask=attention_mask, past_key_value=cache.layer(i),
                                      cos_cached=self.cos_cached, sin_cached=self.sin_cached, use_cache=False)
            cache.advance(input_ids.shape[1])
            return self.norm(hidden_states)
        presents = [] if use_cache else None
        hidden_states = self.embed(input_ids)
        past_key_values = past_key_values or [None] * len(self.layers)
        for layer, past in zip(self.layers, past_key_values):
            hidden_states = layer(hidden_states, attention_mask=attention_mask, past_key_value=past,
                                  cos_cached=self.cos_cached, sin_cached=self.sin_cached, use_cache=use_cache)
            if use_cache:
                hidden_states, present = hidden_states
                presents.append(present)
        hidden_states = self.norm(hidden_states)
        if use_cache and set_cache is not None:
            set_cache(presents)
        return hidden_states


class CrossEntropyLoss(nn.Module):
    """Per-token vocab-parallel CE; negative labels are mapped to 0 (= ignored by ``SFTLoss``)."""

    def forward(self, logits, target):
        target = target * (target >= 0)
        if logits.dim() == 2:
            logits = logits.view(target.shape[0], target.shape[1], -1)
        topo = dutil.get_dist_util()
        v_local = logits.shape[-1]
        return OF.vocab_parallel_cross_entropy(
            logits, target, vocab_start=topo.tp_rank * v_local if topo.tensor_parallel_size > 1 else 0,
            group=topo.tp_group if topo.tensor_parallel_size > 1 else None,
        ), target


class SFTLoss(nn.Module):
    def __init__(self) -> None:
        super().__init__()
        self.lm_loss = CrossEntropyLoss()

    def forward(self, logits, lm_labels):
        loss, target = self.lm_loss(logits, lm_labels)
        keep = (target != 0).to(loss.dtype)  # ignore_index = 0 (reference :505-507)
        return {"lm_loss": (loss * keep).sum() / keep.sum().clamp(min=1.0)}


class LlamaForCausalLM(nn.Module, PipelineStageMixin, Generator, KVCacheOwner):

    # `train.dist.sequence_parallel = "auto"` resolves to True for this model (token-sharded activations between
    # the tensor-parallel blocks are handled by its embeddings / heads)
    supports_sequence_parallel = True
    @configurable
    def __init__(self, hidden_layers, vocab_size, hidden_size, intermediate_size, num_attention_heads,
                 max_position_embeddings=1024, rms_norm_eps=1e-5, initializer_range=0.02,
                 use_scaled_init_for_output_weights=True, scale_mask_softmax_fusion=False, amp_enabled=False,
                 qkv_bias=False, rope_base=10000.0, cfg=None):
        super().__init__()
        self.cfg = cfg
        self.hidden_layers = hidden_layers
        self.model = LlamaModel(
            hidden_layers=hidden_layers, vocab_size=vocab_size, hidden_size=hidden_size,
            intermediate_size=intermediate_size, num_attention_heads=num_attention_heads,
            max_position_embeddings=max_position_embeddings, rms_norm_eps=rms_norm_eps,
            initializer_range=initializer_range,
            use_scaled_init_for_output_weights=use_scaled_init_for_output_weights,
            scale_mask_softmax_fusion=scale_mask_softmax_fusion, amp_enabled=amp_enabled, qkv_bias=qkv_bias,
            rope_base=rope_base,
        )
        self.casual_mask = CasualMask(max_position_embeddings, layer_idx=0)
        self.lm_head = Linear(hidden_size, vocab_size, bias=False, parallel="col",
                              init_method=init_method_normal(initializer_range), layer_idx=-1)
        self.loss_func = SFTLoss()
        self.kv_cache: Optional[StaticKVCache] = None
        self.past_length = 0

    @classmethod
    def from_config(cls, cfg):
        keys = ("hidden_layers vocab_size hidden_size intermediate_size num_attention_heads max_position_embeddings "
                "rms_norm_eps initializer_range use_scaled_init_for_output_weights scale_mask_softmax_fusion "
                "amp_enabled").split()
        out = {k: cfg[k] for k in keys}
        for k in ("qkv_bias", "rope_base"):
            if k in cfg:
                out[k] = cfg[k]
        out["cfg"] = cfg
        return out

    # ---- pipeline protocol ----------------------------------------------------------------------
    def stage_pre(self, input_ids, **_):
        return self.model.embed(input_ids)

    def stage_layers(self):
        return self.model.layers

    def stage_layer_call(self, layer, hidden, batch):
        return layer(hidden, cos_cached=self.model.cos_cached, sin_cached=self.model.sin_cached)

    def stage_post(self, hidden, labels=None, **_):
        logits = self.lm_head(self.model.norm(hidden))
        if labels is not None:
            return self.loss_func(logits, labels)
        return {"logits": self._full_logits(logits)}

    def _full_logits(self, logits):
        topo = dutil.get_dist_util()
        if logits.dim() == 2 and topo.sequence_parallel:
            b, s = get_sp_shape()
            logits = logits.view(b, s, -1)
        return mappings.gather_from_tp(logits) if topo.tensor_parallel_size > 1 else logits

    def forward(self, input_ids, attention_mask=None, labels=None, use_cache=False):
        if not use_cache and attention_mask is None:
            return self.forward_stage({"input_ids": input_ids, "labels": labels})
        # generation / padded batches: explicit masks and the KV cache (single pipeline stage)
        if not use_cache:
            mask = None if attention_mask is None else self.casual_mask(input_ids, attention_mask=attention_mask)
            output = self.model(input_ids, attention_mask=mask)
        else:
            cache = self._prepare_cache(input_ids, max_positions=self.model.cos_cached.shape[0])
            self.past_length = past = cache.length
            mask = None
            if attention_mask is not None:
                if past == 0:
                    kv_start = left_padding(attention_mask) if attention_mask.dim() == 2 else None
                    cache.dense_mask = kv_start is None
                    if kv_start is not None:
                        cache.kv_start.copy_(kv_start)
                if past == 0 or cache.dense_mask:
                    # the prefill of a padded prompt (and every step of a mask kv_start cannot express) is dense
                    mask = self.casual_mask(input_ids, past_length=past, attention_mask=attention_mask)
            output = self.model(input_ids, attention_mask=mask, past_key_values=cache)
            self.past_length = cache.length
        logits = self.lm_head(output)
        if labels is not None:
            return self.loss_func(logits, labels)
        return {"logits": self._full_logits(logits)}

    # ---- KV cache (KVCacheOwner) ----------------------------------------------------------------
    def _cache_attention_modules(self):
        return [layer.self_attn for layer in self.model.layers]

    def prepare_inputs_for_generation(self, input_ids, past=None, attention_mask=None, use_cache=None, **kwargs):
        """With a warm cache only the newest token is fed; the padding mask always covers cache + new tokens."""
        if past is not None and use_cache:
            input_ids = input_ids[:, -1:]
        out = {"input_ids": input_ids, "use_cache": bool(use_cache)}
        if attention_mask is not None and not bool(attention_mask.all()):
            out["attention_mask"] = attention_mask
        return out

    @staticmethod
    def set_pipeline_stage_id(model):
        return model

    @staticmethod
    def set_activation_checkpoint(model):
        model.activation_checkpoint = True
        return model
