"""ChatGLM2/3-6B: RMSNorm, half-dimension interleaved rotary, multi-query attention, SwiGLU, optional P-tuning prefix.

Spec: reference projects/ChatGLM/chatglm.py — ``PrefixEncoder`` (:42-71), ``RotaryEmbedding`` with a
``[seq, d/4, 2]`` cos/sin cache applied to the first half of every head in interleaved pairs (:74-115 and
``apply_rotary_pos_emb``), ``SelfAttention`` with ``multi_query_group_num`` KV heads in one fused
``[a·d | g·d | g·d]`` projection (:228-370), ``MLP`` with a fused ``[2·ffn]`` up-projection and
``silu(x₀)·x₁`` (:373-416), ``GLMBlock`` / ``GLMTransformer`` (:419-577), ``ChatGLMModel`` (:668-785),
``ChatGLMForConditionalGeneration`` with generation hooks and ``chat`` (:788-990).  Parameter names follow the
original checkpoint (``transformer.encoder.layers.N.self_attention.query_key_value`` …) so the HF loader is 1:1.

Parallelism: data / pipeline parallel (the fused multi-query projection is not split over heads here).
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional

import torch
from torch import nn

from libai_b200.inference.generator.generation_utils import Generator
from libai_b200.inference.kv_cache import KVCacheLayer, KVCacheOwner, StaticKVCache, padding_bounds
from libai_b200.layers import LayerNorm, Linear, RMSLayerNorm
from libai_b200.layers._param import create_parameter
from libai_b200.models.utils.weight_init import init_method_normal
from libai_b200.ops import functional as OF
from libai_b200.ops import use_native


class PrefixEncoder(nn.Module):
    """P-tuning v2: ``[pre_seq_len]`` virtual tokens → per-layer key/value prefixes."""

    def __init__(self, cfg):
        super().__init__()
        self.prefix_projection = cfg.prefix_projection
        kv_size = cfg.num_layers * cfg.kv_channels * cfg.multi_query_group_num * 2
        if self.prefix_projection:
            self.embedding = nn.Embedding(cfg.pre_seq_len, kv_size)
            self.trans = nn.Sequential(nn.Linear(kv_size, cfg.hidden_size), nn.Tanh(), nn.Linear(cfg.hidden_size, kv_size))
        else:
            self.embedding = nn.Embedding(cfg.pre_seq_len, kv_size)

    def forward(self, prefix):
        tokens = self.embedding(prefix)
        return self.trans(tokens) if self.prefix_projection else tokens


rope_cache = OF.glm_rope_table   # ``[seq, rotary_dim/2, 2]`` (cos, sin) table; ``rotary_dim`` = half of the head dim
apply_rotary_pos_emb = OF.apply_glm_rotary   # x ``[b, s, heads, d]`` rotated by the first ``s`` rows of a table


class AttentionInputs(NamedTuple):
    """What every layer's attention takes besides its hidden states, decided once per forward: the rotary table and
    positions of the new tokens, and how keys are masked — ``mask`` (a dense ``[b, 1, q, k]`` visibility for the
    reference math), ``kv_lens`` (right padding) or ``kv_start`` (left padding), none of them for plain causal.
    ``pos_base`` (int32 device tensor): the new tokens sit at ``pos_base[0] + pos_offset + i`` (a cached step reads its
    positions from the cache's lengths)."""

    table: torch.Tensor
    pos_offset: int = 0
    position_ids: Optional[torch.Tensor] = None
    mask: Optional[torch.Tensor] = None
    kv_lens: Optional[torch.Tensor] = None
    kv_start: Optional[torch.Tensor] = None
    pos_base: Optional[torch.Tensor] = None


class RotaryEmbedding(nn.Module):
    """``rope(max_seq_len)`` → the ``[seq, rotary_dim/2, 2]`` (cos, sin) cache consumed by :func:`apply_rotary_pos_emb`
    (reference projects/ChatGLM/chatglm.py RotaryEmbedding)."""

    def __init__(self, dim, original_impl=False, device=None, dtype=None, base: float = 10000.0):
        super().__init__()
        self.dim, self.original_impl, self.base = dim, original_impl, base

    def forward(self, max_seq_len, offset=0, device=None):
        return rope_cache(max_seq_len, self.dim, self.base, device=device)


class CoreAttention(nn.Module):
    """Scaled-dot-product core on ``[b, heads, s, d]`` tensors → ``[b, s, heads·d]``: the flash kernel when no explicit
    mask is given (causal, bottom-right aligned when there are more keys than queries; ``kv_start`` = left padding),
    the masked reference math otherwise."""

    def __init__(self, cfg=None, layer_number=1):
        super().__init__()
        self.layer_number = max(1, layer_number)
        self.attention_dropout = float(cfg.attention_dropout) if cfg is not None else 0.0

    def forward(self, query_layer, key_layer, value_layer, attention_mask=None, kv_start=None):
        b, a, s, d = query_layer.shape
        ctx = OF.attention(query_layer, key_layer, value_layer, causal=attention_mask is None, scale=1.0 / math.sqrt(d),
                           mask=attention_mask, dropout_p=self.attention_dropout, training=self.training,
                           kv_start=kv_start)
        return ctx.transpose(1, 2).reshape(b, s, a * d)


class SelfAttention(nn.Module):
    def __init__(self, cfg, layer_number):
        super().__init__()
        self.layer_number = max(1, layer_number)
        self.heads, self.d = cfg.num_attention_heads, cfg.kv_channels
        self.groups = cfg.multi_query_group_num if cfg.multi_query_attention else cfg.num_attention_heads
        proj = self.heads * self.d
        init = init_method_normal(0.02)
        self.query_key_value = Linear(cfg.hidden_size, proj + 2 * self.groups * self.d,
                                      bias=cfg.add_bias_linear or cfg.add_qkv_bias, parallel="data", init_method=init,
                                      layer_idx=layer_number - 1)
        self.dense = Linear(proj, cfg.hidden_size, bias=cfg.add_bias_linear, parallel="data", init_method=init,
                            layer_idx=layer_number - 1)
        self.attention_dropout = cfg.attention_dropout
        self.core_attention = CoreAttention(cfg, layer_number)
        # what a StaticKVCache sizes itself by (KVCacheOwner): the cache holds the g key/value heads
        self.head_size, self.local_heads, self.local_kv_heads = self.d, self.heads, self.groups

    def forward(self, hidden, inputs: AttentionInputs, kv_cache=None):
        """``kv_cache``: this layer's :class:`KVCacheLayer` (cached generation), or the P-tuning prefix ``(k, v)``
        (``[b, g, pre, d]`` each, never rotated), or None."""
        b, s, _ = hidden.shape
        a, g, d = self.heads, self.groups, self.d
        mixed = self.query_key_value(hidden)
        if isinstance(kv_cache, KVCacheLayer):   # GLM rotary into the grouped layout the cache appends from
            qkv = OF.apply_glm_rotary_qkv(mixed, heads=a, kv_heads=g, table=inputs.table, pos_offset=inputs.pos_offset,
                                          position_ids=inputs.position_ids, grouped=True, pos_base=inputs.pos_base)
            ctx = kv_cache.attend(kv_cache.append(qkv), scale=1.0 / math.sqrt(d), mask=inputs.mask)
            return self.dense(ctx.reshape(b, s, a * d))
        # per-head [b, s, a, 3d]: every query head with its own copy of its group's K/V (multi-query attention)
        qkv = OF.apply_glm_rotary_qkv(mixed, heads=a, kv_heads=g, table=inputs.table, pos_offset=inputs.pos_offset,
                                      position_ids=inputs.position_ids)
        if kv_cache is None and inputs.mask is None and inputs.kv_start is None and OF.attention_qkvpacked_supported(
                qkv, None, self.attention_dropout, self.training):
            ctx = OF.attention_qkvpacked(qkv, causal=True, scale=1.0 / math.sqrt(d), kv_lens=inputs.kv_lens,
                                         dropout_p=self.attention_dropout, training=self.training)
            return self.dense(ctx.reshape(b, s, a * d))
        q, k, v = (t.transpose(1, 2) for t in OF.split_qkv(qkv))   # [b, a, s, d] views
        if kv_cache is not None:   # P-tuning v2: the prefix keys / values go in front of the tokens'
            k = torch.cat((kv_cache[0].repeat_interleave(a // g, dim=1).type_as(k), k), dim=2)
            v = torch.cat((kv_cache[1].repeat_interleave(a // g, dim=1).type_as(v), v), dim=2)
        return self.dense(self.core_attention(q, k, v, inputs.mask, kv_start=inputs.kv_start))


class MLP(nn.Module):
    def __init__(self, cfg, layer_idx):
        super().__init__()
        init = init_method_normal(0.02)
        self.dense_h_to_4h = Linear(cfg.hidden_size, cfg.ffn_hidden_size * 2, bias=cfg.add_bias_linear, parallel="data",
                                    init_method=init, layer_idx=layer_idx)
        self.dense_4h_to_h = Linear(cfg.ffn_hidden_size, cfg.hidden_size, bias=cfg.add_bias_linear, parallel="data",
                                    init_method=init, layer_idx=layer_idx)

    def forward(self, hidden):
        gate, up = self.dense_h_to_4h(hidden).chunk(2, dim=-1)
        return self.dense_4h_to_h(OF.swiglu(gate.contiguous(), up.contiguous()))


class GLMBlock(nn.Module):
    def __init__(self, cfg, layer_number):
        super().__init__()
        self.layer_number, self.layer_idx = layer_number, layer_number - 1
        self.apply_residual_connection_post_layernorm = cfg.apply_residual_connection_post_layernorm
        norm = RMSLayerNorm if cfg.rmsnorm else LayerNorm
        self.input_layernorm = norm(cfg.hidden_size, eps=cfg.layernorm_epsilon, layer_idx=self.layer_idx)
        self.self_attention = SelfAttention(cfg, layer_number)
        self.hidden_dropout = cfg.hidden_dropout
        self.post_attention_layernorm = norm(cfg.hidden_size, eps=cfg.layernorm_epsilon, layer_idx=self.layer_idx)
        self.mlp = MLP(cfg, self.layer_idx)

    def forward(self, hidden, inputs: AttentionInputs, kv_cache=None):
        ln = self.input_layernorm(hidden)
        attn = self.self_attention(ln, inputs, kv_cache=kv_cache)
        residual = ln if self.apply_residual_connection_post_layernorm else hidden
        x = residual + torch.nn.functional.dropout(attn, p=self.hidden_dropout, training=self.training)
        ln2 = self.post_attention_layernorm(x)
        residual = ln2 if self.apply_residual_connection_post_layernorm else x
        return residual + torch.nn.functional.dropout(self.mlp(ln2), p=self.hidden_dropout, training=self.training)


class GLMTransformer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.num_layers, self.post_layer_norm = cfg.num_layers, cfg.post_layer_norm
        self.layers = nn.ModuleList([GLMBlock(cfg, i + 1) for i in range(cfg.num_layers)])
        if self.post_layer_norm:
            norm = RMSLayerNorm if cfg.rmsnorm else LayerNorm
            self.final_layernorm = norm(cfg.hidden_size, eps=cfg.layernorm_epsilon, layer_idx=-1)

    def forward(self, hidden, inputs: AttentionInputs, kv_caches=None):
        """``kv_caches``: one entry per layer (see :meth:`SelfAttention.forward`), or None."""
        kv_caches = kv_caches or [None] * self.num_layers
        for layer, cache in zip(self.layers, kv_caches):
            hidden = layer(hidden, inputs, kv_cache=cache)
        if self.post_layer_norm:
            hidden = self.final_layernorm(hidden)
        return hidden


class EmbeddingLayer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.word_embeddings = nn.Embedding(cfg.padded_vocab_size, cfg.hidden_size)

    def forward(self, input_ids):
        return self.word_embeddings(input_ids)


class ChatGLMPreTrainedModel:
    """Helpers shared by the ChatGLM model classes (reference projects/ChatGLM/chatglm.py ChatGLMPreTrainedModel:
    ``_init_weights`` / ``get_masks`` / ``get_position_ids``); a mixin — parameters are initialised by the layer
    constructors, so ``_init_weights`` has nothing left to do."""

    def _init_weights(self, module: nn.Module):
        return

    def get_position_ids(self, input_ids):
        b, s = input_ids.shape
        return torch.arange(s, dtype=torch.long, device=input_ids.device).unsqueeze(0).repeat(b, 1)


class ChatGLMModel(nn.Module, ChatGLMPreTrainedModel):
    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        self.embedding = EmbeddingLayer(cfg)
        self.num_layers, self.groups, self.kv_channels = cfg.num_layers, cfg.multi_query_group_num, cfg.kv_channels
        self.seq_length = cfg.seq_length
        self.rotary_dim = cfg.kv_channels // 2
        self.encoder = GLMTransformer(cfg)
        self.output_layer = Linear(cfg.hidden_size, cfg.padded_vocab_size, bias=False, parallel="data",
                                   init_method=init_method_normal(0.02), layer_idx=-1)
        self.pre_seq_len = cfg.pre_seq_len
        if self.pre_seq_len is not None:
            for p in self.parameters():
                p.requires_grad = False
            self.register_buffer("prefix_tokens", torch.arange(self.pre_seq_len).long(), persistent=False)
            self.prefix_encoder = PrefixEncoder(cfg)
            self.dropout = nn.Dropout(0.1)
        self._rope = None

    def get_input_embeddings(self):
        return self.embedding.word_embeddings

    def get_prompt(self, batch_size, device, dtype):
        tokens = self.prefix_tokens.unsqueeze(0).expand(batch_size, -1).to(device)
        kv = self.prefix_encoder(tokens).to(dtype)
        kv = kv.view(batch_size, self.pre_seq_len, self.num_layers * 2, self.groups, self.kv_channels)
        kv = self.dropout(kv).permute(2, 0, 3, 1, 4)  # [layers*2, b, groups, pre, d]
        return [(kv[2 * i], kv[2 * i + 1]) for i in range(self.num_layers)]

    def get_masks(self, input_ids, past_length, padding_mask=None):
        """Boolean visibility ``[b, 1, q, k]`` (None = plain causal without cache → kernel handles it)."""
        b, q = input_ids.shape
        if past_length == 0 and (padding_mask is None or bool(padding_mask.all())):
            return None
        k = past_length + q
        mask = torch.ones(k, k, dtype=torch.bool, device=input_ids.device).tril()[k - q :][None, None].expand(b, 1, q, k)
        if padding_mask is not None:
            mask = mask & padding_mask.bool()[:, None, None, :k]
        return mask

    def _flash_attention(self, hidden) -> bool:
        """True when the layers' attention runs the flash kernels (see :func:`OF.attention_supported`), which take
        right / left padding as ``kv_lens`` / ``kv_start`` instead of a dense mask."""
        return use_native(hidden) and hidden.dtype == torch.bfloat16 and OF.flash_head_dim_supported(self.kv_channels)

    def forward(self, input_ids, position_ids=None, attention_mask=None, past_key_values=None):
        """``past_key_values``: the :class:`StaticKVCache` of cached generation (appended to in place), or None.
        ``attention_mask`` ``[b, past + s]``: 1 = token, 0 = padding.  ``position_ids`` ``[b, s]``: the rotary positions
        of the tokens (the first row serves the batch); by default they continue from the cache."""
        b, q = input_ids.shape
        hidden = self.embedding(input_ids)
        if self._rope is None or self._rope.device != input_ids.device or self._rope.shape[0] < self.seq_length:
            self._rope = rope_cache(self.seq_length, self.rotary_dim, device=input_ids.device)
        pre = self.pre_seq_len or 0
        if isinstance(past_key_values, StaticKVCache):
            cache = past_key_values
            # the prompt's padding sits behind the P-tuning prefix rows, where kv_start cannot describe it
            dense = cache.step_needs_dense_mask(attention_mask, flash=cache.flash_attention(), kv_start_ok=not pre)
            if cache.length == 0 and pre:   # prefill: the prefix rows first
                for i, (k, v) in enumerate(self.get_prompt(b, input_ids.device, hidden.dtype)):
                    if i in cache.owned:
                        cache.write_rows(i, k, v)
                cache.advance(pre)
            past = cache.length
            # the default positions continue from the cache: seqlens (every sample's rows, the prefix's included)
            # minus the prefix, read on the device
            inputs = AttentionInputs(self._rope, -pre, position_ids,
                                     mask=self.get_masks(input_ids, past, attention_mask) if dense else None,
                                     pos_base=cache.seqlens if position_ids is None else None)
            hidden = self.encoder(hidden, inputs, kv_caches=[cache.layer(i) for i in range(self.num_layers)])
            cache.advance(q)
            return hidden
        padded = attention_mask is not None and not bool(attention_mask.all())
        inputs = AttentionInputs(self._rope, 0, position_ids)
        if not self._flash_attention(hidden) or (padded and pre):
            inputs = inputs._replace(mask=self.get_masks(input_ids, pre, attention_mask if padded else None))
        elif padded:
            bounds = padding_bounds(attention_mask)
            if bounds is None:   # neither a right- nor a left-padded batch
                inputs = inputs._replace(mask=self.get_masks(input_ids, 0, attention_mask))
            else:
                inputs = inputs._replace(kv_lens=bounds[0], kv_start=bounds[1])
        prefix = self.get_prompt(b, input_ids.device, hidden.dtype) if pre else None
        return self.encoder(hidden, inputs, kv_caches=prefix)


class ChatGLMForConditionalGeneration(nn.Module, ChatGLMPreTrainedModel, KVCacheOwner, Generator):
    speculative_decoding = True

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        self.transformer = ChatGLMModel(cfg)
        if cfg.get("lora_enable", False):
            from projects.ChatGLM.lora.lora_model import LoraModel

            self.transformer = LoraModel(self.transformer, cfg.lora_cfg, "default")

    @property
    def glm(self) -> ChatGLMModel:
        """The transformer, unwrapped from a :class:`LoraModel`."""
        return self.transformer if isinstance(self.transformer, ChatGLMModel) else self.transformer.model

    def forward(self, input_ids, position_ids=None, attention_mask=None, labels=None, use_cache=False):
        cache = None
        if use_cache:
            pre = self.glm.pre_seq_len or 0
            cache = self._prepare_cache(input_ids, max_positions=self.glm.seq_length + pre)
            if cache.length == 0:
                cache.reserve(pre + input_ids.shape[1])
        hidden = self.transformer(input_ids, position_ids, attention_mask, cache)
        if cache is not None:
            self.past_length = cache.length
        logits = self.glm.output_layer(hidden)
        if labels is not None:
            shift_logits = logits[:, :-1].float().reshape(-1, logits.shape[-1])
            shift_labels = labels[:, 1:].reshape(-1)
            loss = torch.nn.functional.cross_entropy(shift_logits, shift_labels, ignore_index=-100)
            return {"loss": loss}
        return {"logits": logits}

    # ---- KV cache (KVCacheOwner) ----------------------------------------------------------------
    def _cache_attention_modules(self):
        return [layer.self_attention for layer in self.glm.encoder.layers]

    @property
    def cache_rows_before_prompt(self) -> int:
        return self.glm.pre_seq_len or 0

    def allocate_kv_cache(self, batch: int, max_length: int) -> StaticKVCache:
        # the cache also holds the P-tuning prefix rows
        return super().allocate_kv_cache(batch, max_length + (self.glm.pre_seq_len or 0))

    def process_response(self, output, history):
        content = ""
        history = list(history)
        for response in output.split("<|assistant|>"):
            if "\n" in response:
                metadata, content = response.split("\n", maxsplit=1)
            else:
                metadata, content = "", response
            if not metadata.strip():
                content = content.strip().replace("[[训练时间]]", "2023年")
                history.append({"role": "assistant", "metadata": metadata, "content": content})
            else:
                history.append({"role": "assistant", "metadata": metadata, "content": content})
        return content, history

    @torch.no_grad()
    def chat(self, tokenizer, query, history=None, role="user", max_length=8192, num_beams=1, do_sample=True, top_p=0.8,
             temperature=0.8, **kwargs):
        history = history or []
        inputs = tokenizer.build_chat_input(query, history=history, role=role)
        ids = inputs["input_ids"].to(next(self.parameters()).device)
        out = self.generate(ids, max_length=max_length, num_beams=num_beams, do_sample=do_sample, top_p=top_p,
                            temperature=temperature, eos_token_id=tokenizer.eos_token_id, **kwargs)
        response = tokenizer.decode(out[0, ids.shape[1] : -1].tolist())
        history.append({"role": role, "content": query})
        return self.process_response(response, history)

    @staticmethod
    def set_activation_checkpoint(model):
        model.activation_checkpoint = True
        return model
