"""T5 v1.0 / v1.1 / mT5 encoder-decoder with relative position bias (HuggingFace-compatible numerics).

Spec: reference projects/MT5/mt5_model.py (``MT5Model`` :31-323 with generation cache + ``prepare_inputs_for_generation``,
``MT5ForPreTraining`` :326-470) and projects/MT5/layers/* — RMS layer norms, un-scaled attention scores with a
bucketed relative position bias owned by the first layer of each stack and shared by the others
(attention_layer.py:268-345), ReLU MLP for ``model_type="t5"`` / gated-GELU (``wi_0``, ``wi_1``) for ``"mt5"``
(mlp_layer.py), shared or separate LM head (``tie_word_embeddings`` rescales by ``hidden_size**-0.5``).
Parameter names follow the reference project so its loader mapping applies.

Cached generation (one pipeline stage) decodes from two preallocated :class:`StaticKVCache` objects: the decoder
self-attention's, appended to at every step, and the cross-attention's, which holds every decoder layer's projection of
the encoder states from the first step on.  The decoder's relative-position bias only depends on the distance
``p − j >= 0`` between query and key and is constant from ``MAX_DISTANCE`` on, so the decode kernel takes it as one
``[heads, MAX_DISTANCE + 1]`` vector per forward.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
from torch import nn

from libai_b200.config import configurable
from libai_b200.inference.generator.generation_utils import Generator
from libai_b200.inference.kv_cache import KVCacheLayer, KVCacheOwner, StaticKVCache, padding_window
from libai_b200.layers import Linear, LMLogits, ParallelCrossEntropyLoss, RMSLayerNorm, VocabEmbedding
from libai_b200.layers._param import create_parameter
from libai_b200.models.utils.weight_init import init_method_normal, scaled_init_method_normal
from libai_b200.ops import functional as OF
from libai_b200.parallel import mappings
from libai_b200.utils import distributed as dutil


class MT5Embedding(nn.Module):
    def __init__(self, hidden_size, vocab_size, embedding_dropout_prob, init_method, amp_enabled=False):
        super().__init__()
        self.word_embeddings = VocabEmbedding(vocab_size, hidden_size, init_method=init_method, amp_enabled=amp_enabled)
        self.embedding_dropout = nn.Dropout(embedding_dropout_prob)

    def forward(self, input_ids):
        return self.embedding_dropout(self.word_embeddings(input_ids))


MAX_DISTANCE = 128   # T5's bucketing saturates at this distance


def relative_position_bucket(relative_position, bidirectional=True, num_buckets=32, max_distance=MAX_DISTANCE):
    """T5 bucketing: half of the buckets are exact offsets, the other half log-spaced up to ``max_distance``."""
    buckets = torch.zeros_like(relative_position)
    if bidirectional:
        num_buckets //= 2
        buckets = buckets + (relative_position > 0).long() * num_buckets
        relative_position = relative_position.abs()
    else:
        relative_position = -torch.min(relative_position, torch.zeros_like(relative_position))
    max_exact = num_buckets // 2
    is_small = relative_position < max_exact
    large = max_exact + (
        torch.log(relative_position.float().clamp(min=1) / max_exact) / math.log(max_distance / max_exact)
        * (num_buckets - max_exact)
    ).long()
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    return buckets + torch.where(is_small, relative_position, large)


class T5Attention(nn.Module):
    def __init__(self, hidden_size, num_attention_heads, head_size, relative_attention_num_buckets, is_cross_attention,
                 is_decoder, attention_dropout_prob, output_dropout_prob, init_method, output_layer_init_method,
                 has_relative_attention_bias, layer_idx):
        super().__init__()
        topo = dutil.get_dist_util()
        self.num_heads, self.head_size = num_attention_heads, head_size
        self.local_heads = num_attention_heads // topo.tensor_parallel_size
        self.is_cross_attention, self.is_decoder = is_cross_attention, is_decoder
        self.num_buckets = relative_attention_num_buckets
        self.has_relative_attention_bias = has_relative_attention_bias
        inner = num_attention_heads * head_size
        if is_cross_attention:
            self.query = Linear(hidden_size, inner, bias=False, parallel="col", init_method=init_method, layer_idx=layer_idx)
            self.key_value = Linear(hidden_size, inner * 2, bias=False, parallel="col", init_method=init_method, layer_idx=layer_idx)
        else:
            self.query_key_value = Linear(hidden_size, inner * 3, bias=False, parallel="col", init_method=init_method,
                                          layer_idx=layer_idx)
        self.dense = Linear(inner, hidden_size, bias=False, parallel="row", init_method=output_layer_init_method,
                            layer_idx=layer_idx)
        self.attn_dropout_p, self.dropout = attention_dropout_prob, nn.Dropout(output_dropout_prob)
        if has_relative_attention_bias:
            # [buckets, heads], split over heads under tensor parallelism
            self.relative_attention_bias = create_parameter(
                (self.num_buckets, num_attention_heads), init_method, tp_dim=1, layer_idx=layer_idx)

    def compute_bias(self, q_len, k_len, device):
        ctx = torch.arange(k_len - q_len, k_len, device=device)[:, None]  # queries are the last q_len positions
        mem = torch.arange(k_len, device=device)[None, :]
        bucket = relative_position_bucket(mem - ctx, bidirectional=not self.is_decoder, num_buckets=self.num_buckets)
        return self.relative_attention_bias[bucket].permute(2, 0, 1).unsqueeze(0)  # [1, a, q, k]

    def relative_bias_vector(self):
        """fp32 ``[a, MAX_DISTANCE + 1]``: the decoder's bias at distance ``p − j = 0 .. MAX_DISTANCE`` (this rank's
        heads); unidirectional buckets saturate at ``num_buckets − 1`` from ``MAX_DISTANCE`` on, so the last column holds
        for every longer distance (the decode kernel clamps the distance to it)."""
        dist = torch.arange(MAX_DISTANCE + 1, device=self.relative_attention_bias.device)
        bucket = relative_position_bucket(-dist, bidirectional=False, num_buckets=self.num_buckets)
        return self.relative_attention_bias[bucket].t().float().contiguous()

    def forward(self, hidden, mask=None, encoder_states=None, past_key_value=None, position_bias=None, use_cache=False,
                cache: Optional[KVCacheLayer] = None):
        if cache is not None:
            # Attention of the new tokens over the layer's cache.  Self-attention appends k, v first and, without a
            # mask, takes the relative-bias vector (built by the first layer, then handed down as position_bias).
            # Cross-attention reads the cache of the encoder projection, without a mask through its window.  A mask
            # (decoder padding, an encoder mask with holes) keeps the dense bias with the mask folded in.
            b, s = hidden.shape[:2]
            a, d = self.local_heads, self.head_size
            causal = not self.is_cross_attention
            if causal:
                q = cache.append(self.query_key_value(hidden).view(b, s, a, 3 * d))
            else:
                q = self.query(hidden).view(b, s, a, d)
            if mask is None:
                if causal and position_bias is None:
                    position_bias = self.relative_bias_vector()
                ctx = cache.attend(q, scale=1.0, causal=causal, rel_bias=position_bias)
            else:
                if position_bias is None:
                    L = mask.shape[-1]
                    position_bias = self.compute_bias(s, L, hidden.device) if causal else \
                        torch.zeros(1, a, s, L, device=hidden.device, dtype=hidden.dtype)
                    position_bias = position_bias + (1.0 - mask.to(position_bias.dtype)) * -10000.0
                ctx = cache.attend(q, scale=1.0, causal=causal, bias=position_bias)
            return self.dropout(self.dense(ctx.reshape(b, s, a * d))), position_bias, None
        b = hidden.shape[0]
        a, d = self.local_heads, self.head_size
        if self.is_cross_attention:
            q = self.query(hidden).view(b, -1, a, d).permute(0, 2, 1, 3)
            if past_key_value is not None:
                k, v = past_key_value
            else:
                kv = self.key_value(encoder_states).view(b, -1, a, 2 * d).permute(0, 2, 1, 3)
                k, v = kv[..., :d], kv[..., d:]
        else:
            qkv = self.query_key_value(hidden).view(b, -1, a, 3 * d).permute(0, 2, 1, 3)
            q, k, v = qkv[..., :d], qkv[..., d : 2 * d], qkv[..., 2 * d :]
            if past_key_value is not None:
                k = torch.cat((past_key_value[0].type_as(k), k), dim=2)
                v = torch.cat((past_key_value[1].type_as(v), v), dim=2)
        present = (k, v) if use_cache else None
        if position_bias is None:
            if self.has_relative_attention_bias:
                position_bias = self.compute_bias(q.shape[2], k.shape[2], hidden.device)
            else:
                position_bias = torch.zeros(1, a, q.shape[2], k.shape[2], device=hidden.device, dtype=hidden.dtype)
            if mask is not None:
                # fold the 0/1 mask into the additive bias ONCE (the stack hands `position_bias` from layer to layer):
                # every layer then runs the flash kernel with a dense bias instead of the O(s²) masked-softmax math
                position_bias = position_bias + (1.0 - mask.to(position_bias.dtype)) * -10000.0
            position_bias._libai_mask_folded = mask is not None
        if getattr(position_bias, "_libai_mask_folded", False):
            mask = None
        ctx = OF.attention(q, k, v, causal=False, scale=1.0, mask=mask, bias=position_bias, dropout_p=self.attn_dropout_p,
                           training=self.training)
        out = self.dropout(self.dense(ctx.transpose(1, 2).reshape(b, -1, a * d)))
        return out, position_bias, present


class T5MLP(nn.Module):
    """T5 v1.0: ``wo(relu(wi(x)))``."""

    def __init__(self, hidden_size, ffn_hidden_size, output_dropout_prob, init_method, output_layer_init_method, layer_idx):
        super().__init__()
        self.dense_h_to_4h = Linear(hidden_size, ffn_hidden_size, bias=False, parallel="col", init_method=init_method, layer_idx=layer_idx)
        self.dense_4h_to_h = Linear(ffn_hidden_size, hidden_size, bias=False, parallel="row", init_method=output_layer_init_method, layer_idx=layer_idx)
        self.dropout = nn.Dropout(output_dropout_prob)

    def forward(self, x):
        return self.dropout(self.dense_4h_to_h(self.dense_h_to_4h(x, act="relu")))


class MT5MLP(nn.Module):
    """T5 v1.1 / mT5: ``wo(gelu_new(wi_0(x)) * wi_1(x))``."""

    def __init__(self, hidden_size, ffn_hidden_size, output_dropout_prob, init_method, output_layer_init_method, layer_idx):
        super().__init__()
        self.wi_0 = Linear(hidden_size, ffn_hidden_size, bias=False, parallel="col", init_method=init_method, layer_idx=layer_idx)
        self.wi_1 = Linear(hidden_size, ffn_hidden_size, bias=False, parallel="col", init_method=init_method, layer_idx=layer_idx)
        self.wo = Linear(ffn_hidden_size, hidden_size, bias=False, parallel="row", init_method=output_layer_init_method, layer_idx=layer_idx)
        self.dropout = nn.Dropout(output_dropout_prob)

    def forward(self, x):
        return self.dropout(self.wo(self.wi_0(x, act="gelu_tanh") * self.wi_1(x)))


class TransformerLayer(nn.Module):
    def __init__(self, hidden_size, ffn_hidden_size, num_attention_heads, head_size, relative_attention_num_buckets,
                 is_decoder=False, attention_dropout_prob=0.0, output_dropout_prob=0.0, layernorm_epsilon=1e-6,
                 init_method=None, output_layer_init_method=None, padding_idx=None, *, layer_idx=0, model_type="mt5",
                 has_relative_attention_bias=False):
        super().__init__()
        self.is_decoder, self.layer_idx = is_decoder, layer_idx
        common = dict(hidden_size=hidden_size, num_attention_heads=num_attention_heads, head_size=head_size,
                      relative_attention_num_buckets=relative_attention_num_buckets, is_decoder=is_decoder,
                      attention_dropout_prob=attention_dropout_prob, output_dropout_prob=output_dropout_prob,
                      init_method=init_method, output_layer_init_method=output_layer_init_method, layer_idx=layer_idx)
        self.input_layernorm = RMSLayerNorm(hidden_size, eps=layernorm_epsilon, layer_idx=layer_idx)
        self.self_attention = T5Attention(is_cross_attention=False, has_relative_attention_bias=has_relative_attention_bias, **common)
        self.post_attention_layernorm = RMSLayerNorm(hidden_size, eps=layernorm_epsilon, layer_idx=layer_idx)
        if is_decoder:
            self.cross_attention = T5Attention(is_cross_attention=True, has_relative_attention_bias=False, **common)
            self.post_cross_attention_layernorm = RMSLayerNorm(hidden_size, eps=layernorm_epsilon, layer_idx=layer_idx)
        mlp_cls = MT5MLP if model_type == "mt5" else T5MLP
        self.mlp = mlp_cls(hidden_size, ffn_hidden_size, output_dropout_prob, init_method, output_layer_init_method, layer_idx)

    def forward(self, hidden, attention_mask=None, encoder_states=None, encoder_attention_mask=None, past_key_value=None,
                position_bias=None, encoder_decoder_position_bias=None, use_cache=False,
                cache: Optional[KVCacheLayer] = None, cross_cache: Optional[KVCacheLayer] = None):
        """``cache`` / ``cross_cache``: the layer's self- and cross-attention caches of cached generation (then
        ``past_key_value`` and ``use_cache`` are unused and no ``present`` is returned)."""
        self_past = past_key_value[:2] if past_key_value is not None else None
        cross_past = past_key_value[2:] if past_key_value is not None and len(past_key_value) == 4 else None
        out, position_bias, present = self.self_attention(self.input_layernorm(hidden), attention_mask,
                                                          past_key_value=self_past, position_bias=position_bias,
                                                          use_cache=use_cache, cache=cache)
        hidden = hidden + out
        if self.is_decoder:
            out, encoder_decoder_position_bias, cross_present = self.cross_attention(
                self.post_attention_layernorm(hidden), encoder_attention_mask, encoder_states=encoder_states,
                past_key_value=cross_past, position_bias=encoder_decoder_position_bias, use_cache=use_cache,
                cache=cross_cache)
            hidden = hidden + out
            hidden = hidden + self.mlp(self.post_cross_attention_layernorm(hidden))
            if use_cache:
                present = present + cross_present
            return hidden, position_bias, encoder_decoder_position_bias, present
        hidden = hidden + self.mlp(self.post_attention_layernorm(hidden))
        return hidden, position_bias


def _extend(mask, causal_len=None):
    """[b, k] padding mask or [b, q, k] mask → boolean [b, 1, q, k]."""
    if mask is None:
        return None
    mask = mask.bool()
    if mask.dim() == 2:
        mask = mask[:, None, None, :]
    elif mask.dim() == 3:
        mask = mask[:, None]
    return mask


class MT5Model(nn.Module, Generator, KVCacheOwner):
    @configurable
    def __init__(self, vocab_size, hidden_size, hidden_layers, num_attention_heads, head_size, intermediate_size,
                 embedding_dropout_prob, hidden_dropout_prob, attention_probs_dropout_prob, relative_attention_num_buckets,
                 padding_idx=None, initializer_range=0.02, layernorm_eps=1e-12, amp_enabled=False, model_type="mt5",
                 cfg=None):
        super().__init__()
        self.cfg, self.model_type, self.hidden_size = cfg, model_type, hidden_size
        init_method = init_method_normal(initializer_range)
        scaled = scaled_init_method_normal(initializer_range, hidden_layers)
        self.embedding = MT5Embedding(hidden_size, vocab_size, embedding_dropout_prob, init_method, amp_enabled)

        def stack(is_decoder, offset):
            layers = nn.ModuleList([
                TransformerLayer(hidden_size, intermediate_size, num_attention_heads, head_size,
                                 relative_attention_num_buckets, is_decoder=is_decoder,
                                 attention_dropout_prob=attention_probs_dropout_prob,
                                 output_dropout_prob=hidden_dropout_prob, layernorm_epsilon=layernorm_eps,
                                 init_method=init_method, output_layer_init_method=scaled, padding_idx=padding_idx,
                                 layer_idx=offset + i, model_type=model_type, has_relative_attention_bias=(i == 0))
                for i in range(hidden_layers)])
            mod = nn.Module()
            mod.layers = layers
            mod.final_layernorm = RMSLayerNorm(hidden_size, eps=layernorm_eps, layer_idx=offset + hidden_layers - 1)
            return mod

        self.encoder = stack(False, 0)
        self.decoder = stack(True, hidden_layers)
        self.past_key_values = [None] * hidden_layers   # the tuple cache of pipeline-parallel inference
        self.encoder_states = None
        self.cross_cache: Optional[StaticKVCache] = None   # the encoder projection of every decoder layer
        self.tie_word_embeddings = bool(cfg.get("tie_word_embeddings", model_type != "mt5")) if cfg is not None else model_type != "mt5"
        if model_type == "mt5":
            self.lm_head = Linear(hidden_size, vocab_size, bias=False, parallel="col", init_method=init_method,
                                  layer_idx=2 * hidden_layers - 1)
        else:
            self.lm_head = LMLogits(vocab_size, bias=False)

    @classmethod
    def from_config(cls, cfg):
        keys = ("vocab_size hidden_size hidden_layers num_attention_heads head_size intermediate_size "
                "embedding_dropout_prob hidden_dropout_prob attention_probs_dropout_prob relative_attention_num_buckets "
                "padding_idx initializer_range layernorm_eps amp_enabled model_type").split()
        out = {k: cfg[k] for k in keys if k in cfg}
        out["cfg"] = cfg
        return out

    def encode(self, encoder_input_ids, encoder_attn_mask=None):
        hidden, bias = self.embedding(encoder_input_ids), None
        mask = _extend(encoder_attn_mask)
        for layer in self.encoder.layers:
            hidden, bias = layer(hidden, mask, position_bias=bias)
        return self.encoder.final_layernorm(hidden)

    # ---- inference under pipeline parallelism -----------------------------------------------------------------
    # (reference tests/inference/test_text_generation.py:41-90: generation with PP4 / TP2xPP2.)  The layers of the two
    # stacks live on different stages; the running state (hidden, relative-position biases) is handed over by a
    # broadcast inside the pipeline group at every stage boundary, every layer keeps its KV cache on its own stage and
    # the last stage's logits go back to everyone so that all ranks take the same decoding decisions.
    def _pp_walk(self, layers, state, step, first_stage=0):
        """``state``: list of tensors / None; ``step(layer, state) -> state`` runs on the owning stage only."""
        from libai_b200.parallel.pipeline import broadcast_from_stage

        topo = dutil.get_dist_util()
        cur = first_stage
        for layer in layers:
            st = topo.get_layer_stage_id(layer.layer_idx)
            if st != cur:
                state = list(broadcast_from_stage(state, cur, topo))
                cur = st
            if topo.pp_rank == st:
                state = step(layer, state)
        return state, cur

    def _forward_pipelined(self, encoder_input_ids, decoder_input_ids, encoder_attn_mask, decoder_attn_mask,
                           encoder_decoder_attn_mask, use_cache, only_encoder):
        from libai_b200.parallel.pipeline import broadcast_from_stage

        topo = dutil.get_dist_util()
        last = topo.pipeline_parallel_size - 1
        if use_cache and self.encoder_states is not None:
            encoder_states = self.encoder_states
        else:
            self.set_cache(None, None)
            self.past_length = 0
            mask = _extend(encoder_attn_mask)
            hidden = self.embedding(encoder_input_ids) if topo.is_first_stage else None

            def enc_step(layer, st):
                h, b = layer(st[0], mask, position_bias=st[1])
                return [h, b]

            state, cur = self._pp_walk(self.encoder.layers, [hidden, None], enc_step)
            ln_stage = topo.get_layer_stage_id(self.encoder.final_layernorm.layer_idx)
            if ln_stage != cur:
                state = list(broadcast_from_stage(state, cur, topo))
            enc = self.encoder.final_layernorm(state[0]) if topo.pp_rank == ln_stage else None
            encoder_states = broadcast_from_stage(enc, ln_stage, topo)      # every decoder stage cross-attends to it
        if only_encoder:
            return encoder_states
        past_len = self.past_length if use_cache else 0
        q_len = decoder_input_ids.shape[1]
        causal = torch.ones(past_len + q_len, past_len + q_len, dtype=torch.bool, device=decoder_input_ids.device).tril()
        dec_mask = causal[past_len:][None, None]
        if decoder_attn_mask is not None:
            extra = _extend(decoder_attn_mask)
            if extra.shape[-1] == past_len + q_len:
                dec_mask = dec_mask & extra[..., -q_len:, :] if extra.shape[-2] > 1 else dec_mask & extra
        cross_mask = _extend(encoder_decoder_attn_mask if encoder_decoder_attn_mask is not None else encoder_attn_mask)
        if cross_mask is not None and cross_mask.shape[-2] > 1:
            cross_mask = cross_mask[..., -q_len:, :]
        hidden = self.embedding(decoder_input_ids) if topo.is_first_stage else None
        presents = {}
        index = {id(layer): i for i, layer in enumerate(self.decoder.layers)}

        def dec_step(layer, st):
            i = index[id(layer)]
            h, b, cb, present = layer(st[0], dec_mask, encoder_states, cross_mask, past_key_value=self.past_key_values[i],
                                      position_bias=st[1], encoder_decoder_position_bias=st[2], use_cache=use_cache)
            presents[i] = present
            return [h, b, cb]

        state, cur = self._pp_walk(self.decoder.layers, [hidden, None, None], dec_step)
        if cur != last:
            state = list(broadcast_from_stage(state, cur, topo))
        if use_cache:
            self.encoder_states = encoder_states
            self.past_key_values = [presents.get(i) for i in range(len(self.decoder.layers))]   # own layers only
            self.past_length = past_len + q_len
        logits = None
        if self.model_type != "mt5" and getattr(self, "_pp_tied_weight", None) is None:
            # tied LM head: the word embedding lives on the first stage; the last stage needs a copy (weights are frozen
            # during inference, so it is fetched once)
            w = self.embedding.word_embeddings.weight.detach() if topo.is_first_stage else None
            self._pp_tied_weight = broadcast_from_stage(w, 0, topo)
        if topo.is_last_stage:
            hidden = self.decoder.final_layernorm(state[0])
            if self.tie_word_embeddings:
                hidden = hidden * (self.hidden_size ** -0.5)
            logits = self.lm_head(hidden) if self.model_type == "mt5" else self.lm_head(hidden, self._pp_tied_weight)
            if topo.tensor_parallel_size > 1:
                logits = mappings.gather_from_tp(logits)
        return {"logits": broadcast_from_stage(logits, last, topo)}

    def forward(self, encoder_input_ids=None, decoder_input_ids=None, encoder_attn_mask=None, decoder_attn_mask=None,
                encoder_decoder_attn_mask=None, use_cache=False, only_encoder=False):
        if dutil.get_dist_util().pipeline_parallel_size > 1 and not torch.is_grad_enabled():
            return self._forward_pipelined(encoder_input_ids, decoder_input_ids, encoder_attn_mask, decoder_attn_mask,
                                           encoder_decoder_attn_mask, use_cache, only_encoder)
        if use_cache and only_encoder and self.encoder_states is not None:
            return self.encoder_states
        if use_cache and not only_encoder:
            return self._forward_cached(encoder_input_ids, decoder_input_ids, encoder_attn_mask, decoder_attn_mask,
                                        encoder_decoder_attn_mask)
        self.set_cache(None, None)
        encoder_states = self.encode(encoder_input_ids, encoder_attn_mask)
        if only_encoder:
            return encoder_states
        past_len = 0
        q_len = decoder_input_ids.shape[1]
        causal = torch.ones(past_len + q_len, past_len + q_len, dtype=torch.bool, device=decoder_input_ids.device).tril()
        dec_mask = causal[past_len:][None, None]
        if decoder_attn_mask is not None:
            extra = _extend(decoder_attn_mask)
            if extra.shape[-1] == past_len + q_len:
                dec_mask = dec_mask & extra[..., -q_len:, :] if extra.shape[-2] > 1 else dec_mask & extra
        cross_mask = _extend(encoder_decoder_attn_mask if encoder_decoder_attn_mask is not None else encoder_attn_mask)
        if cross_mask is not None and cross_mask.shape[-2] > 1:
            cross_mask = cross_mask[..., -q_len:, :]
        hidden = self.embedding(decoder_input_ids)
        bias, cross_bias = None, None
        for layer in self.decoder.layers:
            hidden, bias, cross_bias = layer(hidden, dec_mask, encoder_states, cross_mask, position_bias=bias,
                                             encoder_decoder_position_bias=cross_bias)[:3]
        return {"logits": self._logits(hidden)}

    def _logits(self, hidden):
        hidden = self.decoder.final_layernorm(hidden)
        if self.tie_word_embeddings:
            hidden = hidden * (self.hidden_size ** -0.5)
        if self.model_type == "mt5":
            logits = self.lm_head(hidden)
        else:
            logits = self.lm_head(hidden, self.embedding.word_embeddings.weight)
        if not self.training and dutil.get_dist_util().tensor_parallel_size > 1:
            logits = mappings.gather_from_tp(logits)
        return logits

    # ---- cached generation on the StaticKVCache (one pipeline stage) -------------------------------
    def _forward_cached(self, encoder_input_ids, decoder_input_ids, encoder_attn_mask, decoder_attn_mask,
                        encoder_decoder_attn_mask):
        """The decoder over the preallocated caches.  The first step (an empty cache) runs the encoder and writes each
        decoder layer's projection of its states into ``cross_cache``, once.  Without a decoder mask that has padding,
        self-attention runs the decode kernels with the relative-bias vector; a 2-D encoder mask whose rows are one
        run of ones (left or right padding) becomes the cross cache's key window, any other one stays a dense mask."""
        cache = self._prepare_cache(decoder_input_ids)
        past, q_len = cache.length, decoder_input_ids.shape[1]
        cross_mask = encoder_decoder_attn_mask if encoder_decoder_attn_mask is not None else encoder_attn_mask
        if past == 0:
            # the mask's window first: its host sync then waits for no encoder work, and the decoder's launches keep
            # overlapping the encoder on the device
            window = padding_window(cross_mask) if cross_mask is not None and cross_mask.dim() == 2 else None
            self.encoder_states = self.encode(encoder_input_ids, encoder_attn_mask)
            self._fill_cross_cache(self.encoder_states, cross_mask is not None and window is None, window)
        self_mask = None
        extra = _extend(decoder_attn_mask)
        if extra is not None and extra.shape[-1] == past + q_len and not bool(extra.all()):
            causal = torch.ones(past + q_len, past + q_len, dtype=torch.bool, device=decoder_input_ids.device).tril()
            self_mask = causal[past:][None, None] & (extra[..., -q_len:, :] if extra.shape[-2] > 1 else extra)
        if self.cross_cache.dense_mask:
            cross_mask = _extend(cross_mask)
            if cross_mask.shape[-2] > 1:
                cross_mask = cross_mask[..., -q_len:, :]
        else:
            cross_mask = None
        hidden, bias, cross_bias = self.embedding(decoder_input_ids), None, None
        for i, layer in enumerate(self.decoder.layers):
            hidden, bias, cross_bias, _ = layer(hidden, self_mask, encoder_attention_mask=cross_mask,
                                                position_bias=bias, encoder_decoder_position_bias=cross_bias,
                                                cache=cache.layer(i), cross_cache=self.cross_cache.layer(i))
        cache.advance(q_len)
        self.past_length = cache.length
        return {"logits": self._logits(hidden)}

    def _fill_cross_cache(self, encoder_states, dense_mask: bool, window):
        b, S = encoder_states.shape[:2]
        attn = self.decoder.layers[0].cross_attention
        a, d = attn.local_heads, attn.head_size
        c = self.cross_cache
        kv_dtype = self.kv_cache_dtype   # the same format as the self-attention cache
        if (c is None or not c.matches(b, encoder_states.dtype, encoder_states.device, kv_dtype)
                or c.capacity < S):
            c = StaticKVCache(len(self.decoder.layers), b, a, d, S, encoder_states.dtype, encoder_states.device,
                              kv_dtype=kv_dtype)
            self._decode_graph = None   # a decode graph of the old cross cache (and its memory pool) goes with it
        kv = (layer.cross_attention.key_value(encoder_states).view(b, S, a, 2 * d).transpose(1, 2).split(d, dim=-1)
              for layer in self.decoder.layers)
        c.fill(kv, S, window)
        c.dense_mask = dense_mask
        self.cross_cache = c

    # ---- generation support ---------------------------------------------------------------------
    def _cache_attention_modules(self):
        return [layer.self_attention for layer in self.decoder.layers]

    def allocate_kv_cache(self, batch: int, max_length: int):
        """The decoder self-attention cache (one pipeline stage; pipeline-parallel inference keeps its tuple cache)."""
        if dutil.get_dist_util().pipeline_parallel_size > 1:
            return None
        return super().allocate_kv_cache(batch, max_length)

    @property
    def past_key_values(self):
        return self.kv_cache if self.kv_cache is not None else self._tuple_cache

    @past_key_values.setter
    def past_key_values(self, value):
        self._tuple_cache = value

    def set_cache(self, encoder_states, past_key_values):
        self.encoder_states = encoder_states
        if isinstance(past_key_values, StaticKVCache):
            self.kv_cache, self.past_length = past_key_values, past_key_values.length
            return
        if past_key_values is None and self.kv_cache is not None:
            self.kv_cache.reset()
        self.past_length = 0 if past_key_values is None else past_key_values[0][0].shape[2]
        self._tuple_cache = [None] * len(self.decoder.layers) if past_key_values is None else list(past_key_values)

    def _reorder_cache(self, past, beam_idx):
        if past is None:
            return None
        if isinstance(past, StaticKVCache):
            # Only the self-attention cache is gathered.  The cross cache and the encoder states stay as they are:
            # _expand_inputs_for_generation gives every beam of a sample the same encoder inputs, and for a sample
            # still decoding BeamSearchScorer.process picks beam_idx among that sample's own beams, so its rows keep
            # their own encoder keys.  A finished sample's beam_idx entries are 0 (its out_indices are never set): its
            # rows take sample 0's self cache, as in HF, while keeping their own cross rows.  Those rows only ever emit
            # pad_token_id from then on, so which keys they attend to changes no output.
            past.reorder_(beam_idx)
            return past
        if self.encoder_states is not None:
            self.encoder_states = self.encoder_states.index_select(0, beam_idx.to(self.encoder_states.device))
        return [None if layer is None else tuple(t.index_select(0, beam_idx.to(t.device)) for t in layer) for layer in past]

    def prepare_inputs_for_generation(self, input_ids, past=None, encoder_attn_mask=None, encoder_decoder_attn_mask=None,
                                      use_cache=None, encoder_input_ids=None, encoder_outputs=None, **kwargs):
        if past is not None and use_cache:
            input_ids = input_ids[:, -1:]
        return {"encoder_input_ids": encoder_input_ids, "decoder_input_ids": input_ids,
                "encoder_attn_mask": encoder_attn_mask, "encoder_decoder_attn_mask": encoder_decoder_attn_mask,
                "use_cache": bool(use_cache)}


class MT5Loss(nn.Module):
    def __init__(self):
        super().__init__()
        self.lm_loss = ParallelCrossEntropyLoss()

    def forward(self, logits, lm_labels, loss_mask):
        per_token = self.lm_loss(logits, lm_labels)
        mask = loss_mask.float()
        return {"masked_lm_loss": (per_token * mask).sum() / mask.sum().clamp(min=1.0)}


class MT5ForPreTraining(nn.Module):
    def __init__(self, cfg) -> None:
        super().__init__()
        self.cfg = cfg
        self.mt5_model = MT5Model(cfg) if cfg.get("model_type", "mt5") == "mt5" else None
        if self.mt5_model is None:
            self.t5_model = MT5Model(cfg)
        self.loss_func = MT5Loss()

    @property
    def backbone(self):
        return self.mt5_model if self.mt5_model is not None else self.t5_model

    def set_cache(self, encoder_states, past_key_values):
        self.backbone.set_cache(encoder_states, past_key_values)

    def forward(self, encoder_input_ids, decoder_input_ids, encoder_attn_mask, decoder_attn_mask,
                encoder_decoder_attn_mask, lm_labels=None, loss_mask=None, use_cache=False):
        logits = self.backbone(encoder_input_ids, decoder_input_ids, encoder_attn_mask, decoder_attn_mask,
                               encoder_decoder_attn_mask, use_cache=use_cache)["logits"]
        if lm_labels is not None:
            return self.loss_func(logits, lm_labels, loss_mask)
        return {"prediction_scores": logits}

    @staticmethod
    def set_pipeline_stage_id(model):
        return model

    @staticmethod
    def set_activation_checkpoint(model):
        return model
