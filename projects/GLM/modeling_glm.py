"""GLM: autoregressive blank-infilling transformer (2-D positions, prefix-LM masks, hidden-state memories).

Spec: reference projects/GLM/modeling_glm.py — ``Transformer`` (:30-80, pre-LN GPT-style blocks whose attention
reads ``[memory; hidden]`` for keys/values), ``GLMModel`` (:83-260: embeddings with position + block-position
tables, ``build_mask_matrix`` from a scalar / per-sample separator = bidirectional context + causal generation part,
``update_mems`` keeping the inputs of every layer as the generation cache), ``GLMLoss``, ``GLMForMultipleChoice``
(:273-309), ``GLMForConditionalGeneration`` (:312-470) and projects/GLM/layers/*.

Attention runs natively as a prefix LM: :func:`prefix_lm` turns GLM's mask inputs into the flash kernels' arguments
(``prefix_lens``, the context's left padding in ``kv_start``), and anything it cannot express keeps the dense mask and
the reference math.  ``generate(use_cache=True)`` decodes on a :class:`StaticKVCache`: the prefill is flash attention
with the prefix, each later step is plain causal decoding over the cache.  ``use_cache=False`` keeps the hidden-state
memories.
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional

import torch
from torch import nn

from libai_b200.config import configurable
from libai_b200.inference.generator.generation_utils import Generator
from libai_b200.inference.kv_cache import KVCacheLayer, KVCacheOwner, StaticKVCache
from libai_b200.layers import Embedding, LayerNorm, Linear, LMLogits, MLP, VocabEmbedding
from libai_b200.models.utils.weight_init import init_method_normal, scaled_init_method_normal
from libai_b200.ops import functional as OF
from libai_b200.ops import use_native
from libai_b200.parallel import mappings
from libai_b200.utils import distributed as dutil


class PrefixLM(NamedTuple):
    """GLM's visibility as the flash kernels take it: key ``j`` is visible to query ``i`` of sample ``b`` iff
    ``kv_start[b] <= j`` and (``j <= i + mem_len`` or ``j < prefix_lens[b]``), int32 ``[b]`` device tensors.  ``order``
    (long ``[b, s]``, or None) is the row order in which the tokens must run for this to hold: ``x.gather(1, order)``
    puts a right-padded context's padding first."""

    prefix_lens: torch.Tensor
    kv_start: Optional[torch.Tensor] = None
    order: Optional[torch.Tensor] = None


def prefix_lm(attention_mask, batch: int, q: int, mem_len: int = 0) -> Optional[PrefixLM]:
    """The flash kernels' arguments for GLM's mask inputs, or None when only the dense mask expresses them.

    - A scalar or per-sample separator ``sep`` (the context is ``[0, sep)``): ``prefix_lens = mem_len + sep``.
    - A dense ``[b, 1, q, q]`` 0/1 mask without memories (the tokenizer's ``generation_attention_mask`` or training
      ``attention_mask``): checked, with one host sync, to equal the prefix-LM rule with a left-padded context
      (``kv_start`` = the padding), or with a right-padded one (``GLMTokenizerMixin.__call__``'s layout), which runs
      with each sample's padding moved in front of its context (``order``).  Moving tokens together with their
      position ids is exact: GLM's positions live in the embeddings, and attention does not depend on key order.
    - Anything else (a hole inside the context, an arbitrary mask, a dense mask over memories): None."""
    m = attention_mask
    device = m.device
    if m.numel() == 1 or (m.numel() == batch and m.dim() <= 1):
        sep = m.reshape(-1).to(device=device, dtype=torch.int32).expand(batch)
        return PrefixLM((sep + mem_len).to(torch.int32).contiguous())
    if mem_len != 0 or m.dim() != 4 or tuple(m.shape) != (batch, 1, q, q):
        return None
    mask = m[:, 0].bool()
    j = torch.arange(q, device=device)
    never = ~mask.any(1)                       # keys no query sees: the context's padding
    n = never.sum(1)
    order = torch.argsort(torch.where(never, j - q, j), dim=1)   # those first, the others in their order
    mp = mask.gather(1, order[:, :, None].expand(-1, q, q)).gather(2, order[:, None, :].expand(-1, q, q))
    pre = torch.where(mp[:, 0], j + 1, 0).amax(1)   # the first row sees the context: it ends the prefix
    first, last = torch.where(never, j, q).amin(1), torch.where(never, j + 1, 0).amax(1)
    # the padding is one run, before the context (left) or right after it (right); every row sees a key
    run = (n == 0) | ((last - first == n) & ((first == 0) | (last == pre)))
    vis = OF.visible_keys(q, q, causal=True, kv_start=n, prefix_lens=pre, device=device)[:, 0]
    ok = (vis == mp).all() & run.all() & (pre > n).all()
    ok, moved = torch.stack((ok, ((n > 0) & (first > 0)).any())).tolist()
    if not ok:
        return None
    return PrefixLM(pre.to(torch.int32), n.to(torch.int32), order if moved else None)


def _native_attention(x: torch.Tensor, head_size: int) -> bool:
    """Whether the layers' attention over activations like ``x`` runs the flash kernels (bf16 on the GPU and a head
    dim they take); only then is it worth classifying a dense mask."""
    return use_native(x) and x.dtype == torch.bfloat16 and OF.flash_head_dim_supported(head_size)


class GLMAttentionInputs(NamedTuple):
    """What every layer's attention sees: a dense 0/1 ``mask`` (reference math), or the prefix-LM rule."""

    mask: Optional[torch.Tensor] = None
    prefix_lens: Optional[torch.Tensor] = None
    kv_start: Optional[torch.Tensor] = None


class GLMEmbedding(nn.Module):
    def __init__(self, vocab_size, hidden_size, max_seq_length, padding_idx=None, init_method=None,
                 embedding_dropout_prob=0.0, amp_enabled=False, block_position_encoding=False):
        super().__init__()
        self.block_position_encoding = block_position_encoding
        self.word_embeddings = VocabEmbedding(vocab_size, hidden_size, padding_idx=padding_idx, init_method=init_method,
                                              amp_enabled=amp_enabled)
        n_pos = max_seq_length + 1 if block_position_encoding else max_seq_length
        self.position_embeddings = Embedding(n_pos, hidden_size, init_method=init_method, amp_enabled=amp_enabled)
        if block_position_encoding:
            self.block_position_embeddings = Embedding(n_pos, hidden_size, init_method=init_method, amp_enabled=amp_enabled)
        self.embedding_dropout = nn.Dropout(embedding_dropout_prob)

    def forward(self, input_ids, position_ids=None):
        b, s = input_ids.shape
        if position_ids is None:
            pos = torch.arange(s, device=input_ids.device)[None].expand(b, s)
            position_ids = torch.stack([pos, torch.zeros_like(pos)], 1) if self.block_position_encoding else pos
        x = self.word_embeddings(input_ids)
        if self.block_position_encoding:
            x = x + self.position_embeddings(position_ids[:, 0]) + self.block_position_embeddings(position_ids[:, 1])
        else:
            x = x + self.position_embeddings(position_ids)
        return self.embedding_dropout(x)


class GLMAttention(nn.Module):
    def __init__(self, hidden_size, num_attention_heads, attention_dropout_prob, output_dropout_prob, init_method,
                 output_layer_init_method, attention_scale, layer_idx):
        super().__init__()
        topo = dutil.get_dist_util()
        self.local_heads = num_attention_heads // topo.tensor_parallel_size
        self.head_size = hidden_size // num_attention_heads   # with local_heads: what a StaticKVCache sizes itself by
        self.attention_scale = attention_scale
        self.query_key_value = Linear(hidden_size, 3 * hidden_size, parallel="col", init_method=init_method, layer_idx=layer_idx)
        self.dense = Linear(hidden_size, hidden_size, parallel="row", init_method=output_layer_init_method, layer_idx=layer_idx)
        self.attention_dropout_prob, self.output_dropout = attention_dropout_prob, nn.Dropout(output_dropout_prob)

    def forward(self, hidden, inputs: GLMAttentionInputs, mem=None, cache: Optional[KVCacheLayer] = None):
        b, q_len, _ = hidden.shape
        a, d = self.local_heads, self.head_size
        scale = 1.0 / math.sqrt(d)
        if cache is not None:   # the new tokens' k, v go to the cache; the prefill alone takes the prefix
            qkv = self.query_key_value(hidden).view(b, q_len, a, 3 * d)   # per-head [q|k|v]
            ctx = cache.attend(cache.append(qkv), scale=scale, mask=inputs.mask, prefix_lens=inputs.prefix_lens)
            return self.output_dropout(self.dense(ctx.reshape(b, q_len, a * d)))
        source = hidden if mem is None else torch.cat((mem, hidden), dim=1)
        qkv = self.query_key_value(source).view(b, -1, a, 3 * d).permute(0, 2, 1, 3)
        q, k, v = qkv[:, :, -q_len:, :d], qkv[..., d : 2 * d], qkv[..., 2 * d :]
        if inputs.prefix_lens is not None:
            ctx = OF.attention(q, k, v, causal=True, scale=scale, prefix_lens=inputs.prefix_lens,
                               kv_start=inputs.kv_start, dropout_p=self.attention_dropout_prob, training=self.training)
        else:
            ctx = OF.attention(q, k, v, causal=False, scale=scale, mask=inputs.mask,
                               dropout_p=self.attention_dropout_prob, training=self.training)
        return self.output_dropout(self.dense(ctx.transpose(1, 2).reshape(b, q_len, a * d)))


class GLMLayer(nn.Module):
    def __init__(self, hidden_size, num_attention_heads, attention_dropout_prob, output_dropout_prob, layernorm_epsilon,
                 init_method, output_layer_init_method, attention_scale, layer_idx):
        super().__init__()
        self.layer_idx = layer_idx
        self.input_layernorm = LayerNorm(hidden_size, eps=layernorm_epsilon, layer_idx=layer_idx)
        self.attention = GLMAttention(hidden_size, num_attention_heads, attention_dropout_prob, output_dropout_prob,
                                      init_method, output_layer_init_method, attention_scale, layer_idx)
        self.post_attention_layernorm = LayerNorm(hidden_size, eps=layernorm_epsilon, layer_idx=layer_idx)
        self.mlp = MLP(hidden_size, 4 * hidden_size, output_dropout_prob, init_method, output_layer_init_method,
                       layer_idx=layer_idx)

    def forward(self, hidden, inputs: GLMAttentionInputs, mem=None, cache: Optional[KVCacheLayer] = None):
        ln = self.input_layernorm(hidden)
        mem = self.input_layernorm(mem) if mem is not None else None
        hidden = hidden + self.attention(ln, inputs, mem, cache)
        return self.mlp(self.post_attention_layernorm(hidden), residual=hidden)


class Transformer(nn.Module):
    def __init__(self, num_layers, hidden_size, num_attention_heads, attention_dropout_prob=0.0, output_dropout_prob=0.0,
                 layernorm_epsilon=1e-5, init_method=None, output_layer_init_method=None, attention_scale=1.0):
        super().__init__()
        self.layers = nn.ModuleList([
            GLMLayer(hidden_size, num_attention_heads, attention_dropout_prob, output_dropout_prob, layernorm_epsilon,
                     init_method, output_layer_init_method, attention_scale, layer_idx=i) for i in range(num_layers)])
        self.final_layernorm = LayerNorm(hidden_size, eps=layernorm_epsilon, layer_idx=-1)

    def forward(self, hidden, inputs: GLMAttentionInputs, memory_states=None, cache: Optional[StaticKVCache] = None):
        if cache is not None:
            for i, layer in enumerate(self.layers):
                hidden = layer(hidden, inputs, cache=cache.layer(i))
            return self.final_layernorm(hidden), []
        mem_layers = [hidden.detach()]
        for i, layer in enumerate(self.layers):
            hidden = layer(hidden, inputs, memory_states[i] if memory_states is not None else None)
            mem_layers.append(hidden.detach())
        return self.final_layernorm(hidden), mem_layers


class GLMModel(nn.Module):
    @configurable
    def __init__(self, num_layers, vocab_size, hidden_size, num_attention_heads, max_sequence_length=1024,
                 embedding_dropout_prob=0.0, attention_dropout_prob=0.0, output_dropout_prob=0.0, layernorm_epsilon=1e-5,
                 initializer_range=0.02, use_scaled_init_for_output_weights=True, bias_gelu_fusion=True,
                 bias_dropout_fusion=True, scale_mask_softmax_fusion=False, apply_query_key_layer_scaling=False,
                 amp_enabled=False, block_position_encoding=False, attention_scale=1.0, padding_idx=None, cfg=None):
        super().__init__()
        self.cfg = cfg
        init_method = init_method_normal(initializer_range)
        out_init = scaled_init_method_normal(initializer_range, num_layers) if use_scaled_init_for_output_weights else init_method
        self.embeddings = GLMEmbedding(vocab_size, hidden_size, max_sequence_length, padding_idx, init_method,
                                       embedding_dropout_prob, amp_enabled, block_position_encoding)
        self.transformer = Transformer(num_layers, hidden_size, num_attention_heads, attention_dropout_prob,
                                       output_dropout_prob, layernorm_epsilon, init_method, out_init, attention_scale)
        self.lm_head = LMLogits(vocab_size, bias=False)

    @classmethod
    def from_config(cls, cfg):
        keys = ("num_layers vocab_size hidden_size num_attention_heads max_sequence_length embedding_dropout_prob "
                "attention_dropout_prob output_dropout_prob layernorm_epsilon initializer_range "
                "use_scaled_init_for_output_weights bias_gelu_fusion bias_dropout_fusion scale_mask_softmax_fusion "
                "apply_query_key_layer_scaling amp_enabled block_position_encoding attention_scale padding_idx").split()
        out = {k: cfg[k] for k in keys if k in cfg}
        out["cfg"] = cfg
        return out

    @staticmethod
    def build_mask_matrix(batch_size, seq_length, sep, memory_length=0, device=None):
        """Prefix-LM visibility: everything before ``sep`` is bidirectional context, the rest is causal."""
        m = torch.ones(seq_length, seq_length, dtype=torch.bool, device=device).tril()[None].repeat(batch_size, 1, 1)
        sep_t = torch.as_tensor(sep, device=device).view(-1, 1).expand(batch_size, 1)
        ctx = torch.arange(seq_length, device=device)[None] < sep_t
        m = m | ctx[:, None, :]
        if memory_length > 0:
            m = torch.cat([torch.ones(batch_size, seq_length, memory_length, dtype=torch.bool, device=device), m], dim=2)
        return m[:, None]

    @staticmethod
    def update_mems(hiddens, mems):
        mem_len = mems[0].shape[1] if mems is not None else 0
        if mem_len == 0:
            return list(hiddens)
        return [torch.cat((m, h), dim=1) for m, h in zip(mems, hiddens)]

    def forward(self, input_ids, position_ids=None, attention_mask=None, memory_states=None, output_predict=True,
                kv_cache: Optional[StaticKVCache] = None):
        """``kv_cache``: the :class:`StaticKVCache` of cached generation (appended to in place; no memories are
        returned), or None for the hidden-state memories."""
        b, q = input_ids.shape
        mem_len = memory_states[0].shape[1] if memory_states is not None else 0
        past = kv_cache.length if kv_cache is not None else mem_len
        if attention_mask is None:   # (a fill on the device: a cached step copies nothing from the host)
            attention_mask = torch.full((), q, dtype=torch.long, device=input_ids.device)
        hidden = self.embeddings(input_ids, position_ids)
        # the prefix-LM rule where the kernels run: every uncached call, and the prefill of a cache (a later step
        # sees every cached row, unless the prefill needed the dense mask)
        prefix = None
        if (kv_cache is None or past == 0) and _native_attention(hidden, self.transformer.layers[0].attention.head_size):
            prefix = prefix_lm(attention_mask, b, q, mem_len)
        if prefix is not None:
            inputs = GLMAttentionInputs(prefix_lens=prefix.prefix_lens, kv_start=prefix.kv_start)
            if prefix.order is not None:
                hidden = hidden.gather(1, prefix.order[..., None].expand_as(hidden))
        elif kv_cache is not None and past > 0 and not kv_cache.dense_mask:
            inputs = GLMAttentionInputs()
        elif attention_mask.numel() == 1 or attention_mask.numel() == b and attention_mask.dim() <= 1:
            inputs = GLMAttentionInputs(mask=self.build_mask_matrix(b, q, attention_mask, past, input_ids.device))
        else:
            mask = attention_mask.bool()
            if mask.dim() == 2:
                mask = mask[:, None, None, :]
            inputs = GLMAttentionInputs(mask=mask[..., -q - past :])
        if kv_cache is not None and past == 0:
            kv_cache.dense_mask = prefix is None
            if prefix is not None and prefix.kv_start is not None:
                kv_cache.kv_start.copy_(prefix.kv_start)
        hidden, mem_layers = self.transformer(hidden, inputs, memory_states, kv_cache)
        if kv_cache is not None:
            kv_cache.advance(q)
        if prefix is not None and prefix.order is not None:   # back to the caller's order
            back = torch.argsort(prefix.order, dim=1)[..., None]
            hidden = hidden.gather(1, back.expand_as(hidden))
            mem_layers = [m.gather(1, back.expand_as(m)) for m in mem_layers]
        mem_layers = self.update_mems(mem_layers, memory_states)
        if output_predict:
            hidden = self.lm_head(hidden, self.embeddings.word_embeddings.weight)
            if not self.training and dutil.get_dist_util().tensor_parallel_size > 1:
                hidden = mappings.gather_from_tp(hidden)
        return hidden, mem_layers


class GLMLoss(nn.Module):
    def forward(self, logits, labels):
        return {"lm_loss": torch.nn.functional.cross_entropy(logits.float().reshape(-1, logits.shape[-1]), labels.reshape(-1),
                                                             ignore_index=-100)}


class GLMForMultipleChoice(nn.Module):
    """Score every choice by the sum of the log-probs of its tokens (cloze-style classification)."""

    def __init__(self, cfg):
        super().__init__()
        self.glm = GLMModel(cfg)
        self.loss_func = GLMLoss()

    def forward(self, input_ids=None, position_ids=None, attention_mask=None, choice_ids=None, choice_indices=None,
                labels=None, mems=None, **kwargs):
        logits, _ = self.glm(input_ids, position_ids, attention_mask, mems)
        lp = torch.log_softmax(logits.float(), dim=-1)
        scores = []
        for out, choices, indices in zip(lp, choice_ids, choice_indices):
            scores.append(torch.stack([out[idx.to(out.device), ch.to(out.device)].sum() for ch, idx in zip(choices, indices)]))
        scores = torch.stack(scores)
        if labels is not None:
            return {"loss": torch.nn.functional.cross_entropy(scores, labels), "logits": scores}
        return {"logits": scores}


class GLMForConditionalGeneration(nn.Module, KVCacheOwner, Generator):
    """``use_cache=True`` decodes on a :class:`StaticKVCache` (``generate(kv_cache_dtype="fp8")`` holds it in FP8);
    ``use_cache=False`` carries the hidden-state memories through ``memory_states`` / ``past_key_values``."""

    # the prefix-LM prompt attends bidirectionally: a row's K/V depend on later tokens, so no page can be reused
    prefix_caching = False

    @configurable
    def __init__(self, cfg=None, **kwargs):
        super().__init__()
        self.cfg = cfg
        self.glm = GLMModel(cfg) if cfg is not None else GLMModel(**kwargs)
        self.loss_func = GLMLoss()

    @classmethod
    def from_config(cls, cfg):
        return {"cfg": cfg}

    def forward(self, input_ids=None, position_ids=None, attention_mask=None, labels=None, memory_states=None,
                use_cache=False, **kwargs):
        cache = self._prepare_cache(input_ids) if use_cache and memory_states is None and labels is None else None
        logits, mems = self.glm(input_ids, position_ids, attention_mask, memory_states, kv_cache=cache)
        if labels is not None:
            return self.loss_func(logits, labels)
        if cache is not None:
            self.past_length = cache.length
            return {"logits": logits}
        return {"logits": logits, "past_key_values": mems}

    # ---- KV cache (KVCacheOwner) ----------------------------------------------------------------
    def _cache_attention_modules(self):
        return [layer.attention for layer in self.glm.transformer.layers]

    def _reorder_cache(self, past, beam_idx):
        if past is None or isinstance(past, StaticKVCache):
            return Generator._reorder_cache(self, past, beam_idx)
        return [m.index_select(0, beam_idx.to(m.device)) for m in past]

    def _apply_reordered_cache(self, past):
        pass  # memories travel through ``model_kwargs["past"]``; a StaticKVCache is reordered in place

    def prepare_inputs_for_generation(self, input_ids, past=None, position_ids=None, generation_attention_mask=None,
                                      use_cache=None, **kwargs):
        mask, seq = generation_attention_mask, input_ids.shape[1]
        if past:
            if position_ids is not None:
                position_ids = position_ids[:, :, seq - 1].unsqueeze(-1)
            if mask is not None:
                mask = mask[:, :, seq - 1, :seq].unsqueeze(-2)
            input_ids = input_ids[:, -1:]
        else:
            if position_ids is not None:
                position_ids = position_ids[:, :, :seq]
            if mask is not None:
                mask = mask[:, :, :seq, :seq]
        out = {"input_ids": input_ids, "position_ids": position_ids, "attention_mask": mask}
        if use_cache:
            out["use_cache"] = True
        else:
            out["memory_states"] = past
        return out

    @staticmethod
    def set_pipeline_stage_id(model):
        return model
