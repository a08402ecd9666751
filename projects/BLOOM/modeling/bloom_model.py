"""BLOOM: ALiBi causal decoder (LayerNorm, GELU, tied embeddings).

Spec: reference projects/BLOOM/modeling/{bloom_model.py,attention.py,mask.py,mlp.py,transformers.py} —
``build_alibi_tensor`` (mask.py:65-101: per-head slopes ``2^(-8i/n)`` with the closest-power-of-two rule, bias =
slope × key position counted over the attention mask), ``BloomAttention`` (fused per-head interleaved qkv,
``baddbmm(alibi, q, kᵀ, beta=1, alpha=1/sqrt(d))``), ``BloomModel`` (:29-255) with embedding LayerNorm and a
final ``ln_f``, ``BloomForCausalLM`` (:258-420) with the generation hooks.  Names follow the HF checkpoint layout
(``word_embeddings``, ``h.N.self_attention.query_key_value`` …) so the loader is a prefix strip.

The kernels evaluate ALiBi from the slopes as ``slope·(j − i − (sk − sq))``.  For a left- or right-padded row that
differs from the bias above (key position counted over the mask) by a constant along each query row, which softmax
ignores, so the flash and decode kernels compute BLOOM's attention exactly with ``kv_start`` / ``kv_lens``.
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional

import torch
from torch import nn

from libai_b200.config import configurable
from libai_b200.inference.generator.generation_utils import Generator
from libai_b200.inference.kv_cache import KVCacheLayer, KVCacheOwner, StaticKVCache, padding_bounds
from libai_b200.layers import LayerNorm, Linear, LMLogits, ParallelCrossEntropyLoss, VocabEmbedding
from libai_b200.models.utils.weight_init import init_method_normal
from libai_b200.ops import functional as OF
from libai_b200.ops import use_native
from libai_b200.parallel import mappings
from libai_b200.utils import distributed as dutil


def alibi_slopes(num_heads: int) -> torch.Tensor:
    closest = 2 ** math.floor(math.log2(num_heads))
    base = 2.0 ** (-(2.0 ** -(math.log2(closest) - 3)))
    slopes = torch.pow(torch.tensor(base), torch.arange(1, closest + 1, dtype=torch.float32))
    if closest != num_heads:
        extra_base = 2.0 ** (-(2.0 ** -(math.log2(2 * closest) - 3)))
        n_extra = min(closest, num_heads - closest)
        slopes = torch.cat([slopes, torch.pow(torch.tensor(extra_base), torch.arange(1, 1 + 2 * n_extra, 2, dtype=torch.float32))])
    return slopes


def build_alibi_tensor(attention_mask: torch.Tensor, num_heads: int, dtype=torch.float32) -> torch.Tensor:
    """``[b, heads, 1, k]`` additive bias; key positions are counted over the non-padded tokens."""
    pos = ((attention_mask.long().cumsum(dim=-1) - 1) * attention_mask.long())[:, None, None, :]
    return (alibi_slopes(num_heads).to(attention_mask.device)[None, :, None, None] * pos).to(dtype)


class AttentionInputs(NamedTuple):
    """What every layer's attention takes besides its hidden states, decided once per forward: the slopes of all heads
    (fp32 ``[n_head]``), and how keys are masked.  ``bias`` + ``mask`` (a dense ALiBi ``[b, heads, 1, k]`` and a
    dense ``[b, 1, q, k]`` visibility) select the reference math; otherwise attention is causal with the slopes,
    ``kv_lens`` carrying right padding and ``kv_start`` left padding (in cached generation: ``cache.kv_start``)."""

    slopes: torch.Tensor
    bias: Optional[torch.Tensor] = None
    mask: Optional[torch.Tensor] = None
    kv_lens: Optional[torch.Tensor] = None
    kv_start: Optional[torch.Tensor] = None


class BloomAttention(nn.Module):
    def __init__(self, hidden_size, n_head, hidden_dropout, attention_dropout, init_method, layer_idx):
        super().__init__()
        topo = dutil.get_dist_util()
        self.num_heads, self.head_dim = n_head, hidden_size // n_head
        self.local_heads = n_head // topo.tensor_parallel_size
        self.head_size = self.head_dim   # what a StaticKVCache sizes itself by (KVCacheOwner)
        self.query_key_value = Linear(hidden_size, 3 * hidden_size, bias=True, parallel="col", init_method=init_method, layer_idx=layer_idx)
        self.dense = Linear(hidden_size, hidden_size, bias=True, parallel="row", init_method=init_method, layer_idx=layer_idx)
        self.attention_dropout, self.hidden_dropout = attention_dropout, nn.Dropout(hidden_dropout)

    def forward(self, hidden, residual, inputs: AttentionInputs, cache: Optional[KVCacheLayer] = None):
        b, s = hidden.shape[:2]
        a, d = self.local_heads, self.head_dim
        rank = dutil.get_dist_util().tp_rank
        slopes = inputs.slopes[rank * a : (rank + 1) * a]   # this rank's heads (a contiguous view)
        bias = None if inputs.bias is None else inputs.bias[:, rank * a : (rank + 1) * a]
        qkv = self.query_key_value(hidden).view(b, s, a, 3 * d)   # per-head [q|k|v]: the MHA packed layout
        if cache is not None:
            ctx = cache.attend(cache.append(qkv), scale=1.0 / math.sqrt(d), mask=inputs.mask, bias=bias,
                               alibi_slopes=slopes)
        else:
            q, k, v = (t.transpose(1, 2) for t in OF.split_qkv(qkv))   # [b, a, s, d] views
            if bias is None:
                ctx = OF.attention(q, k, v, causal=True, scale=1.0 / math.sqrt(d), alibi_slopes=slopes,
                                   kv_lens=inputs.kv_lens, kv_start=inputs.kv_start,
                                   dropout_p=self.attention_dropout, training=self.training)
            else:
                ctx = OF.attention(q, k, v, causal=False, scale=1.0 / math.sqrt(d), mask=inputs.mask, bias=bias,
                                   dropout_p=self.attention_dropout, training=self.training)
            ctx = ctx.transpose(1, 2)
        out = self.dense(ctx.reshape(b, s, a * d))
        return residual + self.hidden_dropout(out)


class BloomMLP(nn.Module):
    def __init__(self, hidden_size, hidden_dropout, init_method, layer_idx):
        super().__init__()
        self.dense_h_to_4h = Linear(hidden_size, 4 * hidden_size, parallel="col", init_method=init_method, layer_idx=layer_idx)
        self.dense_4h_to_h = Linear(4 * hidden_size, hidden_size, parallel="row", init_method=init_method, layer_idx=layer_idx)
        self.dropout = nn.Dropout(hidden_dropout)

    def forward(self, hidden, residual):
        return residual + self.dropout(self.dense_4h_to_h(self.dense_h_to_4h(hidden, act="gelu_tanh")))


class BloomBlock(nn.Module):
    def __init__(self, hidden_size, n_head, layer_norm_epsilon, hidden_dropout, attention_dropout,
                 apply_residual_connection_post_layernorm, init_method, layer_idx):
        super().__init__()
        self.layer_idx = layer_idx
        self.input_layernorm = LayerNorm(hidden_size, eps=layer_norm_epsilon, layer_idx=layer_idx)
        self.self_attention = BloomAttention(hidden_size, n_head, hidden_dropout, attention_dropout, init_method, layer_idx)
        self.post_attention_layernorm = LayerNorm(hidden_size, eps=layer_norm_epsilon, layer_idx=layer_idx)
        self.mlp = BloomMLP(hidden_size, hidden_dropout, init_method, layer_idx)
        self.post_ln_residual = apply_residual_connection_post_layernorm

    def forward(self, hidden, inputs: AttentionInputs, cache: Optional[KVCacheLayer] = None):
        ln = self.input_layernorm(hidden)
        attn = self.self_attention(ln, ln if self.post_ln_residual else hidden, inputs, cache)
        ln2 = self.post_attention_layernorm(attn)
        return self.mlp(ln2, ln2 if self.post_ln_residual else attn)


class BloomModel(nn.Module):
    @configurable
    def __init__(self, vocab_size, hidden_size, hidden_layers, n_head, padding_idx=None, pretraining_tp=1,
                 slow_but_exact=False, initializer_range=0.02, apply_residual_connection_post_layernorm=False,
                 hidden_dropout=0.0, attention_dropout=0.0, amp_enabled=False, layer_norm_epsilon=1e-12, cfg=None):
        super().__init__()
        self.cfg, self.n_head, self.hidden_layers = cfg, n_head, hidden_layers
        self.head_dim = hidden_size // n_head
        init_method = init_method_normal(initializer_range)
        self.word_embeddings = VocabEmbedding(vocab_size, hidden_size, padding_idx=padding_idx, init_method=init_method,
                                              amp_enabled=amp_enabled)
        self.word_embeddings_layernorm = LayerNorm(hidden_size, eps=layer_norm_epsilon, layer_idx=0)
        self.h = nn.ModuleList([
            BloomBlock(hidden_size, n_head, layer_norm_epsilon, hidden_dropout, attention_dropout,
                       apply_residual_connection_post_layernorm, init_method, layer_idx=i)
            for i in range(hidden_layers)])
        self.ln_f = LayerNorm(hidden_size, eps=layer_norm_epsilon, layer_idx=-1)
        # the slopes of all heads (each tensor-parallel rank reads its own); not a checkpoint entry
        self.register_buffer("alibi_slopes", alibi_slopes(n_head), persistent=False)

    @classmethod
    def from_config(cls, cfg):
        keys = ("vocab_size hidden_size hidden_layers n_head padding_idx pretraining_tp slow_but_exact initializer_range "
                "apply_residual_connection_post_layernorm hidden_dropout attention_dropout amp_enabled layer_norm_epsilon").split()
        out = {k: cfg[k] for k in keys if k in cfg}
        out["cfg"] = cfg
        return out

    def _dense_inputs(self, slopes, input_ids, past: int, attention_mask) -> AttentionInputs:
        """The reference math's inputs: HF's ALiBi (key positions counted over the mask) and the causal padding mask."""
        b, q = input_ids.shape
        k = past + q
        if attention_mask is None:
            attention_mask = torch.ones(b, k, dtype=torch.long, device=input_ids.device)
        causal = torch.ones(k, k, dtype=torch.bool, device=input_ids.device).tril()[k - q :]
        mask = causal[None, None] & attention_mask.bool()[:, None, None, :]
        return AttentionInputs(slopes, bias=build_alibi_tensor(attention_mask, self.n_head, torch.float32), mask=mask)

    def forward(self, input_ids, attention_mask=None, past_key_values=None):
        """``past_key_values``: the :class:`StaticKVCache` of cached generation (appended to in place), or None.
        ``attention_mask`` ``[b, past + s]``: 1 = token, 0 = padding."""
        hidden = self.word_embeddings_layernorm(self.word_embeddings(input_ids))
        if self.alibi_slopes.device != hidden.device or self.alibi_slopes.dtype != torch.float32:
            # a model placed on the GPU or cast (``.to(torch.bfloat16)`` casts buffers too): the kernels take fp32
            self.alibi_slopes = alibi_slopes(self.n_head).to(hidden.device)
        slopes = self.alibi_slopes
        if isinstance(past_key_values, StaticKVCache):
            cache = past_key_values
            dense = cache.step_needs_dense_mask(attention_mask, flash=cache.flash_attention())
            inputs = self._dense_inputs(slopes, input_ids, cache.length, attention_mask) if dense else \
                AttentionInputs(slopes)
            for i, block in enumerate(self.h):
                hidden = block(hidden, inputs, cache.layer(i))
            cache.advance(input_ids.shape[1])
            return self.ln_f(hidden)
        # the flash kernels take right / left padding as kv_lens / kv_start instead of a dense mask
        flash = use_native(hidden) and hidden.dtype == torch.bfloat16 and OF.flash_head_dim_supported(self.head_dim)
        padded = attention_mask is not None and not bool(attention_mask.all())
        inputs = AttentionInputs(slopes)
        bounds = padding_bounds(attention_mask) if padded and flash else None
        if bounds is not None:
            inputs = inputs._replace(kv_lens=bounds[0], kv_start=bounds[1])
        elif padded or not hidden.is_cuda:
            inputs = self._dense_inputs(slopes, input_ids, 0, attention_mask)
        for block in self.h:
            hidden = block(hidden, inputs)
        return self.ln_f(hidden)


class BloomForCausalLM(nn.Module, KVCacheOwner, Generator):
    speculative_decoding = True
    continuous_batching = True

    @configurable
    def __init__(self, cfg=None, **kwargs):
        super().__init__()
        self.cfg = cfg
        self.transformer = BloomModel(cfg=cfg, **kwargs) if cfg is None else BloomModel(cfg)
        self.lm_head = LMLogits(self.transformer.word_embeddings.num_embeddings, bias=False)
        self.loss = ParallelCrossEntropyLoss()

    @classmethod
    def from_config(cls, cfg):
        return {"cfg": cfg}

    def forward(self, input_ids, attention_mask=None, labels=None, use_cache=False):
        cache = self._prepare_cache(input_ids) if use_cache else None
        hidden = self.transformer(input_ids, attention_mask, cache)
        if cache is not None:
            self.past_length = cache.length
        logits = self.lm_head(hidden, self.transformer.word_embeddings.weight)
        if labels is not None:
            shift = self.loss(logits[:, :-1].contiguous(), labels[:, 1:].contiguous())
            return {"loss": shift.mean()}
        if dutil.get_dist_util().tensor_parallel_size > 1:
            logits = mappings.gather_from_tp(logits)
        return {"logits": logits}

    # ---- KV cache (KVCacheOwner) ----------------------------------------------------------------
    def _cache_attention_modules(self):
        return [block.self_attention for block in self.transformer.h]

    def continuous_batching_logits(self, input_ids, cache):
        """The logits ``[1, T, vocab]`` of one step of a ``GenerationEngine`` on its ``RaggedPagedKVCache``: ALiBi
        scores each key by its distance inside its own sequence."""
        return self.lm_head(self.transformer(input_ids, None, cache), self.transformer.word_embeddings.weight)

    def continuous_batching_max_length(self):
        return None   # ALiBi: no position table
