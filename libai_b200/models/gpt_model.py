"""GPT-2 language model.

Spec: reference libai/models/gpt_model.py — ``GPTModel`` (:71-215; VocabEmbedding + learned
positions + L causal ``TransformerLayer`` + final LN + tied ``LMLogits``), ``GPTEmbedding``
(:217-255), ``Transformer`` (:258-309), ``GPTLoss`` (:312-320, mean over all tokens),
``GPTForPreTraining`` (:323-357; returns ``{"lm_loss"}`` with labels else
``{"prediction_scores"}``).  Parameter names match the reference so checkpoints / HF loaders
line up.  ``CasualMask`` (:35-68) is kept for API parity; the attention kernel applies
causality itself and never materialises a ``[b,1,s,s]`` mask.
"""
from __future__ import annotations

import torch
from torch import nn

from libai_b200.layers.dropout import Dropout

from libai_b200.config import configurable
from libai_b200.layers import (
    Embedding,
    LayerNorm,
    LMLogits,
    ParallelCrossEntropyLoss,
    TransformerLayer,
    VocabEmbedding,
)
from libai_b200.layers._param import create_parameter, xavier_normal_
from libai_b200.layers.attention import AttnMaskType
from libai_b200.layers.embedding import set_sp_shape
from libai_b200.parallel import mappings
from libai_b200.utils import distributed as dutil

from .utils.pipeline_model import PipelineStageMixin
from .utils.weight_init import init_method_normal, scaled_init_method_normal


class CasualMask(nn.Module):
    """Lower-triangular ``[1, 1, s, s]`` mask combined with an optional padding mask."""

    def __init__(self, max_positions=1024, *, layer_idx=0):
        super().__init__()
        self.max_positions = max_positions

    def forward(self, input_ids, past_length=0, attention_mask=None):
        bsz, tgt_len = input_ids.shape
        src_len = past_length + tgt_len
        mask = torch.ones(src_len, src_len, dtype=torch.int8, device=input_ids.device).tril()
        mask = mask[src_len - tgt_len : src_len, :src_len][None, None].expand(bsz, 1, tgt_len, src_len)
        if attention_mask is not None:
            assert attention_mask.dim() == 4, "please extend the attention mask first"
            mask = mask * attention_mask.to(mask.dtype)
        return mask


class GPTEmbedding(nn.Module):
    def __init__(self, vocab_size, hidden_size, max_seq_length, init_method=xavier_normal_,
                 embedding_dropout_prob=0.0, amp_enabled=False):
        super().__init__()
        self.token_embeddings = VocabEmbedding(vocab_size, hidden_size, init_method=init_method, amp_enabled=amp_enabled)
        self.position_embeddings = Embedding(max_seq_length, hidden_size, init_method=init_method, amp_enabled=amp_enabled)
        self.dropout = Dropout(embedding_dropout_prob)
        self.max_seq_length = max_seq_length

    def forward(self, input_ids, past_length=0, position_ids=None):
        """``position_ids`` (int64 ``[s]``, shared by the batch): the positions of the tokens, by default
        ``past_length + i``; a cached step derives them from its cache's lengths on the device."""
        bsz, seq_length = input_ids.shape
        if position_ids is None:
            position_ids = torch.arange(past_length, past_length + seq_length, device=input_ids.device)
        token_embeds = self.token_embeddings(input_ids)
        position_embeds = self.position_embeddings(position_ids)
        x = self.dropout(token_embeds + position_embeds.unsqueeze(0))
        if dutil.get_dist_util().sequence_parallel:
            set_sp_shape(bsz, seq_length)
            x = mappings.scatter_to_sp(x.reshape(-1, x.shape[-1]))
        return x


class Transformer(nn.Module):
    def __init__(
        self, hidden_layers, hidden_size, ffn_hidden_size, num_attention_heads,
        attention_dropout_prob=0.0, output_dropout_prob=0.0, layernorm_epsilon=1e-5,
        init_method=xavier_normal_, output_layer_init_method=None, bias_gelu_fusion=False,
        bias_dropout_fusion=False, scale_mask_softmax_fusion=False,
        apply_query_key_layer_scaling=False, apply_residual_post_layernorm=False,
    ):
        super().__init__()
        self.hidden_layers = hidden_layers
        self.layers = nn.ModuleList(
            [
                TransformerLayer(
                    hidden_size, ffn_hidden_size, num_attention_heads,
                    attention_dropout_prob=attention_dropout_prob,
                    output_dropout_prob=output_dropout_prob,
                    layernorm_epsilon=layernorm_epsilon,
                    init_method=init_method, output_layer_init_method=output_layer_init_method,
                    bias_gelu_fusion=bias_gelu_fusion, bias_dropout_fusion=bias_dropout_fusion,
                    scale_mask_softmax_fusion=scale_mask_softmax_fusion,
                    apply_query_key_layer_scaling=apply_query_key_layer_scaling,
                    apply_residual_post_layernorm=apply_residual_post_layernorm,
                    attn_mask_type=AttnMaskType.causal, layer_idx=i,
                )
                for i in range(hidden_layers)
            ]
        )
        self.layernorm_f = LayerNorm(hidden_size, eps=layernorm_epsilon, layer_idx=-1)

    def forward(self, hidden_states, attention_mask=None):
        for layer in self.layers:
            hidden_states = layer(hidden_states, attention_mask)
        return self.layernorm_f(hidden_states)


class GPTModel(nn.Module, PipelineStageMixin):
    """GPT-2; ``forward`` returns the (vocab-split) logits."""

    # `train.dist.sequence_parallel = "auto"` resolves to True for this model (token-sharded activations between
    # the tensor-parallel blocks are handled by its embeddings / heads)
    supports_sequence_parallel = True

    @configurable
    def __init__(
        self, hidden_layers, vocab_size, hidden_size, ffn_hidden_size, num_attention_heads,
        max_seq_length=1024, embedding_dropout_prob=0.0, attention_dropout_prob=0.0,
        output_dropout_prob=0.0, layernorm_epsilon=1e-5, initializer_range=0.02,
        use_scaled_init_for_output_weights=True, bias_gelu_fusion=False, bias_dropout_fusion=False,
        scale_mask_softmax_fusion=False, apply_query_key_layer_scaling=False,
        apply_residual_post_layernorm=False, amp_enabled=False,
    ):
        super().__init__()
        init_method = init_method_normal(sigma=initializer_range)
        output_layer_init_method = (
            scaled_init_method_normal(initializer_range, hidden_layers)
            if use_scaled_init_for_output_weights
            else init_method
        )
        self.hidden_size, self.vocab_size = hidden_size, vocab_size
        self.embeddings = GPTEmbedding(
            vocab_size, hidden_size, max_seq_length, init_method=init_method,
            embedding_dropout_prob=embedding_dropout_prob, amp_enabled=amp_enabled,
        )
        self.transformer = Transformer(
            hidden_layers, hidden_size, ffn_hidden_size, num_attention_heads,
            attention_dropout_prob=attention_dropout_prob, output_dropout_prob=output_dropout_prob,
            layernorm_epsilon=layernorm_epsilon, init_method=init_method,
            output_layer_init_method=output_layer_init_method, bias_gelu_fusion=bias_gelu_fusion,
            bias_dropout_fusion=bias_dropout_fusion, scale_mask_softmax_fusion=scale_mask_softmax_fusion,
            apply_query_key_layer_scaling=apply_query_key_layer_scaling,
            apply_residual_post_layernorm=apply_residual_post_layernorm,
        )
        self.lm_head = LMLogits(vocab_size, bias=False)
        # Tied embedding under pipeline parallelism: the last stage keeps its own copy of the word
        # embedding (same init); the engine all-reduces the two gradients over the embedding group
        # (the reference ships the weight stage0→last every step: lm_logits.py:44).
        topo = dutil.get_dist_util()
        self.tied_weight_copy = None
        if topo.pipeline_parallel_size > 1:
            self.tied_weight_copy = create_parameter(
                (vocab_size, hidden_size), init_method, tp_dim=0, layer_idx=-1,
                shared_with=self.embeddings.token_embeddings.weight,
            )
            self.tied_weight_copy.shared_from = "embeddings.token_embeddings.weight"
            self.embeddings.token_embeddings.weight.is_tied_source = True

    @classmethod
    def from_config(cls, cfg):
        keys = (
            "hidden_layers vocab_size hidden_size ffn_hidden_size num_attention_heads max_seq_length "
            "embedding_dropout_prob attention_dropout_prob output_dropout_prob layernorm_epsilon "
            "initializer_range use_scaled_init_for_output_weights bias_gelu_fusion bias_dropout_fusion "
            "scale_mask_softmax_fusion apply_query_key_layer_scaling apply_residual_post_layernorm amp_enabled"
        ).split()
        return {k: cfg[k] for k in keys}

    def word_embeddings_weight(self):
        topo = dutil.get_dist_util()
        if topo.pipeline_parallel_size > 1 and topo.is_last_stage and not topo.is_first_stage:
            return self.tied_weight_copy
        return self.embeddings.token_embeddings.weight

    # ---- pipeline protocol ---------------------------------------------------------------------
    def stage_pre(self, input_ids, **_):
        return self.embeddings(input_ids, 0)

    def stage_layers(self):
        return self.transformer.layers

    def stage_post(self, hidden, **_):
        hidden = self.transformer.layernorm_f(hidden)
        logits = self.lm_head(hidden, self.word_embeddings_weight())
        return logits

    def forward(self, input_ids):
        return self.forward_stage({"input_ids": input_ids})


class GPTLoss(nn.Module):
    def __init__(self) -> None:
        super().__init__()
        self.lm_loss = ParallelCrossEntropyLoss()

    def forward(self, logits, lm_labels):
        if logits.dim() == 2:  # token-flattened logits (sequence-parallel path)
            logits = logits.view(lm_labels.shape[0], lm_labels.shape[1], -1)
        return {"lm_loss": self.lm_loss(logits, lm_labels).mean()}


class GPTForPreTraining(nn.Module, PipelineStageMixin):
    """GPT-2 with the LM loss on top."""

    # `train.dist.sequence_parallel = "auto"` resolves to True for this model (token-sharded activations between
    # the tensor-parallel blocks are handled by its embeddings / heads)
    supports_sequence_parallel = True

    def __init__(self, cfg) -> None:
        super().__init__()
        self.GPT_model = GPTModel(cfg)
        self.loss_func = GPTLoss()

    def forward(self, input_ids, labels=None):
        return self.forward_stage({"input_ids": input_ids, "labels": labels})

    # pipeline protocol: delegate to the backbone, add the loss on the last stage
    def stage_pre(self, input_ids, **_):
        return self.GPT_model.stage_pre(input_ids)

    def stage_layers(self):
        return self.GPT_model.stage_layers()

    def stage_post(self, hidden, labels=None, **_):
        logits = self.GPT_model.stage_post(hidden)
        if labels is not None:
            return self.loss_func(logits, labels)
        if logits.dim() == 2:
            logits = logits.view(-1, *([1] * 0), logits.shape[-1])
        return {"prediction_scores": logits}

    @staticmethod
    def set_pipeline_stage_id(model: nn.Module):
        """Kept for API parity: stage placement is decided at construction time through each
        layer's ``layer_idx`` (embeddings → stage of layer 0, final LN / head / loss → stage of
        layer −1), so there is nothing left to tag."""
        return model

    @staticmethod
    def set_activation_checkpoint(model):
        model.activation_checkpoint = True
        return model
