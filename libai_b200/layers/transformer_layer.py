"""One transformer block (encoder or decoder flavour).

Spec: reference libai/layers/transformer_layer.py:26-248 — pre-LN by default
(``apply_residual_post_layernorm`` takes the residual *after* the LN instead), optional
cross-attention for decoders, DropPath on both residual branches, KV cache passthrough.
The pipeline hand-off the reference performs inside ``forward`` (``to_global(placement=…)``,
:158) is done by the pipeline engine between stages, not here.
"""
from torch import nn

from libai_b200.inference.kv_cache import KVCacheLayer

from ._param import xavier_normal_
from .attention import AttnMaskType, MultiheadAttention
from .droppath import DropPath
from .layer_norm import LayerNorm
from .mlp import MLP


class TransformerLayer(nn.Module):
    def __init__(
        self,
        hidden_size,
        ffn_hidden_size,
        num_attention_heads,
        is_decoder=False,
        attention_dropout_prob=0.0,
        output_dropout_prob=0.0,
        drop_path_prob=0.0,
        layernorm_epsilon=1e-5,
        init_method=xavier_normal_,
        output_layer_init_method=None,
        bias_gelu_fusion=False,
        bias_dropout_fusion=False,
        scale_mask_softmax_fusion=False,
        apply_query_key_layer_scaling=False,
        apply_residual_post_layernorm=False,
        attn_mask_type=AttnMaskType.padding,
        *,
        layer_idx=0,
    ):
        super().__init__()
        self.hidden_size = hidden_size
        self.ffn_hidden_size = ffn_hidden_size
        self.num_attention_heads = num_attention_heads
        self.attention_dropout_prob = attention_dropout_prob
        self.output_dropout_prob = output_dropout_prob
        self.layernorm_epsilon = layernorm_epsilon
        self.attn_mask_type = attn_mask_type
        self.layer_idx = layer_idx
        self.is_decoder = is_decoder
        self.bias_gelu_fusion = bias_gelu_fusion
        self.bias_dropout_fusion = bias_dropout_fusion
        self.scale_mask_softmax_fusion = scale_mask_softmax_fusion
        self.apply_query_key_layer_scaling = apply_query_key_layer_scaling
        self.apply_residual_post_layernorm = apply_residual_post_layernorm
        self.init_method = init_method
        self.output_layer_init_method = output_layer_init_method or init_method
        self.drop_path = DropPath(drop_path_prob) if drop_path_prob > 0.0 else nn.Identity()
        self.plain_residual = drop_path_prob == 0.0

        self.input_layernorm = LayerNorm(hidden_size, eps=layernorm_epsilon, layer_idx=layer_idx)
        self.self_attention = self.build_attention(is_cross_attention=False)
        self.post_attention_layernorm = LayerNorm(hidden_size, eps=layernorm_epsilon, layer_idx=layer_idx)
        if self.is_decoder:
            self.cross_attention = self.build_attention(is_cross_attention=True)
            self.post_cross_attention_layernorm = LayerNorm(hidden_size, eps=layernorm_epsilon, layer_idx=layer_idx)
        self.mlp = MLP(
            hidden_size, ffn_hidden_size, output_dropout_prob, init_method,
            output_layer_init_method=self.output_layer_init_method,
            bias_gelu_fusion=bias_gelu_fusion, bias_dropout_fusion=bias_dropout_fusion, layer_idx=layer_idx,
        )

    def _branch(self, fn, residual, **kw):
        """residual + drop_path(fn(...)); the add is fused into fn's epilogue when no DropPath."""
        if self.plain_residual:
            return fn(residual=residual, **kw)
        out = fn(residual=None, **kw)
        if isinstance(out, tuple):
            return (residual + self.drop_path(out[0]),) + tuple(out[1:])
        return residual + self.drop_path(out)

    def forward(
        self,
        hidden_states,
        attention_mask=None,
        encoder_states=None,
        encoder_attention_mask=None,
        past_key_value=None,
        use_cache=False,
    ):
        """``past_key_value``: ``(self_k, self_v[, cross_k, cross_v])``; returns hidden states, and
        the updated cache tuple when ``use_cache``."""
        self_past = cross_past = None
        if isinstance(past_key_value, KVCacheLayer):   # preallocated self-attention cache (decoder-only models)
            self_past = past_key_value
        elif past_key_value is not None:
            self_past = past_key_value[:2]
            cross_past = past_key_value[2:] if len(past_key_value) > 2 else None
            cross_past = cross_past or None

        if self.apply_residual_post_layernorm:
            ln = self.input_layernorm(hidden_states)
            residual = ln
        else:   # pre-LN: the skip gradient is folded into the LayerNorm backward kernel
            ln, residual = self.input_layernorm.forward_with_skip(hidden_states)
        attn = self._branch(
            lambda residual, **kw: self.self_attention(ln, residual=residual, **kw),
            residual, attention_mask=attention_mask, past_key_value=self_past, use_cache=use_cache,
        )
        presents = None
        if use_cache:
            attn, presents = attn
        hidden_states = attn

        if self.apply_residual_post_layernorm or self.is_decoder:
            ln = self.post_attention_layernorm(hidden_states)
            post_skip = hidden_states
        else:
            ln, post_skip = self.post_attention_layernorm.forward_with_skip(hidden_states)
        if self.is_decoder:
            residual = ln if self.apply_residual_post_layernorm else hidden_states
            cross = self._branch(
                lambda residual, **kw: self.cross_attention(ln, residual=residual, **kw),
                residual, encoder_states=encoder_states, attention_mask=encoder_attention_mask,
                past_key_value=cross_past, use_cache=use_cache,
            )
            if use_cache:
                cross, cross_kv = cross
                presents = tuple(presents) + tuple(cross_kv)
            hidden_states = cross
            ln = self.post_cross_attention_layernorm(hidden_states)
            residual = ln if self.apply_residual_post_layernorm else hidden_states
        elif self.apply_residual_post_layernorm:
            residual = ln
        else:
            residual = post_skip
        output = self._branch(lambda residual: self.mlp(ln, residual=residual), residual)
        if use_cache:
            return output, presents
        return output

    def build_attention(self, is_cross_attention=False):
        return MultiheadAttention(
            self.hidden_size, self.num_attention_heads,
            is_cross_attention=is_cross_attention,
            attention_dropout_prob=self.attention_dropout_prob,
            output_dropout_prob=self.output_dropout_prob,
            init_method=self.init_method, output_layer_init_method=self.output_layer_init_method,
            bias_dropout_fusion=self.bias_dropout_fusion,
            scale_mask_softmax_fusion=self.scale_mask_softmax_fusion,
            apply_query_key_layer_scaling=self.apply_query_key_layer_scaling,
            attn_mask_type=self.attn_mask_type, layer_idx=self.layer_idx,
        )
