"""LLaMA-Adapter: zero-init gated attention over learnable adaption prompts in the last ``adapter_layer`` layers.

Spec: reference projects/Llama/adapter/adapter_model.py — ``adapter_query`` embedding of
``adapter_len · adapter_layer`` rows (:487-489, reshaped per layer :553), adapter keys/values from the frozen
``query_key_value`` projection (:219-228, no rotary), per-head ``gate`` with
``softmax(scores_adapter)·tanh(gate)`` concatenated to the ordinary softmax (:252-266).

H100 decomposition: ``softmax([A | S])`` is never formed — the sequence part stays on the flash-attention kernel
(``attention_qkvpacked``) and the adapter part (``adapter_len`` ≈ 10 keys) is a small dense attention added on
top: ``ctx = flash(q, k, v) + tanh(gate) · softmax(q·k_aᵀ) · v_a``.
"""
import torch
from torch import nn

from libai_b200.config import configurable
from libai_b200.inference.kv_cache import KVCacheLayer
from libai_b200.layers import Embedding
from libai_b200.layers._param import create_parameter, zeros_
from libai_b200.models.llama_model import LlamaAttention, LlamaForCausalLM as _BaseLlama
from libai_b200.models.utils.weight_init import init_method_normal
from libai_b200.ops import functional as OF


class AdapterAttention(LlamaAttention):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        layer_idx = kwargs.get("layer_idx", 0)
        self.gate = create_parameter((1, self.local_heads, 1, 1), zeros_, layer_idx=layer_idx)
        self.adapter = None  # [1, adapter_len, hidden]; set per forward by the model

    def forward(self, hidden_states, attention_mask=None, past_key_value=None, cos_cached=None, sin_cached=None,
                use_cache=False):
        out = super().forward(hidden_states, attention_mask, past_key_value, cos_cached, sin_cached, use_cache)
        if self.adapter is None:
            return out
        base, cache = (out if use_cache else (out, None))
        a, d = self.local_heads, self.head_size
        bsz = hidden_states.shape[0]
        # queries need the same rotary phase as in the main path
        qkv = self.query_key_value(hidden_states).view(bsz, -1, a, 3 * d)
        past_len, positions = 0, None
        if isinstance(past_key_value, KVCacheLayer):
            # the cache's rows before this step (the lengths advance after the last layer), read on the device: a
            # cached step holds no host-side position, so a CUDA graph of it replays at the current length
            s = hidden_states.shape[1]
            positions = past_key_value.seqlens[:, None] + torch.arange(s, dtype=torch.int32, device=qkv.device)
        elif past_key_value is not None:
            past_len = past_key_value[0].shape[2]
        q = OF.apply_rotary_qkv(qkv, cos_cached, sin_cached, past_len, positions)[..., :d].permute(0, 2, 1, 3)
        akv = self.query_key_value(self.adapter.to(hidden_states.dtype)).view(1, -1, a, 3 * d).permute(0, 2, 1, 3)
        ak, av = akv[..., d : 2 * d], akv[..., 2 * d :]
        scores = torch.matmul(q.float(), ak.float().transpose(-1, -2)) * self.norm_factor
        probs = torch.softmax(scores, dim=-1) * torch.tanh(self.gate.float())
        extra = torch.matmul(probs, av.float()).to(hidden_states.dtype).transpose(1, 2).reshape(bsz, -1, a * d)
        base = base + self.o_proj(extra)
        return (base, cache) if use_cache else base


class LlamaForCausalLM(_BaseLlama):
    # the adapter's query rotary takes its positions from a StaticKVCache's per-sample seqlens
    continuous_batching = False

    @configurable
    def __init__(self, *args, adapter_len=10, adapter_layer=30, cfg=None, **kwargs):
        super().__init__(*args, **kwargs)  # (without `cfg`: the base initialiser would re-enter from_config)
        self.cfg = cfg
        self.adapter_len, self.adapter_layer = adapter_len, min(adapter_layer, self.hidden_layers)
        hidden = self.model.embed_tokens.embedding_dim
        self.model.adapter_query = Embedding(self.adapter_len * self.adapter_layer, hidden,
                                             init_method=init_method_normal(0.02))
        # swap in the gated attention for the adapted layers (weights are shared with the originals)
        for layer in self.model.layers[-self.adapter_layer:]:
            old = layer.self_attn
            if old.num_kv_heads != old.num_heads:
                # the adapter keys / values are read from the per-head [q|k|v] view of query_key_value
                raise ValueError("LLaMA-Adapter needs num_key_value_heads == num_attention_heads")
            new = AdapterAttention(old.hidden_size, old.num_heads, None, layer_idx=layer.layer_idx)
            new.query_key_value, new.o_proj = old.query_key_value, old.o_proj
            layer.self_attn = new
        self.register_forward_pre_hook(self._bind_adapters)

    @classmethod
    def from_config(cls, cfg):
        out = _BaseLlama.from_config.__func__(cls, cfg)
        out["adapter_len"] = cfg.get("adapter_len", 10)
        out["adapter_layer"] = cfg.get("adapter_layer", 30)
        return out

    def _bind_adapters(self, module, args):
        prompts = self.model.adapter_query.weight.view(self.adapter_layer, 1, self.adapter_len, -1)
        for i, layer in enumerate(self.model.layers[-self.adapter_layer:]):
            layer.self_attn.adapter = prompts[i]

    def freeze_backbone(self):
        """Only the adaption prompts and the gates train (reference projects/Llama/adapter/train_net.py:41-53)."""
        for name, param in self.named_parameters():
            param.requires_grad = ("adapter_query" in name) or name.endswith(".gate")
        return self
