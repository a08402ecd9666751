"""PaLM: parallel attention + feed-forward blocks, multi-query attention, rotary positions, SwiGLU.

Spec: reference projects/PaLM/palm_model.py — ``RotaryEmbedding`` / ``apply_rotary_pos_emb`` (:30-65),
``SwiGLU`` feed-forward of width ``2·mult·dim`` (:68-81), ``PalmTransformerLayer`` (:84-190: one shared LayerNorm
(no bias), queries per head but a *single* key/value head, ``out = x + attn(norm(x)) + ffwd(x)`` – note the
reference feeds the un-normalised ``x`` to the feed-forward, :189), ``PalmHead`` tied to the embedding with the LM
loss (:193-208), ``PaLM`` (:211-300).

H100 mapping: queries are column-parallel over heads; the single KV head is replicated (it is tiny:
``2·dim_head`` columns); attention runs through ``ops.attention`` (flash kernel when shapes allow: the KV head is
expanded as a zero-copy stride-0 view → falls back to the library path, the GEMMs stay native).
"""
from __future__ import annotations

import torch
from torch import nn

from libai_b200.config import configurable
from libai_b200.layers import LayerNorm, Linear, LMLogits, ParallelCrossEntropyLoss, VocabEmbedding
from libai_b200.models.utils.pipeline_model import PipelineStageMixin
from libai_b200.models.utils.weight_init import init_method_normal
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dutil


def rotary_positions(seq_len, dim, device):
    inv_freq = 1.0 / (10000 ** (torch.arange(0, dim, 2, device=device).float() / dim))
    freqs = torch.outer(torch.arange(seq_len, device=device).float(), inv_freq)
    return torch.cat((freqs, freqs), dim=-1)


def rotate_half(x):
    x1, x2 = x[..., : x.shape[-1] // 2], x[..., x.shape[-1] // 2 :]
    return torch.cat((-x2, x1), dim=-1)


def apply_rotary_pos_emb(pos, t):
    return (t.float() * pos.cos() + rotate_half(t.float()) * pos.sin()).to(t.dtype)


class RotaryEmbedding(nn.Module):
    """``rope(max_seq_len, device=…)`` → rotary angles ``[seq, dim]`` (reference projects/PaLM/palm_model.py)."""

    def __init__(self, dim, *, layer_idx=0):
        super().__init__()
        self.dim = dim

    def forward(self, max_seq_len, *, device=None):
        return rotary_positions(max_seq_len, self.dim, device)


class SwiGLU(nn.Module):
    """``silu(gate) * x`` on a tensor whose last dimension holds ``[x, gate]`` halves (the fused kernel when on GPU)."""

    def forward(self, x):
        x, gate = x.chunk(2, dim=-1)
        return OF.swiglu(gate.contiguous(), x.contiguous())


class FeedForward(nn.Module):
    def __init__(self, dim, mult=4, *, layer_idx=0, init_method=None):
        super().__init__()
        inner = int(dim * mult)
        self.wi_gate = Linear(dim, inner, bias=False, parallel="col", init_method=init_method, layer_idx=layer_idx)
        self.wi_up = Linear(dim, inner, bias=False, parallel="col", init_method=init_method, layer_idx=layer_idx)
        self.wo = Linear(inner, dim, bias=False, parallel="row", init_method=init_method, layer_idx=layer_idx)

    def forward(self, x):
        return self.wo(OF.swiglu(self.wi_gate(x), self.wi_up(x)))


class PalmTransformerLayer(nn.Module):
    def __init__(self, dim, dim_head=64, num_heads=8, ffn_mult=4, layernorm_epsilon=1e-5, *, layer_idx=0, init_method=None):
        super().__init__()
        topo = dutil.get_dist_util()
        self.num_heads, self.dim_head, self.layer_idx = num_heads, dim_head, layer_idx
        self.local_heads = num_heads // topo.tensor_parallel_size
        self.to_q = Linear(dim, dim_head * num_heads, bias=False, parallel="col", init_method=init_method, layer_idx=layer_idx)
        self.to_kv = Linear(dim, dim_head * 2, bias=False, parallel="data", init_method=init_method, layer_idx=layer_idx)
        self.to_out = Linear(dim_head * num_heads, dim, bias=False, parallel="row", init_method=init_method, layer_idx=layer_idx)
        self.ffwd = FeedForward(dim, ffn_mult, layer_idx=layer_idx, init_method=init_method)
        self.norm = LayerNorm(dim, eps=layernorm_epsilon, bias=False, layer_idx=layer_idx)
        self.scale = dim_head ** -0.5

    def forward(self, x):
        b, s, _ = x.shape
        ln = self.norm(x)
        q = self.to_q(ln).view(b, s, self.local_heads, self.dim_head).permute(0, 2, 1, 3)
        k, v = self.to_kv(ln).chunk(2, dim=-1)
        pos = rotary_positions(s, self.dim_head, x.device)
        q, k = apply_rotary_pos_emb(pos, q), apply_rotary_pos_emb(pos, k)
        k = k[:, None].expand(b, self.local_heads, s, self.dim_head)   # one shared key / value head
        v = v[:, None].expand(b, self.local_heads, s, self.dim_head)
        ctx = OF.attention(q, k, v, causal=True, scale=self.scale)
        attn_out = self.to_out(ctx.transpose(1, 2).reshape(b, s, -1))
        return self.ffwd(x) + attn_out + x


class PalmHead(nn.Module):
    def __init__(self, vocab_size):
        super().__init__()
        self.lm_head = LMLogits(vocab_size, bias=False)
        self.loss_func = ParallelCrossEntropyLoss()

    def forward(self, x, word_embedding_weight, lm_labels=None):
        logits = self.lm_head(x, word_embedding_weight)
        if lm_labels is not None:
            return {"lm_loss": self.loss_func(logits, lm_labels).mean()}
        return {"prediction_scores": logits}


class PaLM(nn.Module, PipelineStageMixin):
    @configurable
    def __init__(self, vocab_size, dim, depth, dim_head=64, num_heads=8, ffn_mult=4, initializer_range=0.02,
                 layernorm_eps=1e-12, amp_enabled=False):
        super().__init__()
        init_method = init_method_normal(initializer_range)
        self.word_embedding = VocabEmbedding(vocab_size, dim, init_method=init_method, amp_enabled=amp_enabled)
        self.net = nn.ModuleList([
            PalmTransformerLayer(dim, dim_head, num_heads, ffn_mult, layernorm_eps, layer_idx=i, init_method=init_method)
            for i in range(depth)])
        self.norm = LayerNorm(dim, eps=layernorm_eps, bias=False, layer_idx=-1)
        self.head = PalmHead(vocab_size)

    @classmethod
    def from_config(cls, cfg):
        return {k: cfg[k] for k in ("vocab_size dim depth dim_head num_heads ffn_mult initializer_range layernorm_eps "
                                    "amp_enabled").split()}

    # pipeline protocol
    def stage_pre(self, input_ids, **_):
        return self.word_embedding(input_ids)

    def stage_layers(self):
        return self.net

    def stage_post(self, hidden, labels=None, **_):
        return self.head(self.norm(hidden), self.word_embedding.weight, labels)

    def forward(self, input_ids, labels=None):
        return self.forward_stage({"input_ids": input_ids, "labels": labels})

    @staticmethod
    def set_activation_checkpoint(model):
        model.activation_checkpoint = True
        return model

    @staticmethod
    def set_pipeline_stage_id(model):
        return model
