"""Embedding layers.

Spec: reference libai/layers/embedding.py — ``Embedding`` (replicated table, :26-101),
``VocabEmbedding`` (table split over the vocabulary dimension, masked gather + TP reduction,
:104-183), ``SinePositionalEmbedding`` (:186-234), ``PatchEmbedding`` (Conv2d stem, :237-290).
``padding_idx`` rows are zero-initialised.
"""
from __future__ import annotations

import math

import torch
from torch import nn

from libai_b200.ops import functional as OF
from libai_b200.parallel import mappings
from libai_b200.utils import distributed as dutil

from ._param import create_parameter, param_device, xavier_normal_, zeros_

_SP_SHAPE = {"b": None, "s": None}


def set_sp_shape(b: int, s: int) -> None:
    """Record the (micro-batch, sequence) shape of the activations that are flattened and token
    sharded under sequence parallelism (attention needs it back)."""
    _SP_SHAPE["b"], _SP_SHAPE["s"] = int(b), int(s)


def get_sp_shape():
    return _SP_SHAPE["b"], _SP_SHAPE["s"]


class Embedding(nn.Module):
    """Replicated lookup table ``[num_embeddings, embedding_dim]``."""

    def __init__(self, num_embeddings, embedding_dim, padding_idx=None, init_method=None, amp_enabled=False,
                 dtype=None, *, layer_idx=0):
        super().__init__()
        self.num_embeddings, self.embedding_dim = num_embeddings, embedding_dim
        if padding_idx is not None:
            if padding_idx > 0:
                assert padding_idx < num_embeddings, "Padding_idx must be within num_embeddings"
            elif padding_idx < 0:
                assert padding_idx >= -num_embeddings, "Padding_idx must be within num_embeddings"
                padding_idx = num_embeddings + padding_idx
        self.padding_idx = padding_idx
        self.init_method = init_method or nn.init.normal_
        self.amp_enabled = amp_enabled
        self.weight = create_parameter((num_embeddings, embedding_dim), self.init_method, layer_idx=layer_idx, dtype=dtype)
        self._fill_padding_idx_with_zero()

    def forward(self, input_ids):
        return OF.embedding(input_ids, self.weight) if input_ids.is_cuda else torch.nn.functional.embedding(input_ids, self.weight)

    def _fill_padding_idx_with_zero(self) -> None:
        if self.padding_idx is not None and self.weight.device.type != "meta":
            with torch.no_grad():
                self.weight[self.padding_idx].zero_()

    def extra_repr(self) -> str:
        s = "num_embeddings={num_embeddings}, embedding_dim={embedding_dim}"
        if self.padding_idx is not None:
            s += ", padding_idx={padding_idx}"
        return s.format(**self.__dict__)


class VocabEmbedding(nn.Module):
    """Table split over the vocabulary across the TP group.

    fwd: gather rows of the local ``[V/t, h]`` shard (zeros for ids owned by other ranks) then
    sum over TP — all-reduce, or reduce-scatter to token shards under sequence parallelism.
    """

    def __init__(self, num_embeddings, embedding_dim, padding_idx=None, init_method=None, amp_enabled=False,
                 dtype=None, *, layer_idx=0):
        super().__init__()
        self.num_embeddings, self.embedding_dim = num_embeddings, embedding_dim
        if padding_idx is not None:
            if padding_idx > 0:
                assert padding_idx < num_embeddings, "Padding_idx must be within num_embeddings"
            elif padding_idx < 0:
                assert padding_idx >= -num_embeddings, "Padding_idx must be within num_embeddings"
                padding_idx = num_embeddings + padding_idx
        self.padding_idx = padding_idx
        self.init_method = init_method or nn.init.normal_
        self.amp_enabled = amp_enabled
        topo = dutil.get_dist_util()
        self.weight = create_parameter(
            (num_embeddings, embedding_dim), self.init_method, tp_dim=0, layer_idx=layer_idx, dtype=dtype
        )
        self.vocab_per_rank = num_embeddings // topo.tensor_parallel_size
        self.vocab_start = topo.tp_rank * self.vocab_per_rank
        if self.padding_idx is not None and self.weight.device.type != "meta":
            local = self.padding_idx - self.vocab_start
            if 0 <= local < self.vocab_per_rank:
                with torch.no_grad():
                    self.weight[local].zero_()

    def forward(self, input_ids, scatter_to_sequence_parallel: bool = False):
        topo = dutil.get_dist_util()
        if topo.tensor_parallel_size == 1:
            return OF.embedding(input_ids, self.weight) if input_ids.is_cuda else torch.nn.functional.embedding(input_ids, self.weight)
        out = OF.embedding(input_ids, self.weight, self.vocab_start)   # zero rows for ids of other vocabulary shards
        if scatter_to_sequence_parallel and topo.sequence_parallel:
            return mappings.reduce_scatter_to_sp(out.reshape(-1, out.shape[-1]))
        return mappings.reduce_from_tp(out)

    def extra_repr(self) -> str:
        s = "num_embeddings={num_embeddings}, embedding_dim={embedding_dim}"
        if self.padding_idx is not None:
            s += ", padding_idx={padding_idx}"
        return s.format(**self.__dict__)


class SinePositionalEmbedding(nn.Module):
    """Fixed sinusoidal table (even dims sin, odd dims cos)."""

    def __init__(self, num_embeddings, embedding_dim, *, layer_idx=0):
        super().__init__()
        self.embedding_dim, self.num_embeddings = embedding_dim, num_embeddings
        pos = torch.arange(num_embeddings, dtype=torch.float32).unsqueeze(1)
        div = torch.exp(torch.arange(0, embedding_dim, 2).float() * (-math.log(10000.0) / embedding_dim)).unsqueeze(0)
        table = torch.zeros(num_embeddings, embedding_dim)
        table[:, 0::2] = torch.sin(pos * div)
        table[:, 1::2] = torch.cos(pos * div)[:, : embedding_dim // 2]
        owned = dutil.get_dist_util().owns_layer(layer_idx)
        self.register_buffer("position_embedding", table.to(param_device()) if owned else table.to("meta"), persistent=False)

    def forward(self, position_ids):
        return (OF.embedding(position_ids, self.position_embedding) if position_ids.is_cuda
                else torch.nn.functional.embedding(position_ids, self.position_embedding))

    def extra_repr(self) -> str:
        return f"num_embeddings={self.num_embeddings}, embedding_dim={self.embedding_dim}"


class PatchEmbedding(nn.Module):
    """2-D image → patch tokens: a stride-``patch`` convolution == patchify + GEMM.

    Implemented as unfold-free reshape + the wgmma GEMM (``[b·n_patches, c·p·p] × [c·p·p, h]``)
    instead of cuDNN; the parameter keeps the Conv2d layout ``[embed_dim, in_chans, p, p]`` so HF
    / reference checkpoints load unchanged."""

    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=768, norm_layer=None, flatten=True,
                 *, layer_idx=0):
        super().__init__()
        img_size = img_size if isinstance(img_size, tuple) else (img_size, img_size)
        patch_size = patch_size if isinstance(patch_size, tuple) else (patch_size, patch_size)
        self.img_size, self.patch_size = img_size, patch_size
        self.grid_size = (img_size[0] // patch_size[0], img_size[1] // patch_size[1])
        self.num_patches = self.grid_size[0] * self.grid_size[1]
        self.flatten = flatten
        self.in_chans, self.embed_dim = in_chans, embed_dim

        class _Proj(nn.Module):
            pass

        self.proj = _Proj()
        fan_in = in_chans * patch_size[0] * patch_size[1]
        bound = 1.0 / math.sqrt(fan_in)

        def conv_init(t, generator=None):
            return t.uniform_(-bound, bound, generator=generator)

        self.proj.weight = create_parameter((embed_dim, in_chans, patch_size[0], patch_size[1]), conv_init, layer_idx=layer_idx)
        self.proj.bias = create_parameter((embed_dim,), conv_init, layer_idx=layer_idx)
        self.norm = norm_layer(embed_dim) if norm_layer else nn.Identity()

    def forward(self, x):
        B, C, H, W = x.shape
        assert H == self.img_size[0], f"Input image height ({H}) doesn't match model ({self.img_size[0]})."
        assert W == self.img_size[1], f"Input image width ({W}) doesn't match model ({self.img_size[1]})."
        ph, pw = self.patch_size
        gh, gw = self.grid_size
        patches = x.reshape(B, C, gh, ph, gw, pw).permute(0, 2, 4, 1, 3, 5).reshape(B * gh * gw, C * ph * pw)
        w = self.proj.weight.reshape(self.embed_dim, -1)
        y = OF.linear(patches.to(w.dtype), w, self.proj.bias).view(B, gh * gw, self.embed_dim)
        if not self.flatten:
            y = y.transpose(1, 2).reshape(B, self.embed_dim, gh, gw)
        return self.norm(y)
