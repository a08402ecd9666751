"""Swin Transformer V2.

Spec: reference libai/models/swin_transformer_v2.py — scaled-cosine window attention with a learned
per-head ``logit_scale`` (clamped at ln 100, :94-107/:241), continuous position bias from ``cpb_mlp``
over a log-spaced ``relative_coords_table`` (:110-160, 16·sigmoid, :245-262), separate ``q_bias``/``v_bias``
(k has no bias, :185-233), res-post-norm blocks (:431-435), ``PatchMerging`` = Linear(4C→2C) then
LN(2C) (:439-479), ``_init_respostnorm`` (:569-574).  Data parallel only.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from libai_b200.config import configurable
from libai_b200.layers import MLP, DropPath, LayerNorm, Linear
from libai_b200.layers._param import create_parameter, zeros_
from libai_b200.ops import functional as OF

from .swin_transformer import (
    PatchEmbed,
    _tn,
    relative_position_index,
    shifted_window_mask,
    window_partition,
    window_reverse,
)


def log_spaced_coords_table(window_size, pretrained_window_size):
    """``[1, 2Wh-1, 2Ww-1, 2]`` table: offsets normalised to ±8 then ``sign·log2(1+|x|)/log2(8)``."""
    h = torch.arange(-(window_size[0] - 1), window_size[0], dtype=torch.float32)
    w = torch.arange(-(window_size[1] - 1), window_size[1], dtype=torch.float32)
    table = torch.stack(torch.meshgrid(h, w, indexing="ij")).permute(1, 2, 0).contiguous().unsqueeze(0)
    denom = pretrained_window_size if pretrained_window_size[0] > 0 else window_size
    table[..., 0] /= max(denom[0] - 1, 1)
    table[..., 1] /= max(denom[1] - 1, 1)
    table *= 8
    return torch.sign(table) * torch.log2(torch.abs(table) + 1.0) / math.log2(8.0)


class WindowAttention(nn.Module):
    def __init__(self, dim, window_size, num_heads, qkv_bias=True, attn_drop=0.0, proj_drop=0.0,
                 pretrained_window_size=(0, 0), fused_bias_add_dropout=False, layer_idx=0):
        super().__init__()
        self.dim, self.window_size, self.num_heads = dim, tuple(window_size), num_heads
        self.pretrained_window_size = tuple(pretrained_window_size)
        self.layer_idx, self.p, self.fused_bias_add_dropout = layer_idx, proj_drop, fused_bias_add_dropout
        self.logit_scale = create_parameter(
            (1, num_heads, 1, 1), lambda t, generator=None: t.fill_(math.log(10.0)), layer_idx=layer_idx
        )
        self.cpb_mlp = nn.Sequential(
            Linear(2, 512, bias=True, layer_idx=layer_idx),
            nn.ReLU(inplace=True),
            Linear(512, num_heads, bias=False, layer_idx=layer_idx),
        )
        self.register_buffer("relative_coords_table",
                             log_spaced_coords_table(self.window_size, self.pretrained_window_size), persistent=False)
        self.register_buffer("relative_position_index", relative_position_index(self.window_size), persistent=False)
        self.qkv = Linear(dim, dim * 3, bias=False, init_method=_tn, layer_idx=layer_idx)
        if qkv_bias:
            self.q_bias = create_parameter((dim,), zeros_, layer_idx=layer_idx)
            self.v_bias = create_parameter((dim,), zeros_, layer_idx=layer_idx)
        else:
            self.q_bias = self.v_bias = None
        self.attn_drop = nn.Dropout(attn_drop)
        self.proj = Linear(dim, dim, init_method=_tn, layer_idx=layer_idx)
        self.proj_drop = nn.Dropout(proj_drop)

    def _bias(self, dtype):
        n = self.window_size[0] * self.window_size[1]
        table = self.cpb_mlp(self.relative_coords_table.to(self.qkv.weight.dtype)).view(-1, self.num_heads)
        bias = table[self.relative_position_index.view(-1)].view(n, n, -1).permute(2, 0, 1).contiguous()
        return (16.0 * torch.sigmoid(bias.float())).unsqueeze(0).to(dtype)

    def forward(self, x, mask=None):
        B_, N, C = x.shape
        qkv = self.qkv(x)
        if self.q_bias is not None:
            qkv = qkv + torch.cat([self.q_bias, torch.zeros_like(self.v_bias), self.v_bias]).to(qkv.dtype)
        qkv = qkv.reshape(B_, N, 3, self.num_heads, C // self.num_heads).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        attn = torch.matmul(F.normalize(q.float(), dim=-1), F.normalize(k.float(), dim=-1).transpose(-1, -2))
        attn = attn * torch.clamp(self.logit_scale.float(), max=math.log(1.0 / 0.01)).exp()
        attn = attn + self._bias(attn.dtype)
        if mask is not None:
            nW = mask.shape[0]
            attn = attn.view(B_ // nW, nW, self.num_heads, N, N) + mask.to(attn.dtype).unsqueeze(1).unsqueeze(0)
            attn = attn.view(-1, self.num_heads, N, N)
        attn = self.attn_drop(torch.softmax(attn, dim=-1).to(v.dtype))
        x = torch.matmul(attn, v).transpose(1, 2).reshape(B_, N, C)
        return self.proj_drop(self.proj(x))

    def forward_image(self, x, H, W, shift):
        """The whole shifted-window cosine attention of the image-ordered tokens ``x`` ``[B, H·W, C]`` in one kernel
        (see :func:`OF.window_attention`).  The fp32 table ``16·sigmoid(cpb_mlp(coords))`` and ``tau = exp(min(logit_scale,
        ln 100))`` are formed here, so autograd carries their gradients to ``cpb_mlp`` and ``logit_scale``."""
        qkv = self.qkv(x)
        if self.q_bias is not None:
            qkv = qkv + torch.cat([self.q_bias, torch.zeros_like(self.v_bias), self.v_bias]).to(qkv.dtype)
        table = self.cpb_mlp(self.relative_coords_table.to(self.qkv.weight.dtype)).view(-1, self.num_heads)
        table = 16.0 * torch.sigmoid(table.float())
        tau = torch.clamp(self.logit_scale.float(), max=math.log(1.0 / 0.01)).exp().view(-1)
        o = OF.window_attention(qkv, H=H, W=W, window=self.window_size[0], shift=shift, heads=self.num_heads, scale=1.0,
                                table=table, tau=tau)
        return self.proj_drop(self.proj(o))


class SwinTransformerBlock(nn.Module):
    def __init__(self, dim, input_resolution, num_heads, window_size=7, shift_size=0, mlp_ratio=4.0, qkv_bias=True,
                 drop=0.0, attn_drop=0.0, drop_path=0.0, act_layer=nn.GELU, norm_layer=LayerNorm,
                 pretrained_window_size=0, layer_idx=0):
        super().__init__()
        self.dim, self.input_resolution, self.num_heads = dim, input_resolution, num_heads
        self.window_size, self.shift_size, self.mlp_ratio, self.layer_idx = window_size, shift_size, mlp_ratio, layer_idx
        if min(input_resolution) <= window_size:
            self.shift_size = 0
            self.window_size = min(input_resolution)
        assert 0 <= self.shift_size < self.window_size, "shift_size must in 0-window_size"
        self.norm1 = norm_layer(dim, layer_idx=layer_idx)
        self.attn = WindowAttention(dim, window_size=(self.window_size, self.window_size), num_heads=num_heads,
                                    qkv_bias=qkv_bias, attn_drop=attn_drop, proj_drop=drop,
                                    pretrained_window_size=(pretrained_window_size, pretrained_window_size),
                                    fused_bias_add_dropout=True, layer_idx=layer_idx)
        self.drop_path = DropPath(drop_path) if drop_path > 0.0 else nn.Identity()
        self.norm2 = norm_layer(dim, layer_idx=layer_idx)
        self.mlp = MLP(hidden_size=dim, ffn_hidden_size=int(dim * mlp_ratio), output_dropout_prob=drop,
                       bias_gelu_fusion=True, bias_dropout_fusion=True, init_method=_tn, layer_idx=layer_idx)
        self._mask_cache = {}

    def _attn_mask(self, device):
        if self.shift_size == 0:
            return None
        key = str(device)
        if key not in self._mask_cache:
            H, W = self.input_resolution
            self._mask_cache[key] = shifted_window_mask(H, W, self.window_size, self.shift_size, device)
        return self._mask_cache[key]

    def forward(self, x):
        H, W = self.input_resolution
        B, L, C = x.shape
        assert L == H * W, "input feature has wrong size"
        shortcut = x
        if OF.window_attention_supported(x, H=H, W=W, window=self.window_size, shift=self.shift_size,
                                         head_dim=C // self.num_heads, attn_drop=self.attn.attn_drop.p,
                                         training=self.training):
            x = self.attn.forward_image(x, H, W, self.shift_size)
        else:
            x = x.view(B, H, W, C)
            if self.shift_size > 0:
                x = torch.roll(x, shifts=(-self.shift_size, -self.shift_size), dims=(1, 2))
            win = window_partition(x, self.window_size).view(-1, self.window_size * self.window_size, C)
            win = self.attn(win, mask=self._attn_mask(x.device)).view(-1, self.window_size, self.window_size, C)
            x = window_reverse(win, self.window_size, H, W)
            if self.shift_size > 0:
                x = torch.roll(x, shifts=(self.shift_size, self.shift_size), dims=(1, 2))
        x = shortcut + self.drop_path(self.norm1(x.view(B, H * W, C)))  # res-post-norm
        return x + self.drop_path(self.norm2(self.mlp(x)))


class PatchMerging(nn.Module):
    """2×2 concat → Linear(4C → 2C) → LN(2C)."""

    def __init__(self, input_resolution, dim, norm_layer=LayerNorm, layer_idx=0):
        super().__init__()
        self.input_resolution, self.dim, self.layer_idx = input_resolution, dim, layer_idx
        self.reduction = Linear(4 * dim, 2 * dim, bias=False, init_method=_tn, layer_idx=layer_idx)
        self.norm = norm_layer(2 * dim, layer_idx=layer_idx)

    def forward(self, x):
        H, W = self.input_resolution
        B, L, C = x.shape
        assert L == H * W and H % 2 == 0 and W % 2 == 0, f"x size ({H}*{W}) are not even."
        x = x.view(B, H, W, C)
        x = torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], -1)
        return self.norm(self.reduction(x.view(B, -1, 4 * C)))


class BasicLayer(nn.Module):
    def __init__(self, dim, input_resolution, depth, num_heads, window_size, mlp_ratio=4.0, qkv_bias=True, drop=0.0,
                 attn_drop=0.0, drop_path=0.0, norm_layer=LayerNorm, downsample=None, pretrained_window_size=0,
                 layer_id_offset=0):
        super().__init__()
        self.dim, self.input_resolution, self.depth, self.layer_id_offset = dim, input_resolution, depth, layer_id_offset
        self.blocks = nn.ModuleList(
            [
                SwinTransformerBlock(
                    dim=dim, input_resolution=input_resolution, num_heads=num_heads, window_size=window_size,
                    shift_size=0 if (i % 2 == 0) else window_size // 2, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias,
                    drop=drop, attn_drop=attn_drop,
                    drop_path=drop_path[i] if isinstance(drop_path, list) else drop_path, norm_layer=norm_layer,
                    pretrained_window_size=pretrained_window_size, layer_idx=layer_id_offset + i,
                )
                for i in range(depth)
            ]
        )
        self.downsample = (
            downsample(input_resolution, dim=dim, norm_layer=norm_layer, layer_idx=layer_id_offset + depth - 1)
            if downsample is not None else None
        )

    def forward(self, x):
        for blk in self.blocks:
            x = blk(x)
        return self.downsample(x) if self.downsample is not None else x

    def _init_respostnorm(self):
        with torch.no_grad():
            for blk in self.blocks:
                for norm in (blk.norm1, blk.norm2):
                    if not norm.weight.is_meta:
                        norm.bias.zero_()
                        norm.weight.zero_()


class SwinTransformerV2(nn.Module):
    @configurable
    def __init__(self, img_size=224, patch_size=4, in_chans=3, num_classes=1000, embed_dim=96, depths=[2, 2, 6, 2],
                 num_heads=[3, 6, 12, 24], window_size=7, mlp_ratio=4.0, qkv_bias=True, drop_rate=0.0,
                 attn_drop_rate=0.0, drop_path_rate=0.1, norm_layer=LayerNorm, ape=False, patch_norm=True,
                 pretrained_window_sizes=[0, 0, 0, 0], loss_func=None):
        super().__init__()
        depths, num_heads = list(depths), list(num_heads)
        self.num_classes, self.num_layers, self.embed_dim = num_classes, len(depths), embed_dim
        self.ape, self.patch_norm, self.mlp_ratio = ape, patch_norm, mlp_ratio
        self.num_features = int(embed_dim * 2 ** (self.num_layers - 1))
        self.patch_embed = PatchEmbed(img_size=img_size, patch_size=patch_size, in_chans=in_chans, embed_dim=embed_dim,
                                      norm_layer=norm_layer if patch_norm else None, layer_idx=0)
        res = self.patch_embed.patches_resolution
        self.patches_resolution = res
        if self.ape:
            self.absolute_pos_embed = create_parameter((1, self.patch_embed.num_patches, embed_dim), _tn, layer_idx=0)
        self.pos_drop = nn.Dropout(p=drop_rate)
        dpr = [x.item() for x in torch.linspace(0, drop_path_rate, sum(depths))]
        self.layers = nn.ModuleList()
        offset = 0
        for i in range(self.num_layers):
            self.layers.append(
                BasicLayer(
                    dim=int(embed_dim * 2 ** i), input_resolution=(res[0] // (2 ** i), res[1] // (2 ** i)),
                    depth=depths[i], num_heads=num_heads[i], window_size=window_size, mlp_ratio=mlp_ratio,
                    qkv_bias=qkv_bias, drop=drop_rate, attn_drop=attn_drop_rate,
                    drop_path=dpr[sum(depths[:i]) : sum(depths[: i + 1])], norm_layer=norm_layer,
                    downsample=PatchMerging if (i < self.num_layers - 1) else None,
                    pretrained_window_size=list(pretrained_window_sizes)[i], layer_id_offset=offset,
                )
            )
            offset += depths[i]
        self.norm = norm_layer(self.num_features, layer_idx=-1)
        self.avgpool = nn.AdaptiveAvgPool1d(1)
        self.head = Linear(self.num_features, num_classes, init_method=_tn, layer_idx=-1) if num_classes > 0 else nn.Identity()
        self.loss_func = nn.CrossEntropyLoss() if loss_func is None else loss_func
        for layer in self.layers:
            layer._init_respostnorm()

    @classmethod
    def from_config(cls, cfg):
        keys = ("img_size patch_size in_chans num_classes embed_dim depths num_heads window_size mlp_ratio qkv_bias "
                "drop_rate drop_path_rate ape patch_norm pretrained_window_sizes loss_func").split()
        return {k: cfg[k] for k in keys}

    def no_weight_decay(self):
        return {"absolute_pos_embed"}

    def no_weight_decay_keywords(self):
        return {"cpb_mlp", "logit_scale", "relative_position_bias_table"}

    def forward_features(self, x):
        x = self.patch_embed(x)
        if self.ape:
            x = x + self.absolute_pos_embed.to(x.dtype)
        x = self.pos_drop(x)
        for layer in self.layers:
            x = layer(x)
        x = self.norm(x)
        return torch.flatten(self.avgpool(x.transpose(1, 2)), 1)

    def forward(self, images, labels=None):
        x = self.head(self.forward_features(images))
        if labels is not None and self.training:
            return {"losses": self.loss_func(x.float(), labels)}
        return {"prediction_scores": x}

    @staticmethod
    def set_pipeline_stage_id(model):
        return model

    @staticmethod
    def set_activation_checkpoint(model):
        return model
