"""Swin Transformer (v1).

Spec: reference libai/models/swin_transformer.py — ``window_partition/reverse`` (:26-37),
``WindowAttention`` (:40-161; learned relative-position-bias table indexed by
``relative_position_index``, additive shifted-window mask), ``SwinTransformerBlock`` (:164-316; pre-norm,
cyclic shift), ``PatchMerging`` (:319-356; LN(4C) then 4C→2C), ``PatchEmbed`` (:359-407),
``BasicLayer`` (:410-492), ``SwinTransformer`` (:495-772).  Data parallel only, like the reference
(Model_Zoo.md:39-42).  Parameter names follow the reference / official checkpoints.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch import nn

from libai_b200.config import configurable
from libai_b200.layers import MLP, DropPath, LayerNorm, Linear
from libai_b200.layers._param import create_parameter, trunc_normal_, zeros_
from libai_b200.ops import functional as OF

from .utils.pipeline_model import PipelineStageMixin


def _tn(t, generator=None):
    return trunc_normal_(t, std=0.02, generator=generator)


def window_partition(x, window_size):
    """``[B, H, W, C]`` → ``[B·nW, ws, ws, C]``."""
    B, H, W, C = x.shape
    x = x.view(B, H // window_size, window_size, W // window_size, window_size, C)
    return x.permute(0, 1, 3, 2, 4, 5).contiguous().view(-1, window_size, window_size, C)


def window_reverse(windows, window_size, H, W):
    B = int(windows.shape[0] / (H * W / window_size / window_size))
    x = windows.view(B, H // window_size, W // window_size, window_size, window_size, -1)
    return x.permute(0, 1, 3, 2, 4, 5).contiguous().view(B, H, W, -1)


def relative_position_index(window_size):
    """``[ws², ws²]`` index into the ``(2ws-1)²`` bias table."""
    coords = torch.stack(torch.meshgrid(torch.arange(window_size[0]), torch.arange(window_size[1]), indexing="ij"))
    flat = torch.flatten(coords, 1)
    rel = (flat[:, :, None] - flat[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += window_size[0] - 1
    rel[:, :, 1] += window_size[1] - 1
    rel[:, :, 0] *= 2 * window_size[1] - 1
    return rel.sum(-1)


def shifted_window_mask(H, W, window_size, shift_size, device):
    """Additive mask ``[nW, ws², ws²]`` (0 / −100) separating the wrapped regions of a cyclic shift."""
    img = torch.zeros((1, H, W, 1), device=device)
    cnt = 0
    for h in (slice(0, -window_size), slice(-window_size, -shift_size), slice(-shift_size, None)):
        for w in (slice(0, -window_size), slice(-window_size, -shift_size), slice(-shift_size, None)):
            img[:, h, w, :] = cnt
            cnt += 1
    win = window_partition(img, window_size).view(-1, window_size * window_size)
    diff = win.unsqueeze(1) - win.unsqueeze(2)
    return diff.masked_fill(diff != 0, -100.0).masked_fill(diff == 0, 0.0)


class WindowAttention(nn.Module):
    def __init__(self, dim, window_size, num_heads, qkv_bias=True, qk_scale=None, attn_drop=0.0, proj_drop=0.0,
                 fused_bias_add_dropout=False, layer_idx=0):
        super().__init__()
        self.dim, self.window_size, self.num_heads = dim, window_size, num_heads
        head_dim = dim // num_heads
        self.scale = qk_scale or head_dim ** -0.5
        self.relative_position_bias_table = create_parameter(
            ((2 * window_size[0] - 1) * (2 * window_size[1] - 1), num_heads), _tn, layer_idx=layer_idx
        )
        self.register_buffer("relative_position_index", relative_position_index(window_size))
        self.qkv = Linear(dim, dim * 3, bias=qkv_bias, init_method=_tn, layer_idx=layer_idx)
        self.attn_drop = nn.Dropout(attn_drop)
        self.proj = Linear(dim, dim, init_method=_tn, layer_idx=layer_idx)
        self.proj_drop = nn.Dropout(proj_drop)
        self.fused_bias_add_dropout = fused_bias_add_dropout
        self.p = proj_drop

    def _bias(self, dtype):
        n = self.window_size[0] * self.window_size[1]
        idx = self.relative_position_index.view(-1).to(self.relative_position_bias_table.device)
        return self.relative_position_bias_table[idx].view(n, n, -1).permute(2, 0, 1).contiguous().unsqueeze(0).to(dtype)

    def forward(self, x, mask):
        B_, N, C = x.shape
        qkv = self.qkv(x).reshape(B_, N, 3, self.num_heads, C // self.num_heads).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0] * self.scale, qkv[1], qkv[2]
        attn = torch.matmul(q, k.transpose(-1, -2)) + self._bias(q.dtype)
        if mask is not None:
            nW = mask.shape[0]
            attn = attn.view(B_ // nW, nW, self.num_heads, N, N) + mask.to(attn.dtype).unsqueeze(1).unsqueeze(0)
            attn = attn.view(-1, self.num_heads, N, N)
        attn = self.attn_drop(torch.softmax(attn.float(), dim=-1).to(v.dtype))
        x = torch.matmul(attn, v).transpose(1, 2).reshape(B_, N, C)
        return self.proj_drop(self.proj(x))

    def forward_image(self, x, H, W, shift):
        """The whole shifted-window attention of the image-ordered tokens ``x`` ``[B, H·W, C]`` in one kernel (see
        :func:`OF.window_attention`): qkv and proj act per token, so they run on the image order and no roll, partition
        or reverse copy is made."""
        o = OF.window_attention(self.qkv(x), H=H, W=W, window=self.window_size[0], shift=shift, heads=self.num_heads,
                                scale=self.scale, table=self.relative_position_bias_table.float())
        return self.proj_drop(self.proj(o))


class SwinTransformerBlock(nn.Module):
    def __init__(self, dim, input_resolution, num_heads, window_size=7, shift_size=0, mlp_ratio=4.0, qkv_bias=True,
                 qk_scale=None, drop=0.0, attn_drop=0.0, drop_path=0.0, act_layer=nn.GELU, norm_layer=LayerNorm,
                 layer_idx=0):
        super().__init__()
        self.dim, self.input_resolution, self.num_heads = dim, input_resolution, num_heads
        self.window_size, self.shift_size, self.mlp_ratio, self.layer_idx = window_size, shift_size, mlp_ratio, layer_idx
        if min(input_resolution) <= window_size:  # window covers the whole map: no partition / shift
            self.shift_size = 0
            self.window_size = min(input_resolution)
        assert 0 <= self.shift_size < self.window_size, "shift_size must in 0-window_size"
        self.norm1 = norm_layer(dim, layer_idx=layer_idx)
        self.attn = WindowAttention(dim, window_size=(self.window_size, self.window_size), num_heads=num_heads,
                                    qkv_bias=qkv_bias, qk_scale=qk_scale, attn_drop=attn_drop, proj_drop=drop,
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

    def _windowed_attention(self, x):
        H, W = self.input_resolution
        B, L, C = x.shape
        assert L == H * W, "input feature has wrong size"
        if OF.window_attention_supported(x, H=H, W=W, window=self.window_size, shift=self.shift_size,
                                         head_dim=C // self.num_heads, attn_drop=self.attn.attn_drop.p,
                                         training=self.training):
            return self.attn.forward_image(x, H, W, self.shift_size)
        x = x.view(B, H, W, C)
        if self.shift_size > 0:
            x = torch.roll(x, shifts=(-self.shift_size, -self.shift_size), dims=(1, 2))
        win = window_partition(x, self.window_size).view(-1, self.window_size * self.window_size, C)
        win = self.attn(win, self._attn_mask(x.device)).view(-1, self.window_size, self.window_size, C)
        x = window_reverse(win, self.window_size, H, W)
        if self.shift_size > 0:
            x = torch.roll(x, shifts=(self.shift_size, self.shift_size), dims=(1, 2))
        return x.view(B, H * W, C)

    def forward(self, x):
        x = x + self.drop_path(self._windowed_attention(self.norm1(x)))
        return x + self.drop_path(self.mlp(self.norm2(x)))


class PatchMerging(nn.Module):
    """2×2 neighbourhood concat → LN(4C) → Linear(4C → 2C)."""

    def __init__(self, input_resolution, dim, norm_layer=LayerNorm, layer_idx=0):
        super().__init__()
        self.input_resolution, self.dim = input_resolution, dim
        self.reduction = Linear(4 * dim, 2 * dim, bias=False, init_method=_tn, layer_idx=layer_idx)
        self.norm = norm_layer(4 * dim, layer_idx=layer_idx)
        self.layer_idx = layer_idx

    def forward(self, x):
        H, W = self.input_resolution
        B, L, C = x.shape
        assert L == H * W and H % 2 == 0 and W % 2 == 0, f"x size ({H}*{W}) are not even."
        x = x.view(B, H, W, C)
        x = torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], -1)
        return self.reduction(self.norm(x.view(B, -1, 4 * C)))


class PatchEmbed(nn.Module):
    def __init__(self, img_size=224, patch_size=4, in_chans=3, embed_dim=96, norm_layer=None, layer_idx=0):
        super().__init__()
        img_size = (img_size, img_size) if isinstance(img_size, int) else tuple(img_size)
        patch_size = (patch_size, patch_size) if isinstance(patch_size, int) else tuple(patch_size)
        self.img_size, self.patch_size = img_size, patch_size
        self.patches_resolution = [img_size[0] // patch_size[0], img_size[1] // patch_size[1]]
        self.num_patches = self.patches_resolution[0] * self.patches_resolution[1]
        self.in_chans, self.embed_dim = in_chans, embed_dim
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)
        self.norm = norm_layer(embed_dim, layer_idx=layer_idx) if norm_layer is not None else None

    def forward(self, x):
        B, C, H, W = x.shape
        assert H == self.img_size[0] and W == self.img_size[1], (
            f"Input image size ({H}*{W}) doesn't match model ({self.img_size[0]}*{self.img_size[1]})."
        )
        x = self.proj(x.to(self.proj.weight.dtype)).flatten(2).transpose(1, 2)
        return self.norm(x) if self.norm is not None else x


class BasicLayer(nn.Module):
    def __init__(self, dim, input_resolution, depth, num_heads, window_size, mlp_ratio=4.0, qkv_bias=True, qk_scale=None,
                 drop=0.0, attn_drop=0.0, drop_path=0.0, norm_layer=LayerNorm, downsample=None, layer_id_offset=0):
        super().__init__()
        self.dim, self.input_resolution, self.depth, self.layer_id_offset = dim, input_resolution, depth, layer_id_offset
        self.blocks = nn.ModuleList(
            [
                SwinTransformerBlock(
                    dim=dim, input_resolution=input_resolution, num_heads=num_heads, window_size=window_size,
                    shift_size=0 if (i % 2 == 0) else window_size // 2, mlp_ratio=mlp_ratio, qkv_bias=qkv_bias,
                    qk_scale=qk_scale, drop=drop, attn_drop=attn_drop,
                    drop_path=drop_path[i] if isinstance(drop_path, list) else drop_path, norm_layer=norm_layer,
                    layer_idx=layer_id_offset + i,
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


class SwinTransformer(nn.Module):
    @configurable
    def __init__(self, img_size=224, patch_size=4, in_chans=3, num_classes=1000, embed_dim=96, depths=[2, 2, 6, 2],
                 num_heads=[3, 6, 12, 24], window_size=7, mlp_ratio=4.0, qkv_bias=True, qk_scale=None, drop_rate=0.0,
                 attn_drop_rate=0.0, drop_path_rate=0.1, norm_layer=LayerNorm, ape=False, patch_norm=True, loss_func=None,
                 **kwargs):
        super().__init__()
        depths, num_heads = list(depths), list(num_heads)
        self.num_classes, self.num_layers, self.embed_dim = num_classes, len(depths), embed_dim
        self.ape, self.patch_norm = ape, patch_norm
        self.num_features = int(embed_dim * 2 ** (self.num_layers - 1))
        self.mlp_ratio = mlp_ratio
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
                    qkv_bias=qkv_bias, qk_scale=qk_scale, drop=drop_rate, attn_drop=attn_drop_rate,
                    drop_path=dpr[sum(depths[:i]) : sum(depths[: i + 1])], norm_layer=norm_layer,
                    downsample=PatchMerging if (i < self.num_layers - 1) else None, layer_id_offset=offset,
                )
            )
            offset += depths[i]
        self.norm = norm_layer(self.num_features, layer_idx=-1)
        self.avgpool = nn.AdaptiveAvgPool1d(1)
        self.head = Linear(self.num_features, num_classes, init_method=_tn, layer_idx=-1) if num_classes > 0 else nn.Identity()
        self.loss_func = nn.CrossEntropyLoss() if loss_func is None else loss_func

    @classmethod
    def from_config(cls, cfg):
        keys = ("img_size patch_size in_chans num_classes embed_dim depths num_heads window_size mlp_ratio qkv_bias "
                "qk_scale drop_rate drop_path_rate ape patch_norm loss_func").split()
        return {k: cfg[k] for k in keys}

    def no_weight_decay(self):
        return {"absolute_pos_embed"}

    def no_weight_decay_keywords(self):
        return {"relative_position_bias_table"}

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
