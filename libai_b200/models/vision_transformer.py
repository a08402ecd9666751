"""Vision Transformer.

Spec: reference libai/models/vision_transformer.py:25-267 — ``PatchEmbedding`` stem, learned
``cls_token`` / ``pos_embed`` (trunc-normal 0.02, no weight decay), ``depth`` pre-LN
``TransformerLayer`` blocks with linearly increasing DropPath, final LN, linear head on the class
token; ``{"losses"}`` when training with labels, else ``{"prediction_scores"}``.
The patch stem runs as patchify + wgmma GEMM (``layers/embedding.py``).
"""
from __future__ import annotations

import torch
from torch import nn

from libai_b200.config import configurable
from libai_b200.layers import LayerNorm, Linear, PatchEmbedding, TransformerLayer
from libai_b200.layers._param import create_parameter, trunc_normal_, zeros_
from libai_b200.utils import distributed as dutil

from .utils.pipeline_model import PipelineStageMixin


def _tn(std):
    def init_(t, generator=None):
        return trunc_normal_(t, std=std, a=-2.0, b=2.0, generator=generator)

    return init_


class VisionTransformer(nn.Module, PipelineStageMixin):
    @configurable
    def __init__(self, img_size=224, patch_size=16, in_chans=3, embed_dim=192, depth=12, num_heads=3, mlp_ratio=4.0,
                 drop_rate=0.0, attn_drop_rate=0.0, drop_path_rate=0.0, num_classes=1000, loss_func=None):
        super().__init__()
        self.img_size, self.num_classes = img_size, num_classes
        self.patch_embed = PatchEmbedding(img_size=img_size, patch_size=patch_size, in_chans=in_chans, embed_dim=embed_dim)
        ffn_size = int(embed_dim * mlp_ratio)
        num_patches = self.patch_embed.num_patches
        self.cls_token = create_parameter((1, 1, embed_dim), _tn(0.02), layer_idx=0)
        self.pos_embed = create_parameter((1, num_patches + 1, embed_dim), _tn(0.02), layer_idx=0)
        self.pos_drop = nn.Dropout(p=drop_rate)
        dpr = [x.item() for x in torch.linspace(0, drop_path_rate, depth)]  # stochastic depth decay rule
        self.blocks = nn.Sequential(
            *[
                TransformerLayer(
                    hidden_size=embed_dim, ffn_hidden_size=ffn_size, num_attention_heads=num_heads,
                    attention_dropout_prob=attn_drop_rate, output_dropout_prob=drop_rate, drop_path_prob=dpr[i],
                    init_method=_tn(0.02), layer_idx=i,
                )
                for i in range(depth)
            ]
        )
        self.norm = LayerNorm(embed_dim, layer_idx=-1)
        self.head = Linear(embed_dim, num_classes, init_method=_tn(0.02), layer_idx=-1)
        self.loss_func = nn.CrossEntropyLoss() if loss_func is None else loss_func

    def no_weight_decay(self):
        return {"pos_embed", "cls_token"}

    @classmethod
    def from_config(cls, cfg):
        keys = "img_size patch_size in_chans embed_dim depth num_heads mlp_ratio drop_rate attn_drop_rate drop_path_rate num_classes loss_func".split()
        return {k: cfg[k] for k in keys}

    # ---- pipeline protocol ------------------------------------------------------------------------------
    def stage_pre(self, images, **_):
        x = self.patch_embed(images)
        cls = self.cls_token.to(x.dtype).expand(x.shape[0], -1, -1)
        x = torch.cat((cls, x), dim=1)
        return self.pos_drop(x + self.pos_embed.to(x.dtype))

    def stage_layers(self):
        return self.blocks

    def stage_post(self, hidden, labels=None, **_):
        x = self.forward_head(hidden)
        if labels is not None and self.training:
            return {"losses": self.loss_func(x.float(), labels)}
        return {"prediction_scores": x}

    def forward_features(self, x):
        x = self.stage_pre(x)
        for blk in self.blocks:
            x = blk(x)
        return x

    def forward_head(self, x):
        x = self.norm(x)
        return self.head(x[:, 0])

    def forward(self, images, labels=None):
        return self.forward_stage({"images": images, "labels": labels})

    @staticmethod
    def set_pipeline_stage_id(model):
        return model

    @staticmethod
    def set_activation_checkpoint(model):
        model.activation_checkpoint = True
        return model
