"""CLIP (ViT and ModifiedResNet image towers + causal text transformer), OpenAI state-dict compatible.

Spec: reference projects/CLIP/clip/model.py — ``Bottleneck`` / ``AttentionPool2d`` / ``ModifiedResNet``,
``LayerNorm`` (fp32 compute), ``QuickGELU``, ``ResidualAttentionBlock``, ``Transformer``, ``VisionTransformer``,
``CLIP`` (``encode_image``, ``encode_text`` taking the features at the EOT token, cosine logits scaled by
``exp(logit_scale)``), ``convert_weights``, ``build_model`` (infers the architecture from a state dict).
Attention runs through ``libai_b200.ops.attention`` (flash kernel for mask-free / causal shapes on H100).
"""
from collections import OrderedDict
from typing import Tuple, Union

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from libai_b200.ops import functional as OF


class LayerNorm(nn.LayerNorm):
    def forward(self, x):
        return OF.layer_norm(x, self.weight, self.bias, self.eps)


class QuickGELU(nn.Module):
    def forward(self, x):
        return x * torch.sigmoid(1.702 * x)


class MultiheadAttention(nn.Module):
    """``nn.MultiheadAttention`` parameter layout (``in_proj_weight`` = [q; k; v]) on the native attention op."""

    def __init__(self, embed_dim, num_heads):
        super().__init__()
        self.embed_dim, self.num_heads = embed_dim, num_heads
        self.in_proj_weight = nn.Parameter(torch.empty(3 * embed_dim, embed_dim))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * embed_dim))
        self.out_proj = nn.Linear(embed_dim, embed_dim)
        nn.init.xavier_uniform_(self.in_proj_weight)

    def forward(self, x, causal=False):  # x: [L, N, E]
        L, N, E = x.shape
        qkv = OF.linear(x, self.in_proj_weight, self.in_proj_bias).view(L, N, 3, self.num_heads, E // self.num_heads)
        q, k, v = (qkv[:, :, i].permute(1, 2, 0, 3) for i in range(3))  # [N, H, L, d]
        ctx = OF.attention(q, k, v, causal=causal)
        return self.out_proj(ctx.permute(2, 0, 1, 3).reshape(L, N, E))


class ResidualAttentionBlock(nn.Module):
    def __init__(self, d_model: int, n_head: int, causal: bool = False):
        super().__init__()
        self.attn = MultiheadAttention(d_model, n_head)
        self.ln_1 = LayerNorm(d_model)
        self.mlp = nn.Sequential(OrderedDict([("c_fc", nn.Linear(d_model, d_model * 4)), ("gelu", QuickGELU()),
                                              ("c_proj", nn.Linear(d_model * 4, d_model))]))
        self.ln_2 = LayerNorm(d_model)
        self.causal = causal

    def forward(self, x):
        x = x + self.attn(self.ln_1(x), causal=self.causal)
        return x + self.mlp(self.ln_2(x))


class MLPClip(nn.Sequential):
    """CLIP's feed-forward ``c_fc → QuickGELU → c_proj`` as a named module (reference projects/CLIP/clip/model.py:188:
    the library MLP with the activation swapped for QuickGELU); same parameter names as the block's ``mlp``."""

    def __init__(self, hidden_size, ffn_hidden_size, **_unused):
        super().__init__(OrderedDict([("c_fc", nn.Linear(hidden_size, ffn_hidden_size)), ("gelu", QuickGELU()),
                                      ("c_proj", nn.Linear(ffn_hidden_size, hidden_size))]))


TransformerLayerClip = ResidualAttentionBlock     # the reference's name for the same pre-LN block


class Transformer(nn.Module):
    def __init__(self, width: int, layers: int, heads: int, causal: bool = False):
        super().__init__()
        self.width, self.layers = width, layers
        self.resblocks = nn.Sequential(*[ResidualAttentionBlock(width, heads, causal) for _ in range(layers)])

    def forward(self, x):
        return self.resblocks(x)


class VisionTransformer(nn.Module):
    def __init__(self, input_resolution: int, patch_size: int, width: int, layers: int, heads: int, output_dim: int):
        super().__init__()
        self.input_resolution, self.output_dim = input_resolution, output_dim
        self.conv1 = nn.Conv2d(3, width, kernel_size=patch_size, stride=patch_size, bias=False)
        scale = width ** -0.5
        self.class_embedding = nn.Parameter(scale * torch.randn(width))
        self.positional_embedding = nn.Parameter(scale * torch.randn((input_resolution // patch_size) ** 2 + 1, width))
        self.ln_pre = LayerNorm(width)
        self.transformer = Transformer(width, layers, heads)
        self.ln_post = LayerNorm(width)
        self.proj = nn.Parameter(scale * torch.randn(width, output_dim))

    def forward(self, x):
        x = self.conv1(x)
        x = x.reshape(x.shape[0], x.shape[1], -1).permute(0, 2, 1)
        cls = self.class_embedding.to(x.dtype) + torch.zeros(x.shape[0], 1, x.shape[-1], dtype=x.dtype, device=x.device)
        x = torch.cat([cls, x], dim=1) + self.positional_embedding.to(x.dtype)
        x = self.ln_pre(x).permute(1, 0, 2)
        x = self.transformer(x).permute(1, 0, 2)
        x = self.ln_post(x[:, 0, :])
        return x @ self.proj if self.proj is not None else x


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1):
        super().__init__()
        self.conv1, self.bn1 = nn.Conv2d(inplanes, planes, 1, bias=False), nn.BatchNorm2d(planes)
        self.conv2, self.bn2 = nn.Conv2d(planes, planes, 3, padding=1, bias=False), nn.BatchNorm2d(planes)
        self.avgpool = nn.AvgPool2d(stride) if stride > 1 else nn.Identity()
        self.conv3, self.bn3 = nn.Conv2d(planes, planes * 4, 1, bias=False), nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = None
        if stride > 1 or inplanes != planes * 4:
            self.downsample = nn.Sequential(OrderedDict([("-1", nn.AvgPool2d(stride)),
                                                         ("0", nn.Conv2d(inplanes, planes * 4, 1, stride=1, bias=False)),
                                                         ("1", nn.BatchNorm2d(planes * 4))]))

    def forward(self, x):
        out = self.relu(self.bn1(self.conv1(x)))
        out = self.avgpool(self.relu(self.bn2(self.conv2(out))))
        out = self.bn3(self.conv3(out))
        return self.relu(out + (x if self.downsample is None else self.downsample(x)))


class AttentionPool2d(nn.Module):
    def __init__(self, spacial_dim: int, embed_dim: int, num_heads: int, output_dim: int = None):
        super().__init__()
        self.positional_embedding = nn.Parameter(torch.randn(spacial_dim ** 2 + 1, embed_dim) / embed_dim ** 0.5)
        self.k_proj, self.q_proj, self.v_proj = (nn.Linear(embed_dim, embed_dim) for _ in range(3))
        self.c_proj = nn.Linear(embed_dim, output_dim or embed_dim)
        self.num_heads = num_heads

    def forward(self, x):
        x = x.reshape(x.shape[0], x.shape[1], -1).permute(2, 0, 1)  # NCHW -> (HW)NC
        x = torch.cat([x.mean(dim=0, keepdim=True), x], dim=0) + self.positional_embedding[:, None, :].to(x.dtype)
        L, N, E = x.shape
        h = self.num_heads
        q = self.q_proj(x[:1]).view(1, N, h, E // h).permute(1, 2, 0, 3)
        k = self.k_proj(x).view(L, N, h, E // h).permute(1, 2, 0, 3)
        v = self.v_proj(x).view(L, N, h, E // h).permute(1, 2, 0, 3)
        ctx = OF.attention(q, k, v, causal=False).permute(2, 0, 1, 3).reshape(1, N, E)
        return self.c_proj(ctx)[0]


class ModifiedResNet(nn.Module):
    """ResNet with a 3-conv stem, anti-aliased strided convs (avg-pool before stride) and attention pooling."""

    def __init__(self, layers, output_dim, heads, input_resolution=224, width=64):
        super().__init__()
        self.output_dim, self.input_resolution = output_dim, input_resolution
        self.conv1, self.bn1 = nn.Conv2d(3, width // 2, 3, stride=2, padding=1, bias=False), nn.BatchNorm2d(width // 2)
        self.conv2, self.bn2 = nn.Conv2d(width // 2, width // 2, 3, padding=1, bias=False), nn.BatchNorm2d(width // 2)
        self.conv3, self.bn3 = nn.Conv2d(width // 2, width, 3, padding=1, bias=False), nn.BatchNorm2d(width)
        self.avgpool, self.relu = nn.AvgPool2d(2), nn.ReLU(inplace=True)
        self._inplanes = width
        self.layer1 = self._make_layer(width, layers[0])
        self.layer2 = self._make_layer(width * 2, layers[1], stride=2)
        self.layer3 = self._make_layer(width * 4, layers[2], stride=2)
        self.layer4 = self._make_layer(width * 8, layers[3], stride=2)
        self.attnpool = AttentionPool2d(input_resolution // 32, width * 32, heads, output_dim)

    def _make_layer(self, planes, blocks, stride=1):
        layers = [Bottleneck(self._inplanes, planes, stride)]
        self._inplanes = planes * Bottleneck.expansion
        layers += [Bottleneck(self._inplanes, planes) for _ in range(1, blocks)]
        return nn.Sequential(*layers)

    def forward(self, x):
        x = x.type(self.conv1.weight.dtype)
        for conv, bn in ((self.conv1, self.bn1), (self.conv2, self.bn2), (self.conv3, self.bn3)):
            x = self.relu(bn(conv(x)))
        x = self.avgpool(x)
        return self.attnpool(self.layer4(self.layer3(self.layer2(self.layer1(x)))))


class CLIP(nn.Module):
    def __init__(self, embed_dim: int, image_resolution: int, vision_layers: Union[Tuple[int, int, int, int], int],
                 vision_width: int, vision_patch_size: int, context_length: int, vocab_size: int, transformer_width: int,
                 transformer_heads: int, transformer_layers: int):
        super().__init__()
        self.context_length = context_length
        if isinstance(vision_layers, (tuple, list)):
            self.visual = ModifiedResNet(vision_layers, embed_dim, vision_width * 32 // 64, image_resolution, vision_width)
        else:
            self.visual = VisionTransformer(image_resolution, vision_patch_size, vision_width, vision_layers,
                                            vision_width // 64, embed_dim)
        self.transformer = Transformer(transformer_width, transformer_layers, transformer_heads, causal=True)
        self.vocab_size = vocab_size
        self.token_embedding = nn.Embedding(vocab_size, transformer_width)
        self.positional_embedding = nn.Parameter(torch.empty(context_length, transformer_width))
        self.ln_final = LayerNorm(transformer_width)
        self.text_projection = nn.Parameter(torch.empty(transformer_width, embed_dim))
        self.logit_scale = nn.Parameter(torch.ones([]) * np.log(1 / 0.07))
        self.initialize_parameters()

    def initialize_parameters(self):
        nn.init.normal_(self.token_embedding.weight, std=0.02)
        nn.init.normal_(self.positional_embedding, std=0.01)
        proj_std = (self.transformer.width ** -0.5) * ((2 * self.transformer.layers) ** -0.5)
        attn_std, fc_std = self.transformer.width ** -0.5, (2 * self.transformer.width) ** -0.5
        for block in self.transformer.resblocks:
            nn.init.normal_(block.attn.in_proj_weight, std=attn_std)
            nn.init.normal_(block.attn.out_proj.weight, std=proj_std)
            nn.init.normal_(block.mlp.c_fc.weight, std=fc_std)
            nn.init.normal_(block.mlp.c_proj.weight, std=proj_std)
        nn.init.normal_(self.text_projection, std=self.transformer.width ** -0.5)

    def build_attention_mask(self):
        return torch.full((self.context_length, self.context_length), float("-inf")).triu_(1)

    @property
    def dtype(self):
        return self.visual.conv1.weight.dtype

    def encode_image(self, image):
        return self.visual(image.type(self.dtype))

    def encode_text(self, text):
        x = self.token_embedding(text).type(self.dtype) + self.positional_embedding.type(self.dtype)
        x = self.transformer(x.permute(1, 0, 2)).permute(1, 0, 2)
        x = self.ln_final(x).type(self.dtype)
        return x[torch.arange(x.shape[0]), text.argmax(dim=-1)] @ self.text_projection  # features at the EOT token

    def forward(self, image, text):
        img, txt = self.encode_image(image), self.encode_text(text)
        img = img / img.norm(dim=1, keepdim=True)
        txt = txt / txt.norm(dim=1, keepdim=True)
        logits_per_image = self.logit_scale.exp() * img @ txt.t()
        return logits_per_image, logits_per_image.t()


def convert_weights(model: nn.Module, dtype=torch.bfloat16):
    """Cast the matmul / conv weights to half precision (bf16 on H100), keep norms in fp32."""

    def _convert(layer):
        if isinstance(layer, (nn.Conv1d, nn.Conv2d, nn.Linear)):
            layer.weight.data = layer.weight.data.to(dtype)
            if layer.bias is not None:
                layer.bias.data = layer.bias.data.to(dtype)
        if isinstance(layer, MultiheadAttention):
            layer.in_proj_weight.data = layer.in_proj_weight.data.to(dtype)
            layer.in_proj_bias.data = layer.in_proj_bias.data.to(dtype)
        for name in ("text_projection", "proj"):
            attr = getattr(layer, name, None)
            if isinstance(attr, nn.Parameter):
                attr.data = attr.data.to(dtype)

    model.apply(_convert)


def build_model(state_dict: dict):
    vit = "visual.proj" in state_dict
    if vit:
        vision_width = state_dict["visual.conv1.weight"].shape[0]
        vision_layers = len([k for k in state_dict if k.startswith("visual.") and k.endswith(".attn.in_proj_weight")])
        vision_patch_size = state_dict["visual.conv1.weight"].shape[-1]
        grid = round((state_dict["visual.positional_embedding"].shape[0] - 1) ** 0.5)
        image_resolution = vision_patch_size * grid
    else:
        counts = [len(set(k.split(".")[2] for k in state_dict if k.startswith(f"visual.layer{b}"))) for b in [1, 2, 3, 4]]
        vision_layers = tuple(counts)
        vision_width = state_dict["visual.layer1.0.conv1.weight"].shape[0]
        output_width = round((state_dict["visual.attnpool.positional_embedding"].shape[0] - 1) ** 0.5)
        vision_patch_size = None
        image_resolution = output_width * 32
    embed_dim = state_dict["text_projection"].shape[1]
    context_length = state_dict["positional_embedding"].shape[0]
    vocab_size = state_dict["token_embedding.weight"].shape[0]
    transformer_width = state_dict["ln_final.weight"].shape[0]
    transformer_layers = len(set(k.split(".")[2] for k in state_dict if k.startswith("transformer.resblocks")))
    model = CLIP(embed_dim, image_resolution, vision_layers, vision_width, vision_patch_size, context_length, vocab_size,
                 transformer_width, transformer_width // 64, transformer_layers)
    for key in ("input_resolution", "context_length", "vocab_size"):
        state_dict.pop(key, None)
    model.load_state_dict(state_dict)
    return model.eval()
