"""ConvNeXt (HF-compatible naming: ``embeddings / encoder.stages.N.layers.M / layernorm / classifier``).

Spec: reference projects/ConvNeXT/modeling/{convnext_layers.py,convnext_model.py,embedding.py,layer_norm.py} —
4×4 patchify stem + channels-first LayerNorm, stages of ``dwconv7×7 → LN → Linear(4×) → GELU → Linear → layer
scale → drop path`` blocks with 2×2 strided down-sampling between stages, global average pooling, LayerNorm,
classifier with the ``problem_type`` dependent loss (:138-170).

H100 mapping: the depth-wise 7×7 convolution stays on cuDNN (channels-last), everything after it runs on the token
layout ``[N·H·W, C]`` through the native LayerNorm and the wgmma GEMM with the GELU epilogue (the 1×1 "pwconv"
layers are the column/row-parallel linears of the fused MLP node).
"""
import torch
from torch import nn

from libai_b200.config import configurable
from libai_b200.layers import DropPath, LayerNorm, Linear
from libai_b200.layers._param import create_parameter, trunc_normal_
from libai_b200.ops import functional as OF


def _tn(t, generator=None):
    return trunc_normal_(t, std=0.02, generator=generator)


class ConvNextLayerNorm(nn.Module):
    """LayerNorm over channels for ``channels_last`` ``[N, H, W, C]`` or ``channels_first`` ``[N, C, H, W]`` inputs."""

    def __init__(self, normalized_shape, eps=1e-6, data_format="channels_last", layer_idx=0):
        super().__init__()
        if data_format not in ("channels_last", "channels_first"):
            raise NotImplementedError(f"Unsupported data format: {data_format}")
        self.norm = LayerNorm(normalized_shape, eps=eps, layer_idx=layer_idx)
        self.data_format = data_format

    @property
    def weight(self):
        return self.norm.weight

    @property
    def bias(self):
        return self.norm.bias

    def forward(self, x):
        if self.data_format == "channels_last":
            return self.norm(x)
        return self.norm(x.permute(0, 2, 3, 1)).permute(0, 3, 1, 2)


class ConvNextEmbeddings(nn.Module):
    def __init__(self, num_channels, hidden_sizes, patch_size, layer_idx=0):
        super().__init__()
        self.patch_embeddings = nn.Conv2d(num_channels, hidden_sizes[0], kernel_size=patch_size, stride=patch_size)
        self.layernorm = ConvNextLayerNorm(hidden_sizes[0], eps=1e-6, data_format="channels_first", layer_idx=layer_idx)
        self.num_channels = num_channels

    def forward(self, x):
        if x.shape[1] != self.num_channels:
            raise ValueError("Make sure that the channel dimension of the pixel values match with the one set in the configuration.")
        return self.layernorm(self.patch_embeddings(x.to(self.patch_embeddings.weight.dtype)))


class ConvNextLayer(nn.Module):
    def __init__(self, dim, eps=1e-6, drop_path=0, layer_scale_init_value=1e-6, layer_idx=0):
        super().__init__()
        self.dwconv = nn.Conv2d(dim, dim, kernel_size=7, padding=3, groups=dim)
        self.layernorm = ConvNextLayerNorm(dim, eps=eps, layer_idx=layer_idx)
        self.pwconv1 = Linear(dim, 4 * dim, parallel="col", init_method=_tn, layer_idx=layer_idx)
        self.pwconv2 = Linear(4 * dim, dim, parallel="row", init_method=_tn, layer_idx=layer_idx)
        self.layer_scale_parameter = (
            create_parameter((dim,), lambda t, generator=None: t.fill_(layer_scale_init_value), layer_idx=layer_idx)
            if layer_scale_init_value > 0 else None
        )
        self.drop_path = DropPath(drop_path) if drop_path > 0.0 else nn.Identity()
        self.layer_idx = layer_idx

    def forward(self, hidden_states):
        x = self.dwconv(hidden_states).permute(0, 2, 3, 1)      # (N, C, H, W) -> (N, H, W, C)
        x = self.pwconv2(self.pwconv1(self.layernorm(x), act="gelu"))
        if self.layer_scale_parameter is not None:
            x = self.layer_scale_parameter.to(x.dtype) * x
        return hidden_states + self.drop_path(x.permute(0, 3, 1, 2))


class ConvNextStage(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size=2, stride=2, depth=2, drop_path_rates=None, layer_idx=0):
        super().__init__()
        if in_channels != out_channels or stride > 1:
            self.downsampling_layer = nn.Sequential(
                ConvNextLayerNorm(in_channels, eps=1e-6, data_format="channels_first", layer_idx=layer_idx),
                nn.Conv2d(in_channels, out_channels, kernel_size=kernel_size, stride=stride),
            )
        else:
            self.downsampling_layer = nn.Identity()
        rates = drop_path_rates or [0.0] * depth
        self.layers = nn.Sequential(*[ConvNextLayer(out_channels, drop_path=rates[j], layer_idx=layer_idx) for j in range(depth)])

    def forward(self, hidden_states):
        return self.layers(self.downsampling_layer(hidden_states))


class ConvNextEncoder(nn.Module):
    def __init__(self, hidden_sizes, depths, num_stages, drop_path_rate):
        super().__init__()
        rates = [x.tolist() for x in torch.linspace(0, drop_path_rate, sum(depths)).split(depths)]
        self.stages = nn.ModuleList()
        prev = hidden_sizes[0]
        for i in range(num_stages):
            self.stages.append(ConvNextStage(prev, hidden_sizes[i], stride=2 if i > 0 else 1, depth=depths[i],
                                             drop_path_rates=rates[i], layer_idx=i))
            prev = hidden_sizes[i]

    def forward(self, hidden_states):
        for stage in self.stages:
            hidden_states = stage(hidden_states)
        return hidden_states


class ConvNextModel(nn.Module):
    @configurable
    def __init__(self, num_channels, patch_size, num_stages, hidden_sizes, depths, layer_norm_eps=1e-12, drop_path_rate=0.0):
        super().__init__()
        self.embeddings = ConvNextEmbeddings(num_channels, hidden_sizes, patch_size)
        self.encoder = ConvNextEncoder(hidden_sizes, list(depths), num_stages, drop_path_rate)
        self.layernorm = LayerNorm(hidden_sizes[-1], eps=layer_norm_eps, layer_idx=-1)

    @classmethod
    def from_config(cls, cfg):
        return {k: cfg[k] for k in ("num_channels patch_size num_stages hidden_sizes depths layer_norm_eps drop_path_rate").split()}

    def forward(self, x):
        x = self.encoder(self.embeddings(x))
        return self.layernorm(x.mean([-2, -1]))      # global average pooling, (N, C, H, W) -> (N, C)


class ConvNextForImageClassification(nn.Module):
    @configurable
    def __init__(self, num_channels, patch_size, num_stages, hidden_sizes, depths, layer_norm_eps=1e-12, drop_path_rate=0.0,
                 num_labels=1000, initializer_range=0.02, problem_type=None, image_size=224):
        super().__init__()
        self.num_labels, self.problem_type = num_labels, problem_type
        self.convnext = ConvNextModel(num_channels, patch_size, num_stages, hidden_sizes, depths, layer_norm_eps, drop_path_rate)
        self.classifier = Linear(hidden_sizes[-1], num_labels, init_method=_tn, layer_idx=-1) if num_labels > 0 else nn.Identity()

    @classmethod
    def from_config(cls, cfg):
        keys = "num_channels patch_size num_stages hidden_sizes depths layer_norm_eps drop_path_rate num_labels initializer_range problem_type".split()
        return {k: cfg[k] for k in keys if k in cfg}

    def forward(self, images, labels=None):
        logits = self.classifier(self.convnext(images))
        if labels is None or not self.training:
            return {"prediction_scores": logits}
        problem = self.problem_type
        if problem is None:
            if self.num_labels == 1:
                problem = "regression"
            elif labels.dtype in (torch.long, torch.int):
                problem = "single_label_classification"
            else:
                problem = "multi_label_classification"
        if problem == "regression":
            loss = nn.functional.mse_loss(logits.float().squeeze(), labels.float().squeeze())
        elif problem == "single_label_classification":
            loss = nn.functional.cross_entropy(logits.float().view(-1, self.num_labels), labels.view(-1))
        elif labels.dim() == 2 and labels.dtype.is_floating_point and float(labels.sum(-1).mean()) <= 1.0 + 1e-3:
            loss = torch.sum(-labels * torch.log_softmax(logits.float(), dim=-1), dim=-1).mean()  # Mixup soft targets
        else:
            loss = nn.functional.binary_cross_entropy_with_logits(logits.float(), labels.float())
        return {"losses": loss}

    @staticmethod
    def set_activation_checkpoint(model):
        return model

    @staticmethod
    def set_pipeline_stage_id(model):
        return model
