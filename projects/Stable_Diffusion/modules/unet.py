"""Conditional latent-diffusion UNet (the ``UNet2DConditionModel`` of Stable Diffusion v1/v2).

The reference project (projects/Stable_Diffusion/modeling.py:17-40) takes this network from the ``diffusers``
package; this framework carries its own implementation so the project has no dependency outside the repo.  Module
and parameter names follow the public diffusers checkpoint layout (``down_blocks.0.attentions.1.transformer_blocks.0
.attn2.to_k.weight`` ...) so released Stable Diffusion weights load by name (``modules/loader.py``).

H100 notes: the transformer blocks are where the time goes at 64×64 latents (4096 tokens): their projections and
the GEGLU feed-forward are ``libai_b200.layers.Linear`` (wgmma GEMM), attention goes through ``ops.attention``
(flash kernel for head_dim 64/128, which covers SD2.x; SD1.x head dims 40/80/160 use the reference math), and
tensors stay channels-last through the convolutions.
"""
import math
from typing import Optional, Sequence

import torch
import torch.nn.functional as F
from torch import nn

from libai_b200.layers import Linear
from libai_b200.ops import functional as OF


def timestep_embedding(timesteps, dim, flip_sin_to_cos=True, freq_shift=0, max_period=10000):
    half = dim // 2
    exponent = -math.log(max_period) * torch.arange(half, dtype=torch.float32, device=timesteps.device)
    emb = timesteps.float()[:, None] * torch.exp(exponent / (half - freq_shift))[None]
    emb = torch.cat([emb.sin(), emb.cos()], dim=-1)
    if flip_sin_to_cos:
        emb = torch.cat([emb[:, half:], emb[:, :half]], dim=-1)
    return F.pad(emb, (0, dim % 2))


class TimestepEmbedding(nn.Module):
    def __init__(self, in_channels, time_embed_dim):
        super().__init__()
        self.linear_1 = Linear(in_channels, time_embed_dim)
        self.linear_2 = Linear(time_embed_dim, time_embed_dim)

    def forward(self, x):
        return self.linear_2(self.linear_1(x, "silu"))


class ResnetBlock2D(nn.Module):
    def __init__(self, in_channels, out_channels, temb_channels=None, groups=32, eps=1e-5):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, padding=1)
        self.time_emb_proj = Linear(temb_channels, out_channels) if temb_channels else None
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=eps)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 1) if in_channels != out_channels else None

    def forward(self, x, temb=None):
        h = self.conv1(F.silu(self.norm1(x)))
        if self.time_emb_proj is not None and temb is not None:
            h = h + self.time_emb_proj(F.silu(temb)).to(h.dtype)[:, :, None, None]
        h = self.conv2(F.silu(self.norm2(h)))
        return (x if self.conv_shortcut is None else self.conv_shortcut(x)) + h


class Attention(nn.Module):
    """Multi-head attention with separate q/k/v projections (self- or cross-); ``lora`` adapters attach here."""

    def __init__(self, query_dim, cross_attention_dim=None, heads=8, dim_head=64, bias=False):
        super().__init__()
        inner = heads * dim_head
        self.heads, self.dim_head = heads, dim_head
        self.to_q = Linear(query_dim, inner, bias=bias)
        self.to_k = Linear(cross_attention_dim or query_dim, inner, bias=bias)
        self.to_v = Linear(cross_attention_dim or query_dim, inner, bias=bias)
        self.to_out = nn.ModuleList([Linear(inner, query_dim), nn.Identity()])
        self.lora = None      # set by modules/lora.py

    def _proj(self, name, layer, x):
        y = layer(x)
        if self.lora is not None:
            y = y + self.lora(name, x).to(y.dtype)
        return y

    def forward(self, x, context=None):
        b, n, _ = x.shape
        ctx = x if context is None else context.to(x.dtype)
        q = self._proj("to_q", self.to_q, x).view(b, n, self.heads, self.dim_head).transpose(1, 2)
        k = self._proj("to_k", self.to_k, ctx).view(b, ctx.shape[1], self.heads, self.dim_head).transpose(1, 2)
        v = self._proj("to_v", self.to_v, ctx).view(b, ctx.shape[1], self.heads, self.dim_head).transpose(1, 2)
        o = OF.attention(q, k, v, causal=False)
        o = o.transpose(1, 2).reshape(b, n, self.heads * self.dim_head)
        return self._proj("to_out", self.to_out[0], o)


class GEGLU(nn.Module):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = Linear(dim_in, dim_out * 2)

    def forward(self, x):
        h, gate = self.proj(x).chunk(2, dim=-1)
        return h * F.gelu(gate)


class FeedForward(nn.Module):
    def __init__(self, dim, mult=4):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, dim * mult), nn.Identity(), Linear(dim * mult, dim)])

    def forward(self, x):
        return self.net[2](self.net[0](x))


class BasicTransformerBlock(nn.Module):
    def __init__(self, dim, heads, dim_head, cross_attention_dim):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim)
        self.attn1 = Attention(dim, None, heads, dim_head)
        self.norm2 = nn.LayerNorm(dim)
        self.attn2 = Attention(dim, cross_attention_dim, heads, dim_head)
        self.norm3 = nn.LayerNorm(dim)
        self.ff = FeedForward(dim)

    def forward(self, x, context):
        x = x + self.attn1(self.norm1(x))
        x = x + self.attn2(self.norm2(x), context)
        return x + self.ff(self.norm3(x))


class Transformer2DModel(nn.Module):
    def __init__(self, heads, dim_head, in_channels, cross_attention_dim, groups=32, use_linear_projection=False):
        super().__init__()
        inner = heads * dim_head
        self.use_linear_projection = use_linear_projection
        self.norm = nn.GroupNorm(groups, in_channels, eps=1e-6)
        self.proj_in = Linear(in_channels, inner) if use_linear_projection else nn.Conv2d(in_channels, inner, 1)
        self.transformer_blocks = nn.ModuleList([BasicTransformerBlock(inner, heads, dim_head, cross_attention_dim)])
        self.proj_out = Linear(inner, in_channels) if use_linear_projection else nn.Conv2d(inner, in_channels, 1)

    def forward(self, x, context):
        b, c, h, w = x.shape
        res = x
        x = self.norm(x)
        if self.use_linear_projection:
            x = self.proj_in(x.permute(0, 2, 3, 1).reshape(b, h * w, c))
        else:
            x = self.proj_in(x).permute(0, 2, 3, 1).reshape(b, h * w, -1)
        for blk in self.transformer_blocks:
            x = blk(x, context)
        if self.use_linear_projection:
            x = self.proj_out(x).reshape(b, h, w, c).permute(0, 3, 1, 2)
        else:
            x = self.proj_out(x.reshape(b, h, w, -1).permute(0, 3, 1, 2))
        return x + res


class Downsample2D(nn.Module):
    def __init__(self, channels, padding=1):
        super().__init__()
        self.padding = padding
        self.conv = nn.Conv2d(channels, channels, 3, stride=2, padding=padding)

    def forward(self, x):
        if self.padding == 0:                    # the VAE encoder pads asymmetrically
            x = F.pad(x, (0, 1, 0, 1))
        return self.conv(x)


class Upsample2D(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, padding=1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


class DownBlock(nn.Module):
    def __init__(self, cin, cout, temb, layers, heads, cross_dim, with_attn, add_down, groups, linear_proj):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if j == 0 else cout, cout, temb, groups) for j in range(layers)])
        self.attentions = nn.ModuleList(
            [Transformer2DModel(heads, cout // heads, cout, cross_dim, groups, linear_proj) for _ in range(layers)]
        ) if with_attn else None
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_down else None

    def forward(self, x, temb, context):
        skips = []
        for j, res in enumerate(self.resnets):
            x = res(x, temb)
            if self.attentions is not None:
                x = self.attentions[j](x, context)
            skips.append(x)
        if self.downsamplers is not None:
            x = self.downsamplers[0](x)
            skips.append(x)
        return x, skips


class UpBlock(nn.Module):
    def __init__(self, cin, cout, cprev, temb, layers, heads, cross_dim, with_attn, add_up, groups, linear_proj):
        super().__init__()
        resnets = []
        for j in range(layers):
            skip_c = cin if j == layers - 1 else cout
            in_c = cprev if j == 0 else cout
            resnets.append(ResnetBlock2D(in_c + skip_c, cout, temb, groups))
        self.resnets = nn.ModuleList(resnets)
        self.attentions = nn.ModuleList(
            [Transformer2DModel(heads, cout // heads, cout, cross_dim, groups, linear_proj) for _ in range(layers)]
        ) if with_attn else None
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_up else None

    def forward(self, x, skips, temb, context):
        for j, res in enumerate(self.resnets):
            x = res(torch.cat([x, skips[-1 - j]], dim=1), temb)
            if self.attentions is not None:
                x = self.attentions[j](x, context)
        if self.upsamplers is not None:
            x = self.upsamplers[0](x)
        return x


class MidBlock(nn.Module):
    def __init__(self, c, temb, heads, cross_dim, groups, linear_proj):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, temb, groups), ResnetBlock2D(c, c, temb, groups)])
        self.attentions = nn.ModuleList([Transformer2DModel(heads, c // heads, c, cross_dim, groups, linear_proj)])

    def forward(self, x, temb, context):
        x = self.resnets[0](x, temb)
        x = self.attentions[0](x, context)
        return self.resnets[1](x, temb)


class UNetOutput:
    def __init__(self, sample):
        self.sample = sample


class UNet2DConditionModel(nn.Module):
    """Defaults are Stable Diffusion v1 (860M parameters)."""

    def __init__(self, in_channels=4, out_channels=4, block_out_channels: Sequence[int] = (320, 640, 1280, 1280),
                 down_block_types=("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
                 up_block_types=("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"),
                 layers_per_block=2, cross_attention_dim=768, attention_head_dim=8, norm_num_groups=32,
                 use_linear_projection=False, flip_sin_to_cos=True, freq_shift=0, **unused):
        super().__init__()
        self.config = dict(in_channels=in_channels, out_channels=out_channels,
                           block_out_channels=list(block_out_channels), down_block_types=list(down_block_types),
                           up_block_types=list(up_block_types), layers_per_block=layers_per_block,
                           cross_attention_dim=cross_attention_dim, attention_head_dim=attention_head_dim,
                           norm_num_groups=norm_num_groups, use_linear_projection=use_linear_projection,
                           flip_sin_to_cos=flip_sin_to_cos, freq_shift=freq_shift)
        ch = list(block_out_channels)
        temb = ch[0] * 4
        g = norm_num_groups
        self.flip_sin_to_cos, self.freq_shift = flip_sin_to_cos, freq_shift
        self.conv_in = nn.Conv2d(in_channels, ch[0], 3, padding=1)
        self.time_embedding = TimestepEmbedding(ch[0], temb)

        def n_heads(i):
            # despite its name the config field holds the head *count* (8 for SD1.x → head dims 40/80/160;
            # [5, 10, 20, 20] for SD2.x → head dim 64 everywhere, the flash-kernel case)
            return attention_head_dim[i] if isinstance(attention_head_dim, (list, tuple)) else attention_head_dim

        self.down_blocks = nn.ModuleList()
        cout = ch[0]
        for i, kind in enumerate(down_block_types):
            cin, cout = cout, ch[i]
            self.down_blocks.append(DownBlock(cin, cout, temb, layers_per_block, n_heads(i), cross_attention_dim,
                                              kind.startswith("CrossAttn"), i < len(ch) - 1, g, use_linear_projection))
        self.mid_block = MidBlock(ch[-1], temb, n_heads(len(ch) - 1), cross_attention_dim, g, use_linear_projection)
        self.up_blocks = nn.ModuleList()
        rev = list(reversed(ch))
        cout = rev[0]
        for i, kind in enumerate(up_block_types):
            cprev, cout = cout, rev[i]
            cin = rev[min(i + 1, len(ch) - 1)]
            self.up_blocks.append(UpBlock(cin, cout, cprev, temb, layers_per_block + 1, n_heads(len(ch) - 1 - i),
                                          cross_attention_dim, kind.startswith("CrossAttn"), i < len(ch) - 1, g,
                                          use_linear_projection))
        self.conv_norm_out = nn.GroupNorm(g, ch[0], eps=1e-5)
        self.conv_out = nn.Conv2d(ch[0], out_channels, 3, padding=1)
        self.gradient_checkpointing = False

    @property
    def dtype(self):
        return self.conv_in.weight.dtype

    def attention_modules(self):
        """name → Attention, in registration order (LoRA attaches one adapter per entry)."""
        return {n: m for n, m in self.named_modules() if isinstance(m, Attention)}

    def _run(self, block, *args):
        if self.gradient_checkpointing and self.training:
            from torch.utils.checkpoint import checkpoint

            return checkpoint(block, *args, use_reentrant=False)
        return block(*args)

    def forward(self, sample, timesteps, encoder_hidden_states):
        if not torch.is_tensor(timesteps):
            timesteps = torch.tensor([timesteps], device=sample.device)
        timesteps = timesteps.reshape(-1).expand(sample.shape[0])
        t = timestep_embedding(timesteps, self.config["block_out_channels"][0], self.flip_sin_to_cos, self.freq_shift)
        temb = self.time_embedding(t.to(self.dtype))
        ctx = encoder_hidden_states.to(self.dtype)
        x = self.conv_in(sample.to(self.dtype))
        skips = [x]
        for blk in self.down_blocks:
            x, s = self._run(blk, x, temb, ctx)
            skips.extend(s)
        x = self._run(self.mid_block, x, temb, ctx)
        for blk in self.up_blocks:
            n = len(blk.resnets)
            take, skips = skips[-n:], skips[:-n]
            x = self._run(blk, x, list(take), temb, ctx)
        x = self.conv_out(F.silu(self.conv_norm_out(x)))
        return UNetOutput(x)
