"""NeRF positional encoding and MLP (spec: reference projects/NeRF/modeling/NeRF.py:22-146).

The MLP is eight 256-wide GEMMs over ``rays × samples`` points (≈200k rows per step at the default batch) — GEMM
shaped work, so the layers are this framework's ``Linear`` with the ReLU fused into the wgmma GEMM epilogue.
The first layer's input (63 channels) and the skip layer's input (319) are zero-padded to multiples of 8 so the
operand rows satisfy TMA's 16-byte alignment; the padding columns of the weights receive zero inputs and therefore
zero gradients."""
import torch
from torch import nn

from libai_b200.layers import Linear


def _pad8(n):
    return (n + 7) // 8 * 8


class Embedding(nn.Module):
    """x → (x, sin(2^k x), cos(2^k x), ...), k < N_freqs."""

    def __init__(self, in_channels, N_freqs, logscale=True):
        super().__init__()
        self.N_freqs = N_freqs
        self.in_channels = in_channels
        self.out_channels = in_channels * (2 * N_freqs + 1)
        bands = 2.0 ** torch.linspace(0, N_freqs - 1, N_freqs) if logscale else \
            torch.linspace(1, 2 ** (N_freqs - 1), N_freqs)
        self.register_buffer("freq_bands", bands, persistent=False)

    def forward(self, x):
        ang = x[..., None, :] * self.freq_bands.to(x.dtype)[:, None]              # [..., F, C]
        enc = torch.stack([ang.sin(), ang.cos()], dim=-2).flatten(-3)            # [..., F*2*C] (sin_k, cos_k order)
        return torch.cat([x, enc], dim=-1)


class PaddedLinear(nn.Module):
    """``Linear`` whose input width is padded up to a multiple of 8 (see module docstring)."""

    def __init__(self, in_features, out_features):
        super().__init__()
        self.in_features = in_features
        self.pad = _pad8(in_features) - in_features
        self.lin = Linear(in_features + self.pad, out_features, bias=True, init_method=_kaiming_uniform)

    def forward(self, x, act=None):
        if self.pad:
            x = torch.nn.functional.pad(x, (0, self.pad))
        return self.lin(x, act)


def _kaiming_uniform(t, generator=None):
    bound = (1.0 / t.shape[1]) ** 0.5
    return t.uniform_(-bound, bound, generator=generator) if generator is not None else t.uniform_(-bound, bound)


class NeRF(nn.Module):
    def __init__(self, D=8, W=256, input_ch=63, input_ch_views=27, output_ch=5, skips=(4,), use_viewdirs=True):
        super().__init__()
        self.D, self.W = D, W
        self.input_ch, self.input_ch_views = input_ch, input_ch_views
        self.skips = tuple(skips)
        self.use_viewdirs = use_viewdirs
        self.pts_linears = nn.ModuleList(
            [PaddedLinear(input_ch, W)]
            + [PaddedLinear(W + input_ch if i in self.skips else W, W) for i in range(D - 1)]
        )
        if use_viewdirs:
            self.views_linears = nn.ModuleList([PaddedLinear(input_ch_views + W, W // 2)])
            self.feature_linear = PaddedLinear(W, W)
            self.alpha_linear = Linear(W, 1, init_method=_kaiming_uniform)
            self.rgb_linear = Linear(W // 2, 3, init_method=_kaiming_uniform)
        else:
            self.output_linear = Linear(W, output_ch, init_method=_kaiming_uniform)

    def forward(self, x, sigma_only=False):
        """x: [B, input_ch (+ input_ch_views)] embedded position (and direction) → [B, 4] rgb+sigma, or [B, 1]
        sigma with ``sigma_only``."""
        if sigma_only:
            input_pts, input_views = x, None
        else:
            input_pts, input_views = torch.split(x, [self.input_ch, self.input_ch_views], dim=-1)
        h = input_pts
        for i, layer in enumerate(self.pts_linears):
            h = layer(h, "relu")
            if i in self.skips:
                h = torch.cat([input_pts, h], dim=-1)
        if not self.use_viewdirs:
            return self.output_linear(h)
        alpha = self.alpha_linear(h)
        if sigma_only:
            return alpha
        h = torch.cat([self.feature_linear(h), input_views], dim=-1)
        for layer in self.views_linears:
            h = layer(h, "relu")
        rgb = self.rgb_linear(h).sigmoid()
        return torch.cat([rgb, alpha], dim=-1)
