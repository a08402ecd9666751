"""Shifted-window attention without a GPU: a Python mirror of the kernel's coordinate math (window_attention_sm90.cu,
``load_window`` and ``score``) reproduces ``relative_position_index`` and ``shifted_window_mask``; the fp64 reference of
the GPU tests agrees with the models' own window path and with autograd; the dispatch keeps the PyTorch path on the
CPU, under ``LIBAI_B200_IMPL=ref``, for unsupported shapes and for attention dropout; ptxas reports no spills."""
import os
import re
import subprocess

import pytest
import torch

from libai_b200.models.swin_transformer import relative_position_index, shifted_window_mask
from libai_b200.ops import build as ops_build
from libai_b200.ops import functional as OF
from tests import window_attention_ref as ref


def kernel_meta(H, W, ws, shift):
    """Per window and local index: (image-order token, rel-position coordinate, region label), as load_window forms
    them."""
    out = []
    for wy in range(H // ws):
        for wx in range(W // ws):
            rows = []
            for i in range(ws * ws):
                yi, xi = divmod(i, ws)
                ry, rx = wy * ws + yi, wx * ws + xi
                y = ry + shift if ry + shift < H else ry + shift - H
                x = rx + shift if rx + shift < W else rx + shift - W
                ly = 0 if ry < H - ws else (1 if ry < H - shift else 2)
                lx = 0 if rx < W - ws else (1 if rx < W - shift else 2)
                rows.append((y * W + x, yi * (2 * ws - 1) + xi, 3 * ly + lx))
            out.append(rows)
    return out


@pytest.mark.parametrize("ws", range(1, 17))
def test_kernel_rel_index_matches_relative_position_index(ws):
    meta = kernel_meta(ws, ws, ws, 0)[0]
    rel0 = (ws - 1) * 2 * ws
    rel = torch.tensor([[mi[1] - mj[1] + rel0 for mj in meta] for mi in meta])
    assert torch.equal(rel, relative_position_index((ws, ws)))


@pytest.mark.parametrize("H,W,ws", [(4, 4, 2), (8, 12, 4), (14, 14, 7), (14, 21, 7), (16, 8, 8), (24, 36, 12),
                                    (32, 16, 16), (3, 6, 3)])
def test_kernel_labels_match_shifted_window_mask(H, W, ws):
    for shift in range(1, ws):
        meta = kernel_meta(H, W, ws, shift)
        mask = torch.tensor([[[0.0 if mi[2] == mj[2] else -100.0 for mj in win] for mi in win] for win in meta])
        assert torch.equal(mask, shifted_window_mask(H, W, ws, shift, "cpu")), shift
        # the token map is roll(-shift) then partition: window_tokens of the reference
        tok = torch.tensor([[m[0] for m in win] for win in meta])
        assert torch.equal(tok, ref.window_tokens(H, W, ws, shift))


def _window_path(qkv, H, W, ws, shift, heads, scale, table, tau):
    """The models' computation (roll -> partition -> scores -> softmax -> reverse -> roll) in fp64 on qkv."""
    from libai_b200.models.swin_transformer import window_partition, window_reverse

    B, L, C3 = qkv.shape
    C, d, N = C3 // 3, C3 // 3 // heads, ws * ws
    x = qkv.view(B, H, W, C3)
    if shift:
        x = torch.roll(x, shifts=(-shift, -shift), dims=(1, 2))
    win = window_partition(x, ws).view(-1, N, 3, heads, d).permute(2, 0, 3, 1, 4)
    q, k, v = win[0], win[1], win[2]
    if tau is None:
        attn = scale * q @ k.transpose(-1, -2)
    else:
        attn = torch.nn.functional.normalize(q, dim=-1) @ torch.nn.functional.normalize(k, dim=-1).transpose(-1, -2)
        attn = attn * tau.view(1, heads, 1, 1)
    attn = attn + table[relative_position_index((ws, ws)).view(-1)].view(N, N, heads).permute(2, 0, 1)
    if shift:
        mask = shifted_window_mask(H, W, ws, shift, "cpu").double()
        nW = mask.shape[0]
        attn = (attn.view(B, nW, heads, N, N) + mask[None, :, None]).view(-1, heads, N, N)
    o = (torch.softmax(attn, -1) @ v).transpose(1, 2).reshape(-1, ws, ws, C)
    o = window_reverse(o, ws, H, W)
    if shift:
        o = torch.roll(o, shifts=(shift, shift), dims=(1, 2))
    return o.reshape(B, H * W, C)


@pytest.mark.parametrize("cosine", [False, True])
@pytest.mark.parametrize("H,W,ws,shift", [(8, 12, 4, 2), (14, 7, 7, 3), (6, 6, 3, 1)])
def test_reference_matches_window_path_and_autograd(H, W, ws, shift, cosine):
    torch.manual_seed(0)
    B, heads, d = 2, 3, 8
    qkv = torch.randn(B, H * W, 3 * heads * d, dtype=torch.float64, requires_grad=True)
    table = torch.randn((2 * ws - 1) ** 2, heads, dtype=torch.float64, requires_grad=True)
    tau = (torch.rand(heads, dtype=torch.float64) * 20 + 1).requires_grad_(True) if cosine else None
    dout = torch.randn(B, H * W, heads * d, dtype=torch.float64)
    o = _window_path(qkv, H, W, ws, shift, heads, 0.3, table, tau)
    o_ref, _ = ref.forward(qkv.detach(), H, W, ws, shift, heads, 0.3, table.detach(),
                           None if tau is None else tau.detach())
    assert torch.allclose(o, o_ref, rtol=1e-12, atol=1e-12)
    o.backward(dout)
    (g, _), (t, _), (u, _) = ref.backward(dout, qkv.detach(), H, W, ws, shift, heads, 0.3, table.detach(),
                                          None if tau is None else tau.detach())
    assert torch.allclose(g, qkv.grad, rtol=1e-10, atol=1e-10)
    assert torch.allclose(t, table.grad, rtol=1e-10, atol=1e-10)
    if cosine:
        assert torch.allclose(u, tau.grad, rtol=1e-10, atol=1e-10)


def test_dispatch(monkeypatch):
    x = torch.zeros(2, 64, 96, dtype=torch.bfloat16)
    ok = dict(H=8, W=8, window=8, shift=4, head_dim=32)
    assert not OF.window_attention_supported(x, **ok)                         # CPU tensors keep the PyTorch path
    monkeypatch.setattr(OF, "use_native", lambda *t: True)                     # as if on the GPU
    assert OF.window_attention_supported(x, **ok)
    assert OF.window_attention_supported(x, **dict(ok, head_dim=8))
    assert OF.window_attention_supported(x, **dict(ok, head_dim=64))
    assert OF.window_attention_supported(x, **dict(ok, H=8, W=24))
    assert OF.window_attention_supported(x, **dict(ok, window=1, shift=0))
    assert OF.window_attention_supported(x, **dict(ok, attn_drop=0.1, training=False))
    for bad in (dict(head_dim=4), dict(head_dim=12), dict(head_dim=72), dict(window=17, H=17, W=17, shift=0),
                dict(H=12), dict(shift=8), dict(shift=-1), dict(attn_drop=0.1, training=True)):
        assert not OF.window_attention_supported(x, **dict(ok, **bad)), bad
    assert not OF.window_attention_supported(x.float(), **ok)
    monkeypatch.undo()
    monkeypatch.setenv("LIBAI_B200_IMPL", "ref")
    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: pytest.fail("the extension must not be reached"))
    assert not OF.window_attention_supported(x, **ok)


@pytest.mark.parametrize("version", [1, 2])
def test_models_keep_window_path_on_cpu(version, monkeypatch):
    from libai_b200.models import swin_transformer as v1
    from libai_b200.models import swin_transformer_v2 as v2

    mod = v1 if version == 1 else v2
    monkeypatch.setattr(mod.WindowAttention, "forward_image",
                        lambda *a, **k: pytest.fail("the native window path must not run on the CPU"))
    block = mod.SwinTransformerBlock(dim=48, input_resolution=(8, 8), num_heads=2, window_size=4, shift_size=2)
    y = block(torch.randn(2, 64, 48))
    assert y.shape == (2, 64, 48) and torch.isfinite(y).all()


def window_reports(log):
    """{mangled kernel name: the ptxas lines reported for it} for every kernel of window_attention_sm90.cu."""
    reports, name = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = m.group(1)
            reports[name] = []
        elif name:
            reports[name].append(line)
    return reports


@pytest.mark.skipif(not os.path.exists(ops_build.NVCC), reason="needs nvcc")
def test_window_kernels_do_not_spill(tmp_path):
    res = subprocess.run([ops_build.NVCC, *ops_build.NVCC_FLAGS, "-I", ops_build.CSRC, "-c",
                          os.path.join(ops_build.CSRC, "window_attention_sm90.cu"), "-o", str(tmp_path / "w.o")],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    reports = window_reports(res.stdout)
    attn = [n for n in reports if "window_attn_fwd_kernel" in n or "window_attn_bwd_kernel" in n]
    assert len(attn) == 16, list(reports)      # forward and backward at 4 padded head dims, plain and cosine
    for name, lines in reports.items():
        spills = [ln for ln in lines if "spill" in ln]
        assert spills, (name, lines)
        for ln in spills:
            assert re.search(r"\b0 bytes spill stores, 0 bytes spill loads", ln), (name, ln)
