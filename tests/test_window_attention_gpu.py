"""Native shifted-window attention on the GPU: every element of O, dqkv, the table gradient and dtau against the fp64
reference of ``tests/window_attention_ref.py``; bit-identical repeats and CUDA-graph replays; and Swin / SwinV2 models
on the native path against the same weights on the PyTorch window path."""
import copy
import math

import pytest
import torch

from tests import window_attention_ref as ref

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


def _inputs(B, H, W, ws, heads, d, cosine, seed, tau_value=10.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    C = heads * d
    qkv = torch.randn(B, H * W, 3 * C, generator=g).to(DEV, torch.bfloat16)
    table = (0.5 * torch.randn((2 * ws - 1) ** 2, heads, generator=g)).to(DEV)
    dout = torch.randn(B, H * W, C, generator=g).to(DEV, torch.bfloat16)
    tau = None
    if cosine:
        tau = (tau_value * (1.0 + 0.1 * torch.rand(heads, generator=g))).clamp(max=100.0).to(DEV)
    return qkv, table, tau, dout


# (B, H, W, ws, shift, heads, d, cosine, tau): every window size, shift 0 / 1 / ws // 2, head dims 8 / 24 / 32 / 64,
# 1 / 3 / 6 heads, B 1 / 2, a non-square map, cosine mode at tau 1, 10 and 100, and shapes with more windows than the
# backward has CTAs (about 2048 / heads)
CASES = [
    (2, 2, 3, 1, 0, 3, 32, False, None),
    (2, 8, 8, 4, 0, 1, 8, False, None),
    (1, 8, 12, 4, 1, 3, 24, False, None),
    (2, 8, 8, 4, 2, 6, 32, False, None),
    (2, 14, 14, 7, 0, 3, 32, False, None),
    (2, 14, 14, 7, 3, 3, 32, False, None),
    (1, 14, 21, 7, 3, 2, 24, False, None),
    (1, 14, 21, 7, 1, 3, 64, False, None),
    (2, 16, 16, 8, 4, 3, 24, False, None),
    (1, 16, 24, 8, 1, 6, 8, False, None),
    (1, 24, 24, 12, 6, 2, 32, False, None),
    (2, 24, 12, 12, 0, 1, 64, False, None),
    (1, 32, 32, 16, 8, 2, 32, False, None),
    (1, 16, 32, 16, 1, 1, 64, False, None),
    (2, 14, 14, 7, 3, 3, 32, True, 1.0),
    (1, 14, 21, 7, 3, 2, 24, True, 10.0),
    (2, 16, 16, 8, 4, 3, 32, True, 100.0),
    (1, 32, 32, 16, 8, 2, 32, True, 100.0),
    (1, 24, 24, 12, 6, 6, 8, True, 10.0),
    (1, 8, 8, 4, 2, 1, 64, True, 100.0),
    # more windows than backward CTAs: each CTA sums dS over several windows
    (2, 56, 56, 4, 2, 6, 8, False, None),
    (4, 56, 56, 7, 3, 12, 32, False, None),
    (2, 48, 48, 12, 6, 12, 16, True, 100.0),
]


def _run(ext, qkv, table, tau, dout, H, W, ws, shift, heads, scale):
    o, lse = ext.window_attn_fwd(qkv, H, W, ws, shift, heads, scale, table, tau)
    dqkv, dt, dtau = ext.window_attn_bwd(dout, qkv, lse, H, W, ws, shift, heads, scale, table, tau)
    return o, lse, dqkv, dt, dtau


@pytest.mark.parametrize("B,H,W,ws,shift,heads,d,cosine,tau_value", CASES)
def test_window_attention_matches_fp64(B, H, W, ws, shift, heads, d, cosine, tau_value):
    ext = _ext()
    qkv, table, tau, dout = _inputs(B, H, W, ws, heads, d, cosine, seed=B * 1000 + H * 31 + ws + shift + d,
                                    tau_value=tau_value or 1.0)
    scale = d ** -0.5
    o, _, dqkv, dt, dtau = _run(ext, qkv, table, tau, dout, H, W, ws, shift, heads, scale)
    torch.cuda.synchronize()
    o_ref, o_mag = ref.forward(qkv, H, W, ws, shift, heads, scale, table, tau)
    ref.assert_close(o, o_ref, o_mag, "O")
    (g_ref, g_mag), (t_ref, t_mag), (u_ref, u_mag) = ref.backward(dout, qkv, H, W, ws, shift, heads, scale, table, tau)
    ref.assert_close(dqkv, g_ref, g_mag, "dqkv")
    ref.assert_close(dt, t_ref, t_mag, "dtable", tol=ref.DS_TOL, out_tol=2.0 ** -20)
    if cosine:
        ref.assert_close(dtau, u_ref, u_mag, "dtau", tol=ref.DS_TOL, out_tol=2.0 ** -20)
    else:
        assert dtau.numel() == 0


@pytest.mark.parametrize("cosine", [False, True])
def test_window_attention_deterministic_and_graph_replay(cosine):
    ext = _ext()
    B, H, W, ws, shift, heads, d = 4, 28, 28, 7, 3, 3, 32
    qkv, table, tau, dout = _inputs(B, H, W, ws, heads, d, cosine, seed=7, tau_value=30.0)
    first = _run(ext, qkv, table, tau, dout, H, W, ws, shift, heads, d ** -0.5)
    second = _run(ext, qkv, table, tau, dout, H, W, ws, shift, heads, d ** -0.5)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            captured = _run(ext, qkv, table, tau, dout, H, W, ws, shift, heads, d ** -0.5)
    torch.cuda.current_stream().wait_stream(stream)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for a, b, c in zip(first, second, captured):
            assert torch.equal(a, b)
            assert torch.equal(a, c)


def _swin_models(version, img, window, embed, heads, depths):
    from libai_b200.layers._param import param_defaults

    if version == 1:
        from libai_b200.models.swin_transformer import SwinTransformer as M
        kw = {}
    else:
        from libai_b200.models.swin_transformer_v2 import SwinTransformerV2 as M
        kw = {"pretrained_window_sizes": [0] * len(depths)}
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
        model = M(img_size=img, patch_size=4, in_chans=3, num_classes=10, embed_dim=embed, depths=depths,
                  num_heads=heads, window_size=window, drop_path_rate=0.0, **kw)
    model.to(device=DEV, dtype=torch.bfloat16)   # the patch-embedding convolution and the buffers
    if version == 2:   # res-post-norm starts at zero; give the blocks non-trivial norms so every block contributes
        g = torch.Generator(device="cpu").manual_seed(5)
        with torch.no_grad():
            for name, prm in model.named_parameters():
                if ".norm1." in name or ".norm2." in name:
                    prm.copy_((1.0 if name.endswith("weight") else 0.0) + 0.1 * torch.randn(prm.shape, generator=g))
    return model


def _step(model, images, labels, train):
    model.zero_grad(set_to_none=True)
    model.train(train)
    if train:
        loss = model(images, labels)["losses"]
        loss.backward()
        grads = {n: p.grad.detach().float().clone() for n, p in model.named_parameters() if p.grad is not None}
        return loss.detach().float(), grads
    with torch.no_grad():
        return model(images)["prediction_scores"].float(), {}


# (version, image, window, embed, heads, depths): head dims 24 and 32 at the recipe window sizes 7, 8 and 12.  The last
# stage's map is no larger than the window, so its blocks use the whole map as the window and drop the shift (at
# window 8 the 4 x 4 map shrinks the window to 4).
MODELS = [
    (1, 112, 7, 48, [2, 4, 8], [2, 2, 2]),
    (1, 64, 8, 64, [2, 4, 8], [2, 2, 2]),
    (1, 96, 12, 64, [2, 4], [2, 2]),
    (2, 64, 8, 64, [2, 4, 8], [2, 2, 2]),
    (2, 112, 7, 48, [2, 4, 8], [2, 2, 2]),
]


@pytest.mark.parametrize("version,img,window,embed,heads,depths", MODELS)
def test_swin_models_native_match_window_path(version, img, window, embed, heads, depths, monkeypatch):
    from libai_b200.models import swin_transformer as v1
    from libai_b200.models import swin_transformer_v2 as v2

    mod = v1 if version == 1 else v2
    model = _swin_models(version, img, window, embed, heads, depths)
    g = torch.Generator(device="cpu").manual_seed(11)
    images = torch.randn(4, 3, img, img, generator=g).to(DEV)
    labels = torch.randint(0, 10, (4,), generator=g).to(DEV)

    # the native run: the PyTorch window path must not be taken anywhere
    def _raise(*a, **k):
        raise AssertionError("PyTorch window path taken")

    with monkeypatch.context() as m:
        m.setattr(mod.WindowAttention, "forward", _raise)
        m.setattr(mod, "window_partition", _raise)
        loss_n, grads_n = _step(model, images, labels, True)
        logits_n, _ = _step(model, images, labels, False)

    # the same weights on the PyTorch window path, in bf16 (what the blocks ran before) and in fp32 (the yardstick)
    model32 = copy.deepcopy(model).float()
    with monkeypatch.context() as m:
        m.setattr(mod.OF, "window_attention_supported", lambda *a, **k: False)
        m.setattr(mod.WindowAttention, "forward_image", _raise)
        m.setattr(torch.backends.cudnn, "allow_tf32", False)
        m.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
        loss_r, grads_r = _step(model, images, labels, True)
        logits_r, _ = _step(model, images, labels, False)
        loss_32, grads_32 = _step(model32, images, labels, True)
        logits_32, _ = _step(model32, images, labels, False)

    # Both bf16 runs differ from the fp32 run by bf16 roundings propagated through the network.  The native run must be
    # no further from fp32 than twice the old path's distance plus 5 % of the quantity's largest element.  The 5 % is
    # for logit_scale, a cancelling sum over every score of a block: in the first SwinV2 blocks the native run was up
    # to 5.9 % of its largest element from fp32 and the old path 1.6 % (H100).  The kernel rounds dS to bf16 for dQ and
    # dK, as flash attention does, where the old path runs the cosine scores' backward in fp32, so the gradient that
    # reaches earlier blocks is noisier.  The kernels themselves are checked element by element above.
    def no_worse(native, old, fp32, what):
        scale = fp32.abs().max().item()
        err_n, err_r = (native - fp32).abs().max().item(), (old - fp32).abs().max().item()
        assert err_n <= 2 * err_r + 5e-2 * scale + 1e-6, (what, err_n, err_r, scale)

    no_worse(logits_n, logits_r, logits_32, "logits")
    no_worse(loss_n, loss_r, loss_32, "loss")
    assert grads_n.keys() == grads_r.keys() == grads_32.keys()
    for name in grads_r:
        no_worse(grads_n[name], grads_r[name], grads_32[name], name)
    # every table-like parameter received a gradient through the kernel
    tables = [n for n in grads_n if "relative_position_bias_table" in n or "logit_scale" in n or "cpb_mlp" in n]
    assert tables and all(grads_n[n].abs().sum() > 0 for n in tables)


def test_predicate_and_errors():
    from libai_b200.ops import functional as OF

    x = torch.zeros(1, 64, 96, device=DEV, dtype=torch.bfloat16)
    assert OF.window_attention_supported(x, H=8, W=8, window=8, shift=4, head_dim=32)
    assert not OF.window_attention_supported(x, H=8, W=8, window=8, shift=4, head_dim=32, attn_drop=0.1, training=True)
    assert OF.window_attention_supported(x, H=8, W=8, window=8, shift=4, head_dim=32, attn_drop=0.1, training=False)
    ext = _ext()
    table = torch.zeros(15 * 15, 3, device=DEV)
    qkv = torch.zeros(1, 64, 3 * 3 * 12, device=DEV, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="multiples of 8 from 8 to 64"):
        ext.window_attn_fwd(qkv, 8, 8, 8, 0, 3, 1.0, table, None)
    qkv = torch.zeros(1, 64, 3 * 3 * 32, device=DEV, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="0 <= shift < window"):
        ext.window_attn_fwd(qkv, 8, 8, 8, 8, 3, 1.0, table, None)
    with pytest.raises(RuntimeError, match="whole number"):
        ext.window_attn_fwd(torch.zeros(1, 60, 3 * 3 * 32, device=DEV, dtype=torch.bfloat16), 6, 10, 8, 0, 3, 1.0,
                            table, None)
    assert math.isfinite(float(ext.window_attn_fwd(qkv, 8, 8, 8, 4, 3, 1.0, table, None)[0].float().sum()))
