"""FP8 (E4M3) weights for inference without a GPU: the per-channel quantization of every ``Linear1D``, the reference
math of ``OF.linear_fp8w``, the guards of the bf16 GEMM entries, dtype casts, and ``generate()`` of every cache model
against the same model holding the dequantized weights in fp32."""
import copy
import sys

import pytest
import torch
import torch.nn.functional as F

from libai_b200.config import DictConfig
from libai_b200.inference import quantize_weights_fp8_
from libai_b200.layers.linear import Linear1D
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist

from tests.test_cached_attention_cpu import MODELS, _prompt

E4M3 = torch.float8_e4m3fn
HEADS = ("lm_head", "output_layer")


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cpu")))


def _linears(model):
    return {n: m for n, m in model.named_modules() if isinstance(m, Linear1D)}


def _param_bytes(model):
    return sum(p.numel() * p.element_size() for p in model.parameters())


def test_quantize_matches_kv_cache_quantizer():
    m = MODELS["llama"]()
    lins = _linears(m)
    lins["model.layers.0.mlp.down_proj"].weight.data[5].zero_()   # an all-zero row
    before = {n: l.weight.detach().clone() for n, l in lins.items()}
    head = lins["lm_head"].weight
    nbytes = _param_bytes(m)
    assert quantize_weights_fp8_(m) is m
    saved = 0
    for n, l in lins.items():
        if n == "lm_head":
            assert l.weight is head and l.weight.dtype == torch.bfloat16 and not l.fp8
            continue
        e, s = OF.kv_cache_quantize_ref(before[n])
        assert l.fp8 and l.compute_dtype == torch.bfloat16 and l.weight_scale.dtype == torch.float32
        assert l.weight.shape == before[n].shape and l.weight_scale.shape == (before[n].shape[0],)
        assert torch.equal(l.weight.view(torch.uint8), e.view(torch.uint8))
        assert torch.equal(l.weight_scale, s)
        assert not l.weight.requires_grad and not l.weight_scale.requires_grad
        saved += before[n].numel() * (2 - 1) - 4 * before[n].shape[0]
    assert lins["model.layers.0.mlp.down_proj"].weight_scale[5].item() == 1.0
    assert not any(p.dtype == torch.bfloat16 and p.dim() == 2 and n.endswith(("proj.weight", "query_key_value.weight"))
                   for n, p in m.named_parameters())
    assert _param_bytes(m) == nbytes - saved
    # a second call changes nothing
    snap = {n: (l.weight, getattr(l, "weight_scale", None)) for n, l in lins.items()}
    quantize_weights_fp8_(m)
    assert all(l.weight is snap[n][0] and getattr(l, "weight_scale", None) is snap[n][1] for n, l in lins.items())


def test_quantize_refuses_other_dtypes():
    m = MODELS["llama"]()
    lin = _linears(m)["model.layers.1.self_attn.o_proj"]
    lin.weight.data = lin.weight.data.to(torch.float64)
    with pytest.raises(TypeError):
        quantize_weights_fp8_(m)
    assert not any(l.fp8 for l in _linears(m).values())   # nothing converted


ACTS = [None, "gelu", "gelu_tanh", "relu", "silu", "quick_gelu"]


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("bias", [False, True])
def test_linear_fp8w_reference_fp64(act, bias):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(5, 3, 48, generator=g)
    e, s = OF.kv_cache_quantize_ref(torch.randn(24, 48, generator=g))
    b = torch.randn(24, generator=g) if bias else None
    y = OF.linear_fp8w(x, e, s, b, act)
    ref = x.double() @ (e.double() * s.double()[:, None]).T
    if bias:
        ref = ref + b.double()
    ref = {None: lambda t: t, "gelu": F.gelu, "gelu_tanh": lambda t: F.gelu(t, approximate="tanh"), "relu": F.relu,
           "silu": F.silu, "quick_gelu": lambda t: t * torch.sigmoid(1.702 * t)}[act](ref)
    assert y.shape == (5, 3, 24) and y.dtype == torch.float32
    torch.testing.assert_close(y.double(), ref, rtol=1e-5, atol=1e-5)
    xb = x.to(torch.bfloat16)   # the output has x's dtype
    assert OF.linear_fp8w(xb, e, s, None if b is None else b.to(torch.bfloat16), act).dtype == torch.bfloat16


def test_bf16_gemm_entries_reject_fp8_weights():
    from libai_b200.ops import comm_gemm, gated_mlp

    x = torch.randn(4, 32, dtype=torch.bfloat16)
    w, _ = OF.kv_cache_quantize_ref(torch.randn(32, 32))
    wb = torch.randn(32, 32, dtype=torch.bfloat16)
    calls = [
        lambda: OF.linear(x, w),
        lambda: OF.mlp(x, w, None, wb),
        lambda: OF.mlp(x, wb, None, w),
        lambda: OF.linear_bias_residual(x, w, None, x),
        lambda: gated_mlp.gated_mlp(x, w, wb, wb),
        lambda: gated_mlp.tp_gated_mlp(x, wb, wb, w, None, None),
        lambda: comm_gemm.column_parallel_linear(x, w, None, None, None),
        lambda: comm_gemm.row_parallel_linear(x, w, None, None, None),
        lambda: comm_gemm.tp_mlp(x, w, None, wb, None, None, "gelu", None),
        lambda: comm_gemm.ag_gemm(x, w, None, None, None),
        lambda: comm_gemm.gemm_rs(x, w, None, None, None),
    ]
    for call in calls:
        with pytest.raises(TypeError, match="float8_e4m3fn"):
            call()


def _dequantized_copy(model):
    """``model`` with every FP8 weight replaced by float(e)·s in fp32 (and no FP8 layers left)."""
    ref = copy.deepcopy(model)
    for l in _linears(ref).values():
        if l.fp8:
            w = l.weight.float() * l.weight_scale[:, None]
            del l.weight_scale
            l.weight = torch.nn.Parameter(w, requires_grad=False)
    return ref.float()


def test_mlp_takes_the_per_linear_path():
    from libai_b200.layers.mlp import MLP

    torch.manual_seed(0)
    mlp = MLP(32, 64).to(torch.bfloat16).eval()
    quantize_weights_fp8_(mlp)
    x = torch.randn(2, 3, 32, dtype=torch.bfloat16)
    r = torch.randn(2, 3, 32, dtype=torch.bfloat16)
    with torch.no_grad():
        y = mlp(x, residual=r)   # OF.mlp would raise on the FP8 weights
        h = OF.linear_fp8w(x, mlp.dense_h_to_4h.weight, mlp.dense_h_to_4h.weight_scale, mlp.dense_h_to_4h.bias, "gelu")
        o = OF.linear_fp8w(h, mlp.dense_4h_to_h.weight, mlp.dense_4h_to_h.weight_scale)
        ref = OF.bias_dropout_add(o, mlp.dense_4h_to_h.bias, r, 0.0, False)
    assert torch.equal(y, ref)


def test_attention_output_projection_takes_the_per_linear_path(monkeypatch):
    from libai_b200.layers.attention import AttnMaskType, MultiheadAttention

    torch.manual_seed(0)
    attn = MultiheadAttention(64, 2, attn_mask_type=AttnMaskType.causal).to(torch.bfloat16).eval()
    quantize_weights_fp8_(attn)

    def packed(qkv, *, causal, scale, **_):   # the flash fast path, computed with the reference math
        q, k, v = OF.split_qkv(qkv)
        return OF.attention_ref(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), causal=causal,
                                scale=scale).transpose(1, 2)

    monkeypatch.setattr(OF, "attention_qkvpacked_supported", lambda *a, **k: True)
    monkeypatch.setattr(OF, "attention_qkvpacked", packed)
    x = torch.randn(2, 5, 64, dtype=torch.bfloat16)
    r = torch.randn(2, 5, 64, dtype=torch.bfloat16)
    with torch.no_grad():
        y = attn(x, residual=r)   # OF.linear_bias_residual would raise on the FP8 weight
        d = attn.dense
        qkv = OF.linear_fp8w(x, attn.query_key_value.weight, attn.query_key_value.weight_scale,
                             attn.query_key_value.bias).view(2, 5, 2, 96)
        ctx = packed(qkv, causal=True, scale=attn.softmax_scale).reshape(2, 5, 64)
        ref = OF.bias_dropout_add(OF.linear_fp8w(ctx, d.weight, d.weight_scale), d.bias, r, 0.0, False)
    assert torch.equal(y, ref)


def test_gradient_raises():
    torch.manual_seed(0)
    lin = Linear1D(32, 16).to(torch.bfloat16).quantize_fp8_()
    x = torch.randn(3, 32, dtype=torch.bfloat16, requires_grad=True)
    with pytest.raises(RuntimeError, match="inference"):
        lin(x)
    with pytest.raises(RuntimeError, match="inference"):   # the bias is still a trainable parameter
        lin(x.detach())
    with torch.no_grad():
        assert lin(x).shape == (3, 16)


@pytest.mark.parametrize("cast", ["to_bf16", "bfloat16", "half", "float", "to_device_dtype"])
def test_casts_keep_bytes_and_scales(cast):
    torch.manual_seed(0)
    lin = Linear1D(32, 16).to(torch.bfloat16).quantize_fp8_()
    w, s = lin.weight.detach().clone(), lin.weight_scale.detach().clone()
    out = {"to_bf16": lambda m: m.to(torch.bfloat16), "bfloat16": lambda m: m.bfloat16(), "half": lambda m: m.half(),
           "float": lambda m: m.float(), "to_device_dtype": lambda m: m.to("cpu", torch.float16)}[cast](lin)
    assert out is lin and lin.fp8
    assert torch.equal(lin.weight.view(torch.uint8), w.view(torch.uint8)) and torch.equal(lin.weight_scale, s)
    assert lin.weight_scale.dtype == torch.float32
    want = {"to_bf16": torch.bfloat16, "bfloat16": torch.bfloat16, "half": torch.float16, "float": torch.float32,
            "to_device_dtype": torch.float16}[cast]
    assert lin.compute_dtype == want and lin.bias.dtype == want
    assert list(dict(lin.named_parameters())) == ["weight", "bias", "weight_scale"]
    with torch.no_grad():
        assert lin(torch.randn(2, 32, dtype=want)).dtype == want
    lin.to("meta")   # a device move moves the bytes and scales
    assert lin.weight.device.type == "meta" and lin.weight.dtype == E4M3 and lin.weight_scale.dtype == torch.float32


def _generate(name, m):
    ids, _ = _prompt("plain")
    with torch.no_grad():
        if name == "t5":
            return m.generate(ids, max_length=6, eos_token_id=None)
        return m.generate(ids, max_length=ids.shape[1] + 5, eos_token_id=None)


@pytest.mark.parametrize("name", list(MODELS))
def test_generate_equals_dequantized_fp32_model(name):
    m = MODELS[name]().float()
    quantize_weights_fp8_(m)
    lins = _linears(m)
    assert all(l.fp8 == (not n.endswith(HEADS)) for n, l in lins.items())
    ref = _dequantized_copy(m)
    out, want = _generate(name, m), _generate(name, ref)
    assert torch.equal(out, want)
    assert m.kv_cache.k[m.kv_cache.owned[0]].dtype == torch.float32   # the activations' dtype, not the weights'


@pytest.mark.parametrize("kv_dtype", [None, E4M3])
def test_cache_keeps_activation_dtype(kv_dtype):
    m = quantize_weights_fp8_(MODELS["llama"]())
    m.kv_cache_dtype = kv_dtype
    c = m.allocate_kv_cache(2, 16)
    assert c.dtype == torch.bfloat16
    assert c.k[c.owned[0]].dtype == (kv_dtype or torch.bfloat16)


def test_pipeline_option_rejects_unknown_dtype():
    from libai_b200.inference.basic import BasePipeline

    class P(BasePipeline):
        _parse_parameters = preprocess = forward = postprocess = None

    with pytest.raises(ValueError, match="weight_dtype"):
        P(None, weight_dtype="int8")


if __name__ == "__main__":
    sys.exit(pytest.main([__file__, "-q"]))
