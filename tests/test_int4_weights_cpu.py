"""Group-wise INT4 weights for inference without a GPU: the quantizer against an independent NumPy implementation of
its rule, the packed layout, the reference math of ``OF.linear_int4w``, the refusals, dtype casts, the guards of the bf16
GEMM entries, the per-``Linear`` paths, ``generate()`` of every cache model against the same model holding Ŵ in fp32,
the pipeline option and the bindings' argument checks."""
import copy
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from libai_b200.config import DictConfig
from libai_b200.inference import quantize_weights_fp8_, quantize_weights_int4_
from libai_b200.layers.linear import Linear1D
from libai_b200.ops import build as ops_build
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist

from tests import op_args_cases as C
from tests.test_cached_attention_cpu import MODELS, _prompt

HEADS = ("lm_head", "output_layer")
U8 = torch.uint8


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cpu")))


def _linears(model):
    return {n: m for n, m in model.named_modules() if isinstance(m, Linear1D)}


# ------------------------------------------------------------------------------------------------ the rule
def _bf16_rn(a):
    """float32 array -> the float32 values of its bf16 round-to-nearest-even (finite inputs)."""
    b = np.asarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(np.float32)


def _quantize_np(w):
    """The rule in NumPy: fp32 IEEE divisions, bf16 scale, half-to-even rounding; returns unpacked q [N, K], s, z."""
    N, K = w.shape
    g = np.asarray(w, dtype=np.float32).reshape(N, K // 128, 128)
    lo = np.minimum(g.min(-1), np.float32(0))
    hi = np.maximum(g.max(-1), np.float32(0))
    s = _bf16_rn(np.float32(hi - lo) / np.float32(15))
    s = np.where(s < np.float32(2.0 ** -126), np.float32(1), s).astype(np.float32)
    z = np.clip(np.round(np.float32(-lo) / s), 0, 15)
    q = np.clip(np.round(g / s[..., None]) + z[..., None], 0, 15)
    return q.reshape(N, K).astype(np.int64), s, z.astype(np.int64)


def _unpack(packed):
    p = packed.numpy().astype(np.int64)
    return np.stack([p & 15, p >> 4], -1).reshape(p.shape[0], -1)


def _special_rows():
    """Rows of 2 groups each that reach the rule's corners."""
    rows = torch.randn(12, 256, generator=torch.Generator().manual_seed(0))
    rows[0] = 0                                    # all-zero groups: s = 1, z = 0, q = 0
    rows[1] = rows[1].abs() + 0.1                  # positive groups: lo = 0, z = 0
    rows[2] = -(rows[2].abs() + 0.1)               # negative groups: hi = 0, z = 15
    rows[3] = rows[3] * 1e-40                      # (hi − lo) / 15 subnormal: s = 1
    rows[4, :128] = 2e-37                          # a scale just past the subnormal boundary in one group
    rows[5] = torch.linspace(-1, 2, 256)           # wide range: q hits both clamps after the scale's rounding
    # ties: s = 1/16 exactly (hi − lo = 15/16), values k/16 + 1/32 sit on a half step
    t = torch.arange(128, dtype=torch.float32) % 15 / 16 - 7 / 16 + 1 / 32
    rows[6, :128] = t
    rows[6, 0], rows[6, 1] = -7 / 16, 8 / 16
    rows[7] = rows[7] * 1e4                        # large values
    rows[8] = torch.tensor([-3.0, 3.0]).repeat(128)
    return rows


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_quantizer_matches_numpy_rule(dtype):
    w = torch.cat([_special_rows(), torch.randn(20, 256, generator=torch.Generator().manual_seed(1)) * 0.05]).to(dtype)
    packed, s, z = OF.int4_quantize_ref(w)
    assert packed.dtype == U8 and packed.shape == (32, 128)
    assert s.dtype == torch.bfloat16 and s.shape == (32, 2) and z.dtype == U8 and z.shape == (32, 2)
    q_np, s_np, z_np = _quantize_np(w.float().numpy())
    assert np.array_equal(_unpack(packed), q_np)
    assert np.array_equal(s.float().numpy(), s_np)
    assert np.array_equal(z.numpy().astype(np.int64), z_np)
    if dtype != torch.float32:
        return
    # the corners were reached
    assert (s[0] == 1).all() and (z[0] == 0).all() and (_unpack(packed)[0] == 0).all()
    assert (z[1] == 0).all() and (z[2] == 15).all() and (s[3] == 1).all()
    assert s[4, 0].item() > 0 and s[4, 0].item() != 1
    tie = w[6, 2:128].float().numpy() / s_np[6, 0]
    assert np.any(np.abs(tie - np.floor(tie) - 0.5) == 0)


def test_clamp_is_reached():
    # s = bf16_rn((hi − lo) / 15) may round down, so that round(hi / s) + z passes 15 and is clamped
    w = torch.zeros(1, 128)
    w[0, 0], w[0, 1] = -0.99950475, 1.0   # s = 0.1328125, z = 8: round(1 / s) + z = 16
    packed, s, z = OF.int4_quantize_ref(w)
    q_np, s_np, z_np = _quantize_np(w.numpy())
    raw = np.round(w.numpy()[0, 1] / s_np[0, 0]) + z_np[0, 0]
    assert raw > 15 and _unpack(packed)[0, 1] == 15 == q_np[0, 1]


def test_nibble_order():
    q = torch.tensor([[3, 12] + [0] * 126], dtype=torch.float32)   # s = 1: w = q − z with z = 0
    q[0, 2] = 15
    packed, s, z = OF.int4_quantize_ref(q)
    assert s[0, 0] == 1 and z[0, 0] == 0
    assert packed[0, 0].item() == 3 | (12 << 4) and packed[0, 1].item() == 15


def test_dequant_ref_is_the_formula():
    w = torch.randn(8, 384, generator=torch.Generator().manual_seed(2))
    packed, s, z = OF.int4_quantize_ref(w)
    got = OF.int4_dequant_ref(packed, s, z)
    q = torch.from_numpy(_unpack(packed)).double()
    want = (q - z.double().repeat_interleave(128, 1)) * s.double().repeat_interleave(128, 1)
    assert got.dtype == torch.bfloat16 and got.shape == (8, 384)
    assert torch.equal(got, want.to(torch.bfloat16))   # the fp64 product is exact, so one rounding either way
    # half a step from rounding w / s, at most half a step more from rounding the zero point
    assert bool(((got.float() - w).abs() <= s.float().repeat_interleave(128, 1)).all())


ACTS = [None, "gelu", "gelu_tanh", "relu", "silu", "quick_gelu"]


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("bias", [False, True])
def test_linear_int4w_reference_fp64(act, bias):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(5, 3, 256, generator=g)
    packed, s, z = OF.int4_quantize_ref(torch.randn(24, 256, generator=g))
    b = torch.randn(24, generator=g) if bias else None
    y = OF.linear_int4w(x, packed, s, z, b, act)
    ref = x.double() @ OF.int4_dequant_ref(packed, s, z).double().T
    if bias:
        ref = ref + b.double()
    ref = {None: lambda t: t, "gelu": F.gelu, "gelu_tanh": lambda t: F.gelu(t, approximate="tanh"), "relu": F.relu,
           "silu": F.silu, "quick_gelu": lambda t: t * torch.sigmoid(1.702 * t)}[act](ref)
    assert y.shape == (5, 3, 24) and y.dtype == torch.float32
    torch.testing.assert_close(y.double(), ref, rtol=1e-5, atol=1e-5)
    xb = x.to(torch.bfloat16)
    assert OF.linear_int4w(xb, packed, s, z, None if b is None else b.to(torch.bfloat16), act).dtype == torch.bfloat16


# ------------------------------------------------------------------------------------------------ the layers
def test_quantize_weights_int4_converts_every_linear_but_the_heads():
    m = MODELS["llama"]()
    lins = _linears(m)
    before = {n: l.weight.detach().clone() for n, l in lins.items()}
    head = lins["lm_head"].weight
    assert quantize_weights_int4_(m) is m
    for n, l in lins.items():
        if n == "lm_head":
            assert l.weight is head and not l.quantized
            continue
        q, s, z = OF.int4_quantize_ref(before[n])
        assert l.int4 and l.quantized and not l.fp8 and l.compute_dtype == torch.bfloat16
        assert torch.equal(l.weight, q) and torch.equal(l.weight_scale, s) and torch.equal(l.weight_zero, z)
        assert l.weight.shape == (before[n].shape[0], before[n].shape[1] // 2)
        assert not any(p.requires_grad for p in (l.weight, l.weight_scale, l.weight_zero))
        assert "weight=int4" in repr(l)
    snap = {n: (l.weight, getattr(l, "weight_scale", None), getattr(l, "weight_zero", None)) for n, l in lins.items()}
    quantize_weights_int4_(m)   # a second call changes nothing
    assert all((l.weight, getattr(l, "weight_scale", None), getattr(l, "weight_zero", None)) == snap[n]
               for n, l in lins.items())


def _refused(mutate, exc):
    m = MODELS["llama"]()
    mutate(_linears(m))
    with pytest.raises(exc):
        quantize_weights_int4_(m)
    assert not any(l.quantized for l in _linears(m).values())   # nothing converted
    return m


def test_refusals_convert_nothing():
    def dtype(lins):
        lins["model.layers.1.self_attn.o_proj"].weight.data = lins["model.layers.1.self_attn.o_proj"].weight.data.double()

    def width(lins):
        lins["model.layers.1.mlp.down_proj"] = l = lins["model.layers.1.mlp.down_proj"]
        l.weight.data = l.weight.data[:, :96].contiguous()

    def nonfinite(lins):
        lins["model.layers.1.mlp.up_proj"].weight.data[3, 7] = float("nan")

    _refused(dtype, TypeError)
    _refused(width, ValueError)
    _refused(nonfinite, ValueError)
    with pytest.raises(ValueError, match="non-finite"):
        OF.int4_quantize_ref(torch.full((1, 128), float("inf")))
    with pytest.raises(ValueError):
        OF.int4_quantize_ref(torch.zeros(2, 96))


def test_fp8_and_int4_layers_refuse_each_other():
    m = quantize_weights_fp8_(MODELS["llama"]())
    with pytest.raises(TypeError, match="float8_e4m3fn"):
        quantize_weights_int4_(m)
    assert not any(l.int4 for l in _linears(m).values())
    m = quantize_weights_int4_(MODELS["llama"]())
    with pytest.raises(TypeError, match="uint8"):
        quantize_weights_fp8_(m)
    with pytest.raises(TypeError):
        _linears(m)["model.layers.0.mlp.up_proj"].quantize_fp8_()


def test_gradient_raises():
    torch.manual_seed(0)
    lin = Linear1D(128, 16).to(torch.bfloat16).quantize_int4_()
    x = torch.randn(3, 128, dtype=torch.bfloat16, requires_grad=True)
    with pytest.raises(RuntimeError, match="inference"):
        lin(x)
    with pytest.raises(RuntimeError, match="inference"):   # the bias is still a trainable parameter
        lin(x.detach())
    with torch.no_grad():
        assert lin(x).shape == (3, 16)


@pytest.mark.parametrize("cast", ["to_bf16", "bfloat16", "half", "float", "to_device_dtype"])
def test_casts_keep_bytes_scales_and_zeros(cast):
    torch.manual_seed(0)
    lin = Linear1D(256, 16).to(torch.bfloat16).quantize_int4_()
    w, s, z = (lin.weight.detach().clone(), lin.weight_scale.detach().clone(), lin.weight_zero.detach().clone())
    out = {"to_bf16": lambda m: m.to(torch.bfloat16), "bfloat16": lambda m: m.bfloat16(), "half": lambda m: m.half(),
           "float": lambda m: m.float(), "to_device_dtype": lambda m: m.to("cpu", torch.float16)}[cast](lin)
    assert out is lin and lin.int4
    assert torch.equal(lin.weight, w) and torch.equal(lin.weight_scale, s) and torch.equal(lin.weight_zero, z)
    assert lin.weight_scale.dtype == torch.bfloat16 and lin.weight_zero.dtype == U8
    want = {"to_bf16": torch.bfloat16, "bfloat16": torch.bfloat16, "half": torch.float16, "float": torch.float32,
            "to_device_dtype": torch.float16}[cast]
    assert lin.compute_dtype == want and lin.bias.dtype == want
    assert list(dict(lin.named_parameters())) == ["weight", "bias", "weight_scale", "weight_zero"]
    with torch.no_grad():
        assert lin(torch.randn(2, 256, dtype=want)).dtype == want
    lin.to("meta")   # a device move moves all three
    assert all(t.device.type == "meta" for t in (lin.weight, lin.weight_scale, lin.weight_zero))
    assert lin.weight.dtype == U8 and lin.weight_scale.dtype == torch.bfloat16 and lin.weight_zero.dtype == U8


def test_bf16_gemm_entries_reject_int4_weights():
    from libai_b200.ops import comm_gemm, gated_mlp

    x = torch.randn(4, 256, dtype=torch.bfloat16)
    w, _, _ = OF.int4_quantize_ref(torch.randn(256, 256))
    wb = torch.randn(256, 256, dtype=torch.bfloat16)
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
        with pytest.raises(TypeError, match="OF.linear_int4w"):
            call()


def test_mlp_takes_the_per_linear_path():
    from libai_b200.layers.mlp import MLP

    torch.manual_seed(0)
    mlp = MLP(128, 256).to(torch.bfloat16).eval()
    quantize_weights_int4_(mlp)
    x = torch.randn(2, 3, 128, dtype=torch.bfloat16)
    r = torch.randn(2, 3, 128, dtype=torch.bfloat16)
    a, b = mlp.dense_h_to_4h, mlp.dense_4h_to_h
    with torch.no_grad():
        y = mlp(x, residual=r)   # OF.mlp would raise on the INT4 weights
        h = OF.linear_int4w(x, a.weight, a.weight_scale, a.weight_zero, a.bias, "gelu")
        o = OF.linear_int4w(h, b.weight, b.weight_scale, b.weight_zero)
        ref = OF.bias_dropout_add(o, b.bias, r, 0.0, False)
    assert torch.equal(y, ref)


def test_attention_output_projection_takes_the_per_linear_path(monkeypatch):
    from libai_b200.layers.attention import AttnMaskType, MultiheadAttention

    torch.manual_seed(0)
    attn = MultiheadAttention(128, 2, attn_mask_type=AttnMaskType.causal).to(torch.bfloat16).eval()
    quantize_weights_int4_(attn)

    def packed(qkv, *, causal, scale, **_):   # the flash fast path, computed with the reference math
        q, k, v = OF.split_qkv(qkv)
        return OF.attention_ref(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), causal=causal,
                                scale=scale).transpose(1, 2)

    monkeypatch.setattr(OF, "attention_qkvpacked_supported", lambda *a, **k: True)
    monkeypatch.setattr(OF, "attention_qkvpacked", packed)
    x = torch.randn(2, 5, 128, dtype=torch.bfloat16)
    r = torch.randn(2, 5, 128, dtype=torch.bfloat16)
    qkv_l, d = attn.query_key_value, attn.dense
    with torch.no_grad():
        y = attn(x, residual=r)   # OF.linear_bias_residual would raise on the INT4 weight
        qkv = OF.linear_int4w(x, qkv_l.weight, qkv_l.weight_scale, qkv_l.weight_zero, qkv_l.bias).view(2, 5, 2, 192)
        ctx = packed(qkv, causal=True, scale=attn.softmax_scale).reshape(2, 5, 128)
        ref = OF.bias_dropout_add(OF.linear_int4w(ctx, d.weight, d.weight_scale, d.weight_zero), d.bias, r, 0.0, False)
    assert torch.equal(y, ref)


def _ref_copy(model):
    """``model`` with every INT4 weight replaced by Ŵ in fp32 (and no INT4 layers left)."""
    ref = copy.deepcopy(model)
    for l in _linears(ref).values():
        if l.int4:
            w = OF.int4_dequant_ref(l.weight, l.weight_scale, l.weight_zero).float()
            del l.weight_scale, l.weight_zero
            l.weight = torch.nn.Parameter(w, requires_grad=False)
    return ref.float()


def _generate(name, m):
    ids, _ = _prompt("plain")
    with torch.no_grad():
        if name == "t5":
            return m.generate(ids, max_length=6, eos_token_id=None)
        return m.generate(ids, max_length=ids.shape[1] + 5, eos_token_id=None)


@pytest.mark.parametrize("name", list(MODELS))
def test_generate_equals_dequantized_fp32_model(name):
    m = MODELS[name]().float()
    quantize_weights_int4_(m)
    lins = _linears(m)
    assert all(l.int4 == (not n.endswith(HEADS)) for n, l in lins.items())
    ref = _ref_copy(m)
    out, want = _generate(name, m), _generate(name, ref)
    assert torch.equal(out, want)
    assert m.kv_cache.k[m.kv_cache.owned[0]].dtype == torch.float32   # the activations' dtype, not the weights'


@pytest.mark.parametrize("kv_dtype", [None, torch.float8_e4m3fn])
def test_cache_keeps_activation_dtype(kv_dtype):
    m = quantize_weights_int4_(MODELS["llama"]())
    m.kv_cache_dtype = kv_dtype
    c = m.allocate_kv_cache(2, 16)
    assert c.dtype == torch.bfloat16
    assert c.k[c.owned[0]].dtype == (kv_dtype or torch.bfloat16)


def test_pipeline_option(monkeypatch):
    from libai_b200 import inference
    from libai_b200.inference.basic import BasePipeline

    class P(BasePipeline):
        _parse_parameters = preprocess = forward = postprocess = None

    with pytest.raises(ValueError, match="'int4'"):
        P(None, weight_dtype="int8")
    seen = []
    monkeypatch.setattr(inference, "quantize_weights_int4_", lambda model: seen.append(model))
    monkeypatch.setattr(BasePipeline, "update_cfg", lambda self, *a: None)
    monkeypatch.setattr(BasePipeline, "load_pretrain_weight", lambda self, *a, **k: torch.nn.Linear(2, 2))
    monkeypatch.setattr(BasePipeline, "_place", lambda self, model: model)
    monkeypatch.setattr(BasePipeline, "build_tokenizer", lambda self, cfg: None)
    monkeypatch.setattr(P, "_parse_parameters", lambda self, **kw: ({}, {}, {}), raising=False)
    cfg = DictConfig(dict(train=DictConfig(dict(dist=DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1,
                                                                          pipeline_parallel_size=1)))),
                          model=DictConfig(dict())))
    p = P(cfg, mode="random", device="cpu", weight_dtype="int4")
    assert seen == [p.model]


# ------------------------------------------------------------------------------------------------ the bindings
def int4_cases(dev):
    """Argument cases of the INT4 ops, in the form of ``tests/op_args_cases.py``."""
    g = torch.Generator().manual_seed(0)

    def r(*shape, dtype=torch.bfloat16):
        return torch.randn(*shape, generator=g).to(dtype).to(dev)

    def u8(*shape, hi=256):
        return torch.randint(0, hi, shape, generator=g, dtype=U8).to(dev)

    return [
        C._c("linear_int4w", dict(x=r(4, 256), w=u8(128, 128), w_scale=r(128, 2).abs(), w_zero=u8(128, 2, hi=16),
                                  bias=r(128), act=0),
             ["x:dtype=float32", "x:misalign", "x:noncontig", "w:misalign", "w:narrow", "w:dtype=int8", "w:device",
              "w_scale:short", "w_scale:narrow", "w_scale:dtype=float32", "w_scale:device", "w_zero:dtype=int32",
              "w_zero:narrow", "w_zero:noncontig", "w_zero:device", "bias:short", "bias:dtype=float32",
              "bias:device"], [(4, 128)]),
        C._c("dequant_int4_rows", dict(w=u8(128, 128), w_scale=r(128, 2).abs(), w_zero=u8(128, 2, hi=16)),
             ["w:noncontig", "w:narrow", "w:misalign", "w_scale:dtype=float32", "w_scale:short", "w_zero:short",
              "w_zero:dtype=int8", "w_zero:device"], [(128, 256)]),
    ]


CASES = int4_cases("cpu")
MUTATIONS = [(c, m) for c in CASES for m in c.mutations]


@pytest.fixture(scope="module")
def ext():
    if not os.path.exists(ops_build.NVCC):
        pytest.skip("needs nvcc to build the extension")
    torch.ops.load_library(ops_build.build(force=False))
    return torch.ops.libai_b200


def _error(fn):
    with pytest.raises(RuntimeError) as e:
        fn()
    return str(e.value).splitlines()[0]


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_valid_arguments_fail_only_for_not_being_on_a_cuda_device(ext, case):
    msg = _error(lambda: getattr(ext, case.op)(*case.values()))
    assert msg.startswith(f"{case.op}: ") and "must be a CUDA tensor" in msg, msg


@pytest.mark.parametrize("case,mutation", MUTATIONS, ids=[f"{c.id}-{n}-{k}" for c, (n, k, _) in MUTATIONS])
def test_each_mutation_is_rejected_by_its_own_rule(ext, case, mutation):
    name, kind, fragment = mutation
    msg = _error(lambda: getattr(ext, case.op)(*C.mutated(case, name, kind, "meta")))
    assert fragment in msg, msg
    assert "must be a CUDA tensor" not in msg, msg


def test_rows_and_activation_are_checked(ext):
    case = CASES[0]
    args = dict(case.args)
    for x, act in ((torch.zeros(65, 256, dtype=torch.bfloat16), 0), (torch.zeros(0, 256, dtype=torch.bfloat16), 0),
                   (args["x"], 6), (args["x"][:, :128].contiguous(), 0)):
        msg = _error(lambda: ext.linear_int4w(x, args["w"], args["w_scale"], args["w_zero"], args["bias"], act))
        assert msg.startswith("linear_int4w: ") and "must be a CUDA tensor" not in msg, msg


if __name__ == "__main__":
    sys.exit(pytest.main([__file__, "-q"]))
