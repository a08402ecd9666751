"""FP8 (E4M3) KV cache on the H100: the quantizing append against the PyTorch mirror applied to the bf16 append, the
fp8 instances of the split-KV decode kernel against fp64 over the dequantized cache (every score kind, head dim, row
mapping and split count, left padding, short windows and a window that ends one row short of the capacity), their
determinism and CUDA-graph replay, the binding's rejections, and generate(kv_cache_dtype="fp8") of every model that
decodes on the cache running natively."""
import pytest
import torch

from libai_b200.config import DictConfig
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests.test_decode_gpu import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FP8 = torch.float8_e4m3fn


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


def i32(xs):
    return torch.tensor(xs, dtype=torch.int32, device=DEV)


# ------------------------------------------------------------------------------------------------ kv_append
@pytest.mark.parametrize("rope", [False, True], ids=["plain", "rope"])
@pytest.mark.parametrize("r", [1, 4, 16])
@pytest.mark.parametrize("D", [64, 128])
def test_kv_append_fp8_matches_mirror_of_bf16_append(ext, D, r, rope):
    from libai_b200.models.llama_model import rotary_tables

    B, sq, G, C = 3, 5, 2, 64
    g = torch.Generator(device=DEV).manual_seed(D + r + rope)
    # per-head [B, sq, A, 3D] for r = 1, grouped [B, sq, G, r + 2, D] otherwise; one all-zero k row (scale 1)
    shape = (B, sq, G, 3 * D) if r == 1 else (B, sq, G, r + 2, D)
    qkv = (torch.randn(*shape, device=DEV, generator=g) * 3).bfloat16()
    if r == 1:
        qkv[0, 1, 0, D : 2 * D] = 0
    else:
        qkv[0, 1, 0, r] = 0
    cos, sin = rotary_tables(D, 128, device=DEV) if rope else (None, None)
    lens = i32([0, 7, C - sq])
    kb, vb = torch.zeros(B, G, C, D, device=DEV, dtype=torch.bfloat16), torch.zeros(B, G, C, D, device=DEV,
                                                                                     dtype=torch.bfloat16)
    q_bf = OF.kv_cache_append(qkv, kb, vb, lens, cos, sin)
    k8, v8 = torch.zeros(B, G, C, D, device=DEV, dtype=FP8), torch.zeros(B, G, C, D, device=DEV, dtype=FP8)
    ks, vs = torch.zeros(B, G, C, device=DEV), torch.zeros(B, G, C, device=DEV)
    q_8 = OF.kv_cache_append(qkv, k8, v8, lens, cos, sin, k_scale=ks, v_scale=vs)
    assert torch.equal(q_8, q_bf)
    written = torch.zeros(B, G, C, dtype=torch.bool, device=DEV)
    for b in range(B):
        written[b, :, int(lens[b]) : int(lens[b]) + sq] = True
    for cache8, scale, bf in ((k8, ks, kb), (v8, vs, vb)):
        e, s = OF.kv_cache_quantize_ref(bf)
        assert torch.equal(cache8.view(torch.uint8)[written], e.view(torch.uint8)[written])
        assert torch.equal(scale[written].view(torch.int32), s[written].view(torch.int32))
        assert not cache8.view(torch.uint8)[~written].any() and not scale[~written].any()   # nothing else written
        assert not torch.isnan(cache8.float()).any()
    assert bool((ks[0, 0, 1] == 1.0) & (k8[0, 0, 1].float() == 0).all())                  # the zero row
    # the largest element of every written row is ±448
    assert bool((k8.float()[written].abs().amax(-1)[ks[written] != 1] == 448).all())
    # without writing q
    k2, v2 = torch.zeros_like(k8), torch.zeros_like(v8)
    assert OF.kv_cache_append(qkv, k2, v2, lens, cos, sin, False, torch.zeros_like(ks), torch.zeros_like(vs)) is None
    assert torch.equal(k2.view(torch.uint8), k8.view(torch.uint8))


# ------------------------------------------------------------------------------------------------ decode_attn
KINDS = ["causal", "alibi", "rel_bias", "window"]


def _fp8_case(B, G, A, D, Sq, lens, kv_start, C, seed):
    """q (bf16), an FP8 cache quantized by the mirror from random bf16 rows, and its fp64 dequantized copy.  Rows the
    kernel never reads (at or past each sample's window end) hold NaN bytes and NaN scales."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = torch.randn(B, Sq, A, D, device=DEV, generator=g).bfloat16()
    k = (torch.randn(B, G, C, D, device=DEV, generator=g) * 2).bfloat16()
    v = torch.randn(B, G, C, D, device=DEV, generator=g).bfloat16()
    (k8, ks), (v8, vs) = OF.kv_cache_quantize_ref(k), OF.kv_cache_quantize_ref(v)
    kd = k8.double() * ks.double()[..., None]
    vd = v8.double() * vs.double()[..., None]
    return q, k8, v8, ks, vs, kd, vd


def _poison(k8, v8, ks, vs, hi):
    for b, h in enumerate(hi):
        for t in (k8, v8):
            t.view(torch.uint8)[b, :, h:] = 0x7F       # E4M3 NaN
        ks[b, :, h:] = float("nan")
        vs[b, :, h:] = float("nan")


def _ref(q, kd, vd, lens, kv_start, scale, kind, bias):
    """fp64 attention over the dequantized cache with the kernel's visibility and bias; zeros without a visible key."""
    B, Sq, A, D = q.shape
    G, C = kd.shape[1], kd.shape[2]
    kd, vd = kd.repeat_interleave(A // G, dim=1), vd.repeat_interleave(A // G, dim=1)
    j = torch.arange(C, device=DEV)[None, None, :]
    i = torch.arange(Sq, device=DEV)[None, :, None]
    end = lens.long()[:, None, None] - 1 if kind == "window" else lens.long()[:, None, None] + i
    vis = ((j >= kv_start.long()[:, None, None]) & (j <= end))[:, None]                     # [B, 1, Sq, C]
    s = torch.einsum("bqhd,bhkd->bhqk", q.double(), kd) * scale
    if kind == "alibi":
        s = s + bias.double()[None, :, None, None] * (j - lens.long()[:, None, None] - i).double()[:, None]
    elif kind == "rel_bias":
        dist_ = (lens.long()[:, None, None] + i - j).clamp(0, bias.shape[1] - 1)                # [B, Sq, C]
        s = s + bias.double()[:, dist_].permute(1, 0, 2, 3)
    s = s.masked_fill(~vis, float("-inf"))
    p = torch.softmax(s, dim=-1).nan_to_num(0.0)
    return torch.einsum("bhqk,bhkd->bqhd", p, vd)


def _run(ext, q, k8, v8, ks, vs, lens, kv_start, scale, splits, kind, bias):
    extra = dict(causal=kind != "window", k_scale=ks, v_scale=vs)
    if kind == "alibi":
        extra["alibi_slopes"] = bias
    if kind == "rel_bias":
        extra["rel_bias"] = bias
    return ext.decode_attn(q, k8, v8, lens, kv_start, scale, splits, **extra)


def _bias(kind, A, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    if kind == "alibi":
        from projects.BLOOM.modeling.bloom_model import alibi_slopes

        return alibi_slopes(A).to(DEV)
    if kind == "rel_bias":
        return torch.randn(A, 33, device=DEV, generator=g)
    return None


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("sq_r", [(1, 1), (4, 4), (16, 1), (1, 16), (4, 16)], ids=lambda t: f"sq{t[0]}_r{t[1]}")
def test_decode_fp8_matches_fp64_over_dequantized_cache(ext, kind, D, sq_r):
    """Four samples: a long window, a left-padded one, one shorter than a tile, and one ending one row short of the
    capacity (its last tile's copies are clipped there).  Tolerance: that of the bf16 kernel's test or tighter."""
    Sq, r = sq_r
    G, B, C = 2, 4, 1104                  # the capacity a multiple of 4, as an FP8 StaticKVCache rounds it
    A = G * r
    short_end = C - 1                     # the window end hi of the last sample
    lens = i32([1000, 300, 5, short_end if kind == "window" else short_end - Sq])
    kv_start = i32([0, 37, 0, 3])
    seed = D * 7 + Sq * 31 + r + KINDS.index(kind) * 1000
    q, k8, v8, ks, vs, kd, vd = _fp8_case(B, G, A, D, Sq, lens, kv_start, C, seed)
    hi = [int(x) + (0 if kind == "window" else Sq) for x in lens.tolist()]
    _poison(k8, v8, ks, vs, hi)
    kd = torch.nan_to_num(kd, 0.0)
    vd = torch.nan_to_num(vd, 0.0)
    bias = _bias(kind, A, seed)
    scale = D ** -0.5
    want = _ref(q, kd, vd, lens, kv_start, scale, kind, bias)
    errs = {}
    for splits in (1, 3, 32, 0):
        o = _run(ext, q, k8, v8, ks, vs, lens, kv_start, scale, splits, kind, bias)
        assert o.shape == (B, Sq, A, D) and o.is_contiguous()
        assert not torch.isnan(o).any()
        errs[splits] = max(rel_err(o[b], want[b]) for b in range(B))
    bad = {s: e for s, e in errs.items() if not e < 1e-2}
    assert not bad, errs


@pytest.mark.parametrize("kind", KINDS)
def test_decode_fp8_no_visible_key_writes_zeros(ext, kind):
    B, G, A, D, Sq, C = 2, 2, 8, 64, 4, 256
    lens = i32([100, 60])
    q, k8, v8, ks, vs, _, _ = _fp8_case(B, G, A, D, Sq, lens, lens, C, seed=5)
    start = (lens + Sq).contiguous()      # beyond the last key of every query
    for splits in (0, 1):
        o = _run(ext, q, k8, v8, ks, vs, lens, start, 0.125, splits, kind, _bias(kind, A, 1))
        assert torch.equal(o, torch.zeros_like(o))


def test_decode_fp8_is_bit_identical_between_calls_and_after_graph_replay(ext):
    B, G, A, D, Sq, C = 3, 2, 8, 128, 4, 4400
    lens = i32([4000, 3000, 17])
    kv_start = i32([0, 11, 0])
    q, k8, v8, ks, vs, _, _ = _fp8_case(B, G, A, D, Sq, lens, kv_start, C, seed=9)
    a = OF.decode_attention(q, k8, v8, lens, kv_start, scale=0.1, k_scale=ks, v_scale=vs)
    b = OF.decode_attention(q, k8, v8, lens, kv_start, scale=0.1, k_scale=ks, v_scale=vs)
    assert torch.equal(a, b)
    lens = i32([500, 200, 17])
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = OF.decode_attention(q, k8, v8, lens, kv_start, scale=0.1, k_scale=ks, v_scale=vs)
    lens.add_(300)                        # on the device, as StaticKVCache.advance does
    graph.replay()
    eager = OF.decode_attention(q, k8, v8, lens, kv_start, scale=0.1, k_scale=ks, v_scale=vs)
    assert torch.equal(out, eager)
    del graph


def test_binding_rejects_bad_scales(ext):
    B, G, A, D, Sq, C = 2, 2, 4, 64, 1, 128
    lens, start = i32([10, 20]), i32([0, 0])
    q, k8, v8, ks, vs, _, _ = _fp8_case(B, G, A, D, Sq, lens, start, C, seed=3)
    qkv = torch.randn(B, 1, A, 3 * D, device=DEV).bfloat16()
    bad = [None, ks.double(), ks[:, :, :64], ks.transpose(0, 1).contiguous().transpose(0, 1), ks.cpu()]
    for s in bad:
        with pytest.raises((RuntimeError, TypeError)):
            ext.decode_attn(q, k8, v8, lens, start, 0.1, 0, None, None, True, s, vs)
        if s is not None:
            with pytest.raises((RuntimeError, TypeError)):
                ext.kv_append_fp8(qkv, k8, v8, s, vs, lens, None, None, True)
    # scales with a bf16 cache; a capacity that is not a multiple of 4
    kb = torch.zeros(B, G, C, D, device=DEV, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):
        ext.decode_attn(q, kb, kb, lens, start, 0.1, 0, None, None, True, ks, vs)
    k_odd, s_odd = k8[:, :, :126].contiguous(), ks[:, :, :126].contiguous()
    with pytest.raises(RuntimeError):
        ext.decode_attn(q, k_odd, k_odd, lens, start, 0.1, 0, None, None, True, s_odd, s_odd)
    with pytest.raises(ValueError):
        OF.decode_attention(q, k8, v8, lens, start, scale=0.1)


# ------------------------------------------------------------------------------------------------ generate()
@pytest.fixture
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    with torch.random.fork_rng(devices=[0]):
        yield


def _model(name):
    from tests.test_cached_attention_cpu import MODELS

    m = MODELS[name]().to(DEV)
    if name == "t5":
        # its builder's initializer range of 0.5 and T5's unscaled scores make the logits chaotic: bf16 rounding alone
        # moves them by 5 % of their largest value between the native and the reference path
        with torch.no_grad():
            for p in m.parameters():
                p.mul_(0.2)
    return m


class _Recorder:
    def __init__(self, ext):
        self.ext, self.calls = ext, []

    def __getattr__(self, name):
        fn = getattr(self.ext, name)
        if name in ("kv_append", "kv_append_fp8", "decode_attn"):
            def wrapped(*a, **k):
                fp8 = name == "kv_append_fp8" or (name == "decode_attn" and len(a) > 10 and a[10] is not None)
                self.calls.append((name, fp8))
                return fn(*a, **k)
            return wrapped
        return fn


def _refuse(*a, **k):
    raise AssertionError("a cached step ran the reference decode attention or cache append")


NAMES = ["llama", "llama_gqa", "gpt2", "bloom", "chatglm", "chatglm_prefix", "t5"]


@pytest.mark.parametrize("name", NAMES)
def test_generate_fp8_runs_native(_topo, ext, monkeypatch, name):
    m = _model(name)
    rec = _Recorder(ext)
    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: rec)
    monkeypatch.setattr(OF, "decode_attention_ref", _refuse)
    monkeypatch.setattr(OF, "kv_cache_append_ref", _refuse)
    ids = torch.randint(3, 100, (3, 7), generator=torch.Generator().manual_seed(1)).to(DEV)
    with torch.no_grad():
        if name == "t5":
            out = m.generate(ids, max_length=6, eos_token_id=None, kv_cache_dtype="fp8")
        else:
            out = m.generate(ids, max_length=13, eos_token_id=None, kv_cache_dtype="fp8")
    assert out.shape[0] == 3
    assert m.kv_cache.kv_dtype == FP8 and m.kv_cache_dtype is None   # the option held for the call only
    if name == "t5":
        assert m.cross_cache.kv_dtype == FP8
    names = {c for c in rec.calls}
    assert ("kv_append_fp8", True) in names and ("decode_attn", True) in names, names
    assert ("kv_append", False) not in names and ("decode_attn", False) not in names, names


def _teacher_forced(m, name):
    """Logits of a prompt, three single steps, a 4-token step and an 18-token continuation on an FP8 cache."""
    ids = torch.randint(3, 100, (3, 7), generator=torch.Generator().manual_seed(1)).to(DEV)
    more = torch.randint(3, 100, (3, 26), generator=torch.Generator().manual_seed(3)).to(DEV)
    chunks = [(0, 1), (1, 2), (2, 3), (3, 7), (7, 25)]
    m.kv_cache_dtype = FP8
    out = []
    with torch.no_grad():
        if name == "t5":
            m.allocate_kv_cache(3, 26)
            out.append(m(ids, more[:, :1], None, use_cache=True)["logits"])
            for lo, hi in chunks:
                out.append(m(ids, more[:, 1 + lo : 1 + hi], None, use_cache=True)["logits"])
        else:
            m.allocate_kv_cache(3, 32)
            out.append(m(ids, use_cache=True)["logits"])
            for lo, hi in chunks:
                out.append(m(more[:, lo:hi], use_cache=True)["logits"])
    m.kv_cache_dtype = None
    m.set_cache(None) if name != "t5" else m.set_cache(None, None)
    return torch.cat(out, dim=1).float()


@pytest.mark.parametrize("name", NAMES)
def test_teacher_forced_fp8_logits_match_dequantized_reference(_topo, monkeypatch, name):
    """The native kernels on an FP8 cache against the reference append and attention over the same format (the window
    dequantized); tolerance that of the bf16 generate() tests.  The two paths may store different bytes where the
    kernel's fp32 rotation and the reference's bf16 one round a k element differently."""
    m = _model(name)
    got = _teacher_forced(m, name)
    monkeypatch.setattr(OF, "_decode_native", lambda *a: False)
    want = _teacher_forced(m, name)
    assert rel_err(got, want) < 3e-2, rel_err(got, want)
