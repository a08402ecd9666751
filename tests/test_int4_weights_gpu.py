"""INT4 weights on the H100: the weight-streaming kernel against fp64 over Ŵ, its determinism, CUDA-graph replay and
batch invariance, the dequantize + bf16 GEMM path for larger M, the bindings' rejections, generate() and teacher-forced
logits of every cache model with INT4 weights, Llama's fused paths declining them, and decode graphs on INT4 weights."""
import pytest
import torch
import torch.nn.functional as F

from libai_b200.config import DictConfig
from libai_b200.inference import quantize_weights_int4_
from libai_b200.layers.linear import Linear1D
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests import op_args_cases as C
from tests.test_decode_gpu import rel_err
from tests.test_int4_weights_cpu import int4_cases

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U8 = torch.uint8
ACT = {None: 0, "gelu": OF.ACT_GELU, "silu": OF.ACT_SILU}
T = OF.INT4W_KERNEL_MAX_M


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


def _case(M, N, K, bias, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, K, device=DEV, generator=g).bfloat16()
    q, s, z = OF.int4_quantize_ref(torch.randn(N, K, device=DEV, generator=g) * 0.05)
    b = (torch.randn(N, device=DEV, generator=g) * 0.5).bfloat16() if bias else None
    return x, (q, s, z), b


def _ref64(x, w, b, act):
    wf = OF.int4_dequant_ref(*w).double()
    y = x.double() @ wf.T
    if b is not None:
        y = y + b.double()
    y = {None: lambda t: t, "gelu": F.gelu, "silu": F.silu}[act](y)
    return y, x.double().abs() @ wf.abs().T   # the result and the sum of |terms| of each dot product


def _check(y, x, w, b, act, K):
    ref, mag = _ref64(x, w, b, act)
    # bf16 rounding of the output, fp32 accumulation over K terms (and the activation's fast math); the tolerance of
    # the FP8-weight kernel's test
    err = (y.double() - ref).abs()
    tol = 2.0 ** -8 * ref.abs() + 2e-6 * mag * (1 + K / 1024) + 1e-5
    assert bool((err <= tol).all()), float((err - tol).max())


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("K", [128, 1024, 11008])
@pytest.mark.parametrize("M", [1, 2, 7, 8, 9, 16, 33, 64])
@pytest.mark.parametrize("epi", [(False, None), (True, "gelu"), (True, "silu")], ids=["plain", "bias_gelu", "bias_silu"])
def test_kernel_matches_fp64(ext, M, K, epi):
    bias, act = epi
    N = 200 + 4096 * (K == 1024)   # not a multiple of the 64-row block
    x, w, b = _case(M, N, K, bias, seed=M * 7 + K)
    y = ext.linear_int4w(x, *w, b, ACT[act])
    assert y.dtype == torch.bfloat16 and y.shape == (M, N)
    _check(y, x, w, b, act, K)


def _split_of(N, K):
    """(splits, range) of ``split_of`` in weight_stream.cuh for the INT4 kernel: 64-row blocks, ranges of at least 256
    columns in 128-column steps (whole groups), enough splits for 4 · 132 CTAs."""
    row_blocks = -(-N // 64)
    splits = min(max(-(-528 // row_blocks), 1), -(-K // 256))
    rng = -(-(-(-K // splits)) // 128) * 128
    return -(-K // rng), rng


# (N, K) -> (splits, range): the paths test_kernel_matches_fp64 does not reach
SPLIT_SHAPES = {
    (37888, 3584): (1, 3584),   # one range: the direct-write epilogue at a real K (Qwen2-7B's packed gate/up)
    (4096, 4352): (9, 512),     # the last range holds 256 columns
    (63, 1152): (5, 256),       # the last range holds one group; one partial row block
    (1, 4096): (16, 256),       # fewer than 16 weight rows: lanes without a valid row
    (8, 4096): (16, 256),
}


@pytest.mark.parametrize("NK", list(SPLIT_SHAPES), ids=[f"N{n}_K{k}" for n, k in SPLIT_SHAPES])
@pytest.mark.parametrize("epi", [(False, None), (True, "silu")], ids=["plain", "bias_silu"])
def test_kernel_split_shapes_match_fp64(ext, NK, epi):
    N, K = NK
    assert _split_of(N, K) == SPLIT_SHAPES[NK]
    bias, act = epi
    x, w, b = _case(64, N, K, bias, seed=N + K)
    full = ext.linear_int4w(x, *w, b, ACT[act])
    for M in (1, 9, 33, 64):
        y = full if M == 64 else ext.linear_int4w(x[:M].contiguous(), *w, b, ACT[act])
        assert y.dtype == torch.bfloat16 and y.shape == (M, N)
        _check(y, x[:M], w, b, act, K)
        if NK == (37888, 3584):   # batch invariance on the direct-write path, at the first and the last rows
            assert torch.equal(y, full[:M]), M
            tail = ext.linear_int4w(x[64 - M :].contiguous(), *w, b, ACT[act])
            assert torch.equal(tail, full[64 - M :]), M


def test_kernel_is_deterministic_graph_safe_and_batch_invariant(ext):
    N, K = 4096 + 40, 4096
    x, w, b = _case(64, N, K, True, seed=5)
    a = ext.linear_int4w(x, *w, b, OF.ACT_GELU)
    assert torch.equal(a, ext.linear_int4w(x, *w, b, OF.ACT_GELU))
    for m in (1, 2, 9, 33):   # every token-tile instance gives each row the same bits
        for r in range(0, 64 - m + 1, 17):
            assert torch.equal(ext.linear_int4w(x[r : r + m].contiguous(), *w, b, OF.ACT_GELU), a[r : r + m]), (m, r)
    xs = x[:3].clone()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ext.linear_int4w(xs, *w, b, OF.ACT_GELU)
    xs.copy_(x[10:13])
    graph.replay()
    assert torch.equal(out, a[10:13])
    del graph


# ------------------------------------------------------------------------------------------------ larger M
def test_dequant_is_bit_equal_to_the_mirror(ext):
    _, w, _ = _case(1, 1000, 4096 + 128, False, seed=2)
    assert torch.equal(ext.dequant_int4_rows(*w), OF.int4_dequant_ref(*w))
    # every nibble against every zero point, at scales of several binades
    q = torch.arange(256, device=DEV, dtype=U8).repeat(16, 1)             # [16, 256]: K = 512, every byte
    z = torch.arange(16, device=DEV, dtype=U8)[:, None].repeat(1, 4)      # row r: zero point r
    s = torch.tensor([0.0078125, 0.3, 1.0, 7.7e3], device=DEV).bfloat16().repeat(16, 1)
    assert torch.equal(ext.dequant_int4_rows(q, s, z), OF.int4_dequant_ref(q, s, z))


@pytest.mark.parametrize("M", [T + 1, 100, 512])
@pytest.mark.parametrize("epi", [(False, None), (True, "gelu")], ids=["plain", "bias_gelu"])
def test_above_threshold_is_the_bf16_gemm_on_the_dequantized_weight(ext, M, epi):
    bias, act = epi
    x, w, b = _case(M, 3072, 1024, bias, seed=M)
    want, _ = ext.linear_fwd(x, OF.int4_dequant_ref(*w), b, ACT[act], False)
    got = OF.linear_int4w(x.view(1, M, 1024), *w, b, act)
    assert got.shape == (1, M, 3072) and torch.equal(got[0], want)


def test_dispatch_by_rows(ext, monkeypatch):
    calls = []

    class Rec:
        def __getattr__(self, name):
            calls.append(name)
            return getattr(ext, name)

    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: Rec())
    monkeypatch.setattr(OF, "linear_int4w_ref", lambda *a, **k: pytest.fail("the reference math ran"))
    x, w, _ = _case(T + 1, 256, 512, False)
    with torch.no_grad():
        OF.linear_int4w(x[:T], *w)
        assert calls == ["linear_int4w"]
        calls.clear()
        OF.linear_int4w(x, *w)
        assert calls == ["dequant_int4_rows", "linear_fwd"]


# ------------------------------------------------------------------------------------------------ the bindings
# ids and mutations from the CPU build of the cases; the tensors are built on the GPU by the fixture
IDS = [c.id for c in int4_cases("cpu")]
MUTATIONS = [(i, m) for i, c in enumerate(int4_cases("cpu")) for m in c.mutations]


@pytest.fixture(scope="module")
def cases():
    return int4_cases(DEV)


@pytest.mark.parametrize("i", range(len(IDS)), ids=IDS)
def test_valid_arguments_run(ext, cases, i):
    case = cases[i]
    out = getattr(ext, case.op)(*case.values())
    assert out.shape == case.outputs[0]


@pytest.mark.parametrize("i,mutation", MUTATIONS, ids=[f"{IDS[i]}-{n}-{k}" for i, (n, k, _) in MUTATIONS])
def test_each_mutation_is_rejected(ext, cases, i, mutation):
    name, kind, fragment = mutation
    case = cases[i]
    with pytest.raises(RuntimeError) as e:
        getattr(ext, case.op)(*C.mutated(case, name, kind, "cpu"))
    assert fragment in str(e.value).splitlines()[0]


def test_rows_and_activation_are_rejected(ext):
    x, w, b = _case(4, 128, 256, True)
    assert ext.linear_int4w(x, *w, b, 0).shape == (4, 128)
    for xx, act in ((torch.randn(65, 256, device=DEV).bfloat16(), 0), (x[:0], 0), (x, 6), (x[:, :128].contiguous(), 0)):
        with pytest.raises(RuntimeError, match="linear_int4w: "):
            ext.linear_int4w(xx, *w, b, act)


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
    if name == "t5":   # as in the FP8 tests: T5's builder makes its logits chaotic at bf16 precision
        with torch.no_grad():
            for p in m.parameters():
                p.mul_(0.2)
    return quantize_weights_int4_(m)


GEMMS = ("linear_fwd", "gemm", "linear_bias_residual", "linear_fp8_fwd", "dgrad_actgrad", "gemm_rs", "ag_gemm")


class _Recorder:
    """Records the linear ops; a bf16 GEMM must never see packed INT4 bytes, and may only see a weight that the
    dequantize kernel produced or one that was not quantized."""

    def __init__(self, ext, plain):
        self.ext, self.calls, self.dequantized, self.plain = ext, [], set(), plain

    def __getattr__(self, name):
        fn = getattr(self.ext, name)
        if name not in GEMMS + ("linear_int4w", "dequant_int4_rows"):
            return fn

        def wrapped(*a, **k):
            if name in GEMMS:
                assert not any(isinstance(t, torch.Tensor) and t.dtype == U8 for t in a), name
            if name in ("linear_fwd", "linear_bias_residual"):
                assert a[1].data_ptr() in self.dequantized or a[1].data_ptr() in self.plain, name
            out = fn(*a, **k)
            if name == "dequant_int4_rows":
                self.dequantized.add(out.data_ptr())
            self.calls.append(name)
            return out
        return wrapped


NAMES = ["llama", "llama_gqa", "gpt2", "bloom", "chatglm", "chatglm_prefix", "t5"]


@pytest.mark.parametrize("kv", [None, "fp8"])
@pytest.mark.parametrize("name", NAMES)
def test_generate_runs_the_int4_weight_kernel(_topo, ext, monkeypatch, name, kv):
    m = _model(name)
    plain = {p.data_ptr() for p in m.parameters() if p.dtype != U8}   # heads, tied embeddings (and scales)
    rec = _Recorder(ext, plain)
    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: rec)
    monkeypatch.setattr(OF, "linear_int4w_ref", lambda *a, **k: pytest.fail("an INT4 linear ran the reference math"))
    ids = torch.randint(3, 100, (3, 7), generator=torch.Generator().manual_seed(1)).to(DEV)
    with torch.no_grad():
        if name == "t5":
            out = m.generate(ids, max_length=6, eos_token_id=None, kv_cache_dtype=kv)
        else:
            out = m.generate(ids, max_length=13, eos_token_id=None, kv_cache_dtype=kv)
    assert out.shape[0] == 3
    assert m.kv_cache.dtype == torch.bfloat16 and m.kv_cache.kv_dtype == (torch.float8_e4m3fn if kv else torch.bfloat16)
    n_int4 = sum(1 for l in m.modules() if isinstance(l, Linear1D) and l.int4)
    assert rec.calls.count("linear_int4w") > n_int4   # the prompt and the decode steps
    assert "dequant_int4_rows" not in rec.calls          # no step has more than T rows here


def _teacher_forced(m, name):
    """Logits of a prompt, three single steps, a 4-token step and a 29-token continuation (3 · 29 rows > 64)."""
    ids = torch.randint(3, 100, (3, 7), generator=torch.Generator().manual_seed(1)).to(DEV)
    more = torch.randint(3, 100, (3, 37), generator=torch.Generator().manual_seed(3)).to(DEV)
    chunks = [(0, 1), (1, 2), (2, 3), (3, 7), (7, 36)]
    out = []
    with torch.no_grad():
        if name == "t5":
            m.allocate_kv_cache(3, 37)
            out.append(m(ids, more[:, :1], None, use_cache=True)["logits"])
            for lo, hi in chunks:
                out.append(m(ids, more[:, 1 + lo : 1 + hi], None, use_cache=True)["logits"])
        else:
            m.allocate_kv_cache(3, 44)
            out.append(m(ids, use_cache=True)["logits"])
            for lo, hi in chunks:
                out.append(m(more[:, lo:hi], use_cache=True)["logits"])
    m.set_cache(None) if name != "t5" else m.set_cache(None, None)
    return torch.cat(out, dim=1).float()


@pytest.mark.parametrize("name", NAMES)
def test_teacher_forced_logits_match_reference_math(_topo, monkeypatch, name):
    """The kernel (and the dequantize + bf16 GEMM path) against the reference math over the same INT4 weights; every
    other op runs natively on both sides.  Tolerance that of the FP8-weight test."""
    m = _model(name)
    got = _teacher_forced(m, name)
    monkeypatch.setattr(OF, "linear_int4w", OF.linear_int4w_ref)
    want = _teacher_forced(m, name)
    assert rel_err(got, want) < 3e-2, rel_err(got, want)


def test_llama_fused_paths_decline_int4_weights(_topo, monkeypatch):
    """Llama's fused gate/up GEMM and Linear1D's fused tensor-parallel paths take bf16 weights only: on INT4 weights
    they decline, and the per-Linear path runs."""
    from libai_b200.ops import gated_mlp

    m = _model("llama")
    mlp = m.model.layers[0].mlp
    x = torch.randn(3, 128, device=DEV).bfloat16()
    monkeypatch.setattr(gated_mlp, "enabled", lambda: True)
    monkeypatch.setattr(gated_mlp, "gated_mlp", lambda *a, **k: pytest.fail("the fused gate/up GEMM ran"))
    topo = dist.get_dist_util()
    monkeypatch.setattr(topo, "fused_tp_comm", True, raising=False)
    monkeypatch.setattr(Linear1D, "_forward_fused", lambda *a, **k: pytest.fail("a fused TP path ran"))
    with torch.no_grad():
        assert mlp._forward_fused_gate_up(x) is None
        assert mlp.down_proj.fused_bias_residual(x, x) is None
        y = mlp(x)
        g, u, d = mlp.gate_proj, mlp.up_proj, mlp.down_proj
        h = OF.swiglu(OF.linear_int4w(x, g.weight, g.weight_scale, g.weight_zero),
                      OF.linear_int4w(x, u.weight, u.weight_scale, u.weight_zero))
        want = OF.linear_int4w(h, d.weight, d.weight_scale, d.weight_zero)
    assert torch.equal(y, want)


# ------------------------------------------------------------------------------------------------ decode graphs
@pytest.mark.parametrize("beams", [1, 4], ids=["greedy", "beams4"])
@pytest.mark.parametrize("kv", [None, "fp8"])
@pytest.mark.parametrize("name", ["llama_gqa", "qwen", "gpt2", "bloom", "chatglm", "glm", "t5", "llama_adapter"])
def test_decode_graphs_are_bit_identical_on_int4_weights(_topo, monkeypatch, name, kv, beams):
    from tests import test_decode_graphs_gpu as G

    m = quantize_weights_int4_(G._model(name))
    captures = G._Captures(monkeypatch)
    kw = dict(kv_cache_dtype=kv, num_beams=beams)
    G._same(G._generate(m, name, False, **kw), G._generate(m, name, True, **kw))
    assert captures.n == 1
