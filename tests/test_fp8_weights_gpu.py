"""FP8 (E4M3) weights on the H100: the weight-streaming kernel against fp64 over float(e)·s, its determinism, CUDA-graph
replay and batch invariance, the dequantize + bf16 GEMM path for larger M against the bf16 GEMM on the same weight,
the binding's rejections, and generate() / teacher-forced logits of every cache model with quantized weights."""
import pytest
import torch
import torch.nn.functional as F

from libai_b200.config import DictConfig
from libai_b200.inference import quantize_weights_fp8_
from libai_b200.layers.linear import Linear1D
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from tests.test_decode_gpu import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FP8 = torch.float8_e4m3fn
ACT = {None: 0, "gelu": OF.ACT_GELU, "silu": OF.ACT_SILU}
T = OF.FP8W_KERNEL_MAX_M


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


def _case(M, N, K, bias, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, K, device=DEV, generator=g).bfloat16()
    e, s = OF.kv_cache_quantize_ref(torch.randn(N, K, device=DEV, generator=g) * 0.05)
    b = (torch.randn(N, device=DEV, generator=g) * 0.5).bfloat16() if bias else None
    return x, e, s, b


def _ref64(x, e, s, b, act):
    w = e.double() * s.double()[:, None]
    y = x.double() @ w.T
    if b is not None:
        y = y + b.double()
    y = {None: lambda t: t, "gelu": F.gelu, "silu": F.silu}[act](y)
    return y, x.double().abs() @ w.abs().T   # the result and the sum of |terms| of each dot product


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("K", [16, 1024, 11008])
@pytest.mark.parametrize("M", [1, 2, 7, 8, 9, 16, 33, 64])
@pytest.mark.parametrize("epi", [(False, None), (True, "gelu"), (True, "silu")], ids=["plain", "bias_gelu", "bias_silu"])
def test_kernel_matches_fp64(ext, M, K, epi):
    bias, act = epi
    N = 200 + 4096 * (K == 1024)   # not a multiple of the 64-row block
    x, e, s, b = _case(M, N, K, bias, seed=M * 7 + K)
    y = ext.linear_fp8w(x, e, s, b, ACT[act])
    assert y.dtype == torch.bfloat16 and y.shape == (M, N)
    ref, mag = _ref64(x, e, s, b, act)
    # bf16 rounding of the output, fp32 accumulation over K terms (and the activation's fast math)
    err = (y.double() - ref).abs()
    tol = 2.0 ** -8 * ref.abs() + 2e-6 * mag * (1 + K / 1024) + 1e-5
    assert bool((err <= tol).all()), float((err - tol).max())


def _split_of(N, K):
    """(splits, range) of ``split_of`` in linear_fp8w_sm90.cu: 64-row blocks, ranges of at least 256 columns in 64-column
    steps, enough splits for 4 · 132 CTAs."""
    row_blocks = -(-N // 64)
    splits = min(max(-(-528 // row_blocks), 1), -(-K // 256))
    rng = -(-(-(-K // splits)) // 64) * 64
    return -(-K // rng), rng


# (N, K) -> (splits, range): the paths test_kernel_matches_fp64 does not reach
SPLIT_SHAPES = {
    (37888, 3584): (1, 3584),   # the direct-write epilogue at a real K (Qwen2-7B's packed gate/up projection)
    (200, 208): (1, 256),       # direct write, K % 64 = 16
    (200, 224): (1, 256),       # K % 64 = 32
    (200, 240): (1, 256),       # K % 64 = 48
    (4096, 4128): (9, 512),     # the last split holds 32 columns
    (63, 1040): (5, 256),       # the last split holds 16 columns; one partial row block
    (1, 4096): (16, 256),       # fewer than 16 weight rows: lanes without a valid row
    (8, 4096): (16, 256),
}


@pytest.mark.parametrize("NK", list(SPLIT_SHAPES), ids=[f"N{n}_K{k}" for n, k in SPLIT_SHAPES])
@pytest.mark.parametrize("epi", [(False, None), (True, "silu")], ids=["plain", "bias_silu"])
def test_kernel_split_shapes_match_fp64(ext, NK, epi):
    N, K = NK
    assert _split_of(N, K) == SPLIT_SHAPES[NK]
    bias, act = epi
    x, e, s, b = _case(64, N, K, bias, seed=N + K)
    full = ext.linear_fp8w(x, e, s, b, ACT[act])
    for M in (1, 9, 33, 64):
        y = full if M == 64 else ext.linear_fp8w(x[:M].contiguous(), e, s, b, ACT[act])
        assert y.dtype == torch.bfloat16 and y.shape == (M, N)
        ref, mag = _ref64(x[:M], e, s, b, act)
        # the tolerance of test_kernel_matches_fp64
        err = (y.double() - ref).abs()
        tol = 2.0 ** -8 * ref.abs() + 2e-6 * mag * (1 + K / 1024) + 1e-5
        assert bool((err <= tol).all()), (M, float((err - tol).max()))
        if NK == (37888, 3584):   # batch invariance on the direct-write path, at the first and the last rows
            assert torch.equal(y, full[:M]), M
            tail = ext.linear_fp8w(x[64 - M :].contiguous(), e, s, b, ACT[act])
            assert torch.equal(tail, full[64 - M :]), M
        del ref, mag


def test_kernel_is_deterministic_graph_safe_and_batch_invariant(ext):
    N, K = 4096 + 40, 4096
    x, e, s, b = _case(64, N, K, True, seed=5)
    a = ext.linear_fp8w(x, e, s, b, OF.ACT_GELU)
    assert torch.equal(a, ext.linear_fp8w(x, e, s, b, OF.ACT_GELU))
    for m in (1, 2, 9, 33):   # every token-tile instance gives each row the same bits
        for r in range(0, 64 - m + 1, 17):
            assert torch.equal(ext.linear_fp8w(x[r : r + m].contiguous(), e, s, b, OF.ACT_GELU), a[r : r + m]), (m, r)
    xs = x[:3].clone()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ext.linear_fp8w(xs, e, s, b, OF.ACT_GELU)
    xs.copy_(x[10:13])
    graph.replay()
    assert torch.equal(out, a[10:13])
    del graph


# ------------------------------------------------------------------------------------------------ larger M
def test_dequant_matches_pytorch(ext):
    _, e, s, _ = _case(1, 1000, 4096 + 16, False, seed=2)
    assert torch.equal(ext.dequant_e4m3_rows(e, s), (e.float() * s[:, None]).to(torch.bfloat16))


@pytest.mark.parametrize("M", [T + 1, 100, 512])
@pytest.mark.parametrize("epi", [(False, None), (True, "gelu")], ids=["plain", "bias_gelu"])
def test_above_threshold_is_the_bf16_gemm_on_the_dequantized_weight(ext, M, epi):
    bias, act = epi
    x, e, s, b = _case(M, 3072, 1024, bias, seed=M)
    want, _ = ext.linear_fwd(x, (e.float() * s[:, None]).to(torch.bfloat16), b, ACT[act], False)
    got = OF.linear_fp8w(x.view(1, M, 1024), e, s, b, act)
    assert got.shape == (1, M, 3072) and torch.equal(got[0], want)


def test_dispatch_by_rows(ext, monkeypatch):
    calls = []

    class Rec:
        def __getattr__(self, name):
            calls.append(name)
            return getattr(ext, name)

    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: Rec())
    x, e, s, _ = _case(T + 1, 256, 512, False)
    with torch.no_grad():
        OF.linear_fp8w(x[:T], e, s)
        assert calls == ["linear_fp8w"]
        calls.clear()
        OF.linear_fp8w(x, e, s)
        assert calls == ["dequant_e4m3_rows", "linear_fwd"]


def test_binding_rejections(ext):
    x, e, s, b = _case(4, 128, 256, True)
    ok = ext.linear_fp8w(x, e, s, b, 0)
    assert ok.shape == (4, 128)
    raw = torch.empty(4 * 256 + 8, device=DEV, dtype=torch.bfloat16)
    x_mis = raw[1 : 1 + 4 * 256].view(4, 256)   # contiguous, 2 bytes past a 16-byte boundary
    x_mis.copy_(x)
    e_raw = torch.empty(128 * 256 + 16, device=DEV, dtype=FP8)
    e_mis = e_raw[1 : 1 + 128 * 256].view(128, 256)
    bad = [
        (x.half(), e, s, b), (x.float(), e, s, b), (x, e.view(torch.uint8), s, b), (x, x[:, :128].t(), s, b),
        (x, e, s.double(), b), (x, e, s.bfloat16(), b), (x, e, s[:64], b), (x, e, s, b.float()), (x, e, s, b[:64]),
        (x[:, :250].contiguous(), e[:, :250].contiguous(), s, b),    # K % 16 != 0
        (x[:, :128].contiguous(), e, s, b),                          # K mismatch
        (torch.randn(65, 256, device=DEV).bfloat16(), e, s, b),     # M > 64
        (x[:0], e, s, b),                                           # M = 0
        (x_mis, e, s, b), (x, e_mis, s, b),                         # misaligned
        (x.t().contiguous().t(), e, s, b),                          # not contiguous
        (x.cpu(), e, s, b), (x, e, s.cpu(), b),
    ]
    for args in bad:
        with pytest.raises((RuntimeError, TypeError)):
            ext.linear_fp8w(*args, 0)
    with pytest.raises(RuntimeError):
        ext.linear_fp8w(x, e, s, b, 6)   # the residual-add id is not an activation
    with pytest.raises(RuntimeError):
        ext.dequant_e4m3_rows(e[:, :250].contiguous(), s)


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
    if name == "t5":   # as in the FP8 cache tests: T5's builder makes its logits chaotic at bf16 precision
        with torch.no_grad():
            for p in m.parameters():
                p.mul_(0.2)
    return quantize_weights_fp8_(m)


GEMMS = ("linear_fwd", "gemm", "linear_bias_residual", "linear_fp8_fwd", "dgrad_actgrad", "gemm_rs", "ag_gemm")


class _Recorder:
    """Records the linear ops; a bf16 GEMM must never see FP8 bytes, and may only see a weight that the dequantize kernel
    produced or one that was not quantized."""

    def __init__(self, ext, plain):
        self.ext, self.calls, self.dequantized, self.plain = ext, [], set(), plain

    def __getattr__(self, name):
        fn = getattr(self.ext, name)
        if name not in GEMMS + ("linear_fp8w", "dequant_e4m3_rows"):
            return fn

        def wrapped(*a, **k):
            assert not any(isinstance(t, torch.Tensor) and t.dtype == FP8 for t in a) or name == "linear_fp8w" \
                or name == "dequant_e4m3_rows", name
            if name in ("linear_fwd", "linear_bias_residual"):
                assert a[1].data_ptr() in self.dequantized or a[1].data_ptr() in self.plain, name
            out = fn(*a, **k)
            if name == "dequant_e4m3_rows":
                self.dequantized.add(out.data_ptr())
            self.calls.append(name)
            return out
        return wrapped


NAMES = ["llama", "llama_gqa", "gpt2", "bloom", "chatglm", "chatglm_prefix", "t5"]


@pytest.mark.parametrize("kv", [None, "fp8"])
@pytest.mark.parametrize("name", NAMES)
def test_generate_runs_the_fp8_weight_kernel(_topo, ext, monkeypatch, name, kv):
    m = _model(name)
    plain = {p.data_ptr() for p in m.parameters() if p.dtype != FP8}   # heads and tied embeddings
    rec = _Recorder(ext, plain)
    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: rec)
    monkeypatch.setattr(OF, "linear_fp8w_ref", lambda *a, **k: pytest.fail("an FP8 linear ran the reference math"))
    ids = torch.randint(3, 100, (3, 7), generator=torch.Generator().manual_seed(1)).to(DEV)
    with torch.no_grad():
        if name == "t5":
            out = m.generate(ids, max_length=6, eos_token_id=None, kv_cache_dtype=kv)
        else:
            out = m.generate(ids, max_length=13, eos_token_id=None, kv_cache_dtype=kv)
    assert out.shape[0] == 3
    assert m.kv_cache.dtype == torch.bfloat16 and m.kv_cache.kv_dtype == (FP8 if kv else torch.bfloat16)
    n_fp8 = sum(1 for l in m.modules() if isinstance(l, Linear1D) and l.fp8)
    assert rec.calls.count("linear_fp8w") > n_fp8   # the prompt and the decode steps
    assert "dequant_e4m3_rows" not in rec.calls           # no step has more than T rows here


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
    """The kernel (and the dequantize + bf16 GEMM path) against the reference math over the same FP8 weights; every
    other op runs natively on both sides.  Tolerance that of the bf16 generate() tests."""
    m = _model(name)
    got = _teacher_forced(m, name)
    monkeypatch.setattr(OF, "linear_fp8w", OF.linear_fp8w_ref)
    want = _teacher_forced(m, name)
    assert rel_err(got, want) < 3e-2, rel_err(got, want)
