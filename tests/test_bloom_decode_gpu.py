"""ALiBi in the split-KV decode kernel on the H100, and BLOOM decoding from the preallocated KV cache: the kernel
against fp64 element by element (tests/attention_ref.py states the bound), its determinism, CUDA-graph replay and the
binding's rejections; then bf16 BLOOM models at head dims 64 and 128 running the native append and decode kernels in
every layer at every step, against the fp32 uncached model."""
import copy

import pytest
import torch

from libai_b200.config import DictConfig, LazyConfig
from libai_b200.layers._param import param_defaults
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from projects.BLOOM.modeling.bloom_model import BloomForCausalLM, alibi_slopes
from tests import attention_ref as R
from tests.dense_ref import check

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


def rand(*shape, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(*shape, device=DEV, generator=g).bfloat16()


def i32(xs):
    return torch.tensor(xs, dtype=torch.int32, device=DEV)


def kernel_bias(slopes, lens, Sq, C):
    """The kernel's ALiBi as a dense per-sample bias [B, A, Sq, C]: slope_h·(j − lens[b] − i)."""
    j = torch.arange(C, device=DEV)[None, None, :]
    i = torch.arange(Sq, device=DEV)[None, :, None]
    rel = (j - lens.long()[:, None, None] - i).double()                       # [B, Sq, C]
    return slopes.double()[None, :, None, None] * rel[:, None]


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("splits", [1, 2, 7, 0])
@pytest.mark.parametrize("heads_sq", [(8, 8, 1), (8, 8, 4), (4, 4, 16), (8, 2, 4)])
def test_decode_alibi_per_element(ext, D, splits, heads_sq):
    A, G, Sq = heads_sq
    B, C = 3, 1100
    lens = i32([1000, 37, 0])                   # the last sample holds no row yet
    kv_start = i32([0, 5, 0])                   # left padding of the second
    seed = 3 * D + splits * 7 + A * G + Sq
    q, kc, vc = rand(B, Sq, A, D, seed=seed), rand(B, G, C, D, seed=seed + 1), rand(B, G, C, D, seed=seed + 2)
    slopes = alibi_slopes(A).to(DEV)
    scale = D ** -0.5
    o = ext.decode_attn(q, kc, vc, lens, kv_start, scale, splits, slopes)
    j = torch.arange(C, device=DEV)[None, None, :]
    i = torch.arange(Sq, device=DEV)[None, :, None]
    vis = (j >= kv_start.long()[:, None, None]) & (j <= lens.long()[:, None, None] + i)
    (ref, bnd), _ = R.attention_fwd_ref(q.permute(0, 2, 1, 3), kc, vc, scale=scale, vis=vis[:, None],
                                        bias=kernel_bias(slopes, lens, Sq, C), tile=64)
    check(o.permute(0, 2, 1, 3), ref, bnd, f"decode alibi D={D} splits={splits} A/G/Sq={heads_sq}")


def test_no_visible_key_gives_zeros(ext):
    q, kc, vc = rand(2, 1, 4, 64, seed=1), rand(2, 4, 64, 64, seed=2), rand(2, 4, 64, 64, seed=3)
    o = ext.decode_attn(q, kc, vc, i32([3, 3]), i32([10, 0]), 0.125, 0, alibi_slopes(4).to(DEV))
    assert torch.equal(o[0], torch.zeros_like(o[0])) and o[1].abs().sum() > 0


def test_two_calls_are_bit_identical(ext):
    q, kc, vc = rand(4, 2, 16, 128, seed=4), rand(4, 16, 2048, 128, seed=5), rand(4, 16, 2048, 128, seed=6)
    lens, kv_start, slopes = i32([2000, 1500, 17, 900]), i32([0, 40, 3, 0]), alibi_slopes(16).to(DEV)
    a = ext.decode_attn(q, kc, vc, lens, kv_start, 0.088, 0, slopes)
    b = ext.decode_attn(q, kc, vc, lens, kv_start, 0.088, 0, slopes)
    assert torch.equal(a, b)


def test_graph_replay_after_lengths_bump_matches_eager(ext):
    B, A, D, C = 3, 16, 64, 1024
    q, kc, vc = rand(B, 1, A, D, seed=7), rand(B, A, C, D, seed=8), rand(B, A, C, D, seed=9)
    lens, kv_start, slopes = i32([100, 400, 7]), i32([0, 12, 2]), alibi_slopes(A).to(DEV)

    def step():
        return OF.decode_attention(q, kc, vc, lens, kv_start, scale=0.125, alibi_slopes=slopes)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for _ in range(3):
        lens.add_(5)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, step())
    del graph


def test_binding_rejects_bad_slopes(ext):
    q, kc, vc = rand(2, 1, 4, 64, seed=10), rand(2, 4, 64, 64, seed=11), rand(2, 4, 64, 64, seed=12)
    lens, kv_start = i32([3, 3]), i32([0, 0])
    good = alibi_slopes(4).to(DEV)
    for bad in (good.double(), good.bfloat16(), good[:3], good.repeat(2), good.view(2, 2), good.cpu(),
                good.repeat_interleave(2)[::2]):
        with pytest.raises(RuntimeError, match="decode_attn: alibi_slopes"):
            ext.decode_attn(q, kc, vc, lens, kv_start, 0.125, 0, bad)


# ------------------------------------------------------------------------------------------------ BLOOM
@pytest.fixture(autouse=True)
def _topo():
    """A one-GPU topology; the tests after these see the global random state they would have seen without them."""
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    with torch.random.fork_rng(devices=[0]):
        yield


def _bloom(n_head, hidden=1024, layers=2):
    cfg = LazyConfig.load("projects/BLOOM/configs/bloom_inference.py").cfg
    cfg.update(dict(vocab_size=256, hidden_size=hidden, hidden_layers=layers, n_head=n_head))
    with param_defaults(dtype=torch.float32, device=DEV, seed=3):
        fp32 = BloomForCausalLM(cfg).eval()
    return fp32, copy.deepcopy(fp32).to(torch.bfloat16)


class _Recorder:
    """The extension, with the calls of the decode ops counted."""

    def __init__(self, ext):
        self.ext, self.calls = ext, []

    def __getattr__(self, name):
        fn = getattr(self.ext, name)
        if name in ("kv_append", "decode_attn", "attn_fwd"):
            def wrapped(*a, **k):
                # (decode_attn and attn_fwd take the slopes as their 8th argument)
                self.calls.append((name, None if name == "kv_append" else a[7]))
                return fn(*a, **k)
            return wrapped
        return fn


@pytest.fixture
def recorder(ext, monkeypatch):
    rec = _Recorder(ext)
    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: rec)
    return rec


def _prompts(b, s, pads, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(4, 256, (b, s), generator=g)
    am = torch.ones_like(ids)
    for i, p in enumerate(pads):
        ids[i, :p], am[i, :p] = 3, 0
    return ids.to(DEV), am.to(DEV)


@pytest.mark.parametrize("n_head", [16, 8], ids=["d64", "d128"])
def test_generate_runs_the_native_decode_kernels_in_every_layer(recorder, n_head):
    _, m = _bloom(n_head)
    ids, am = _prompts(3, 24, (0, 5, 11), seed=1)
    new = 6
    with torch.no_grad():
        out = m.generate(ids, attention_mask=am, max_length=24 + new, eos_token_id=None)
    assert out.shape == (3, 24 + new)
    names = [c[0] for c in recorder.calls]
    assert names.count("kv_append") == 2 * new
    assert names.count("attn_fwd") == 2                                  # the prefill of each layer
    steps = [c for c in recorder.calls if c[0] == "decode_attn"]
    assert len(steps) == 2 * (new - 1)
    assert all(c[1] is not None and c[1].dtype == torch.float32 and c[1].is_cuda for c in steps)


@pytest.mark.parametrize("n_head", [16, 8], ids=["d64", "d128"])
def test_beam_search_runs_on_the_cache(recorder, n_head):
    _, m = _bloom(n_head)
    ids, am = _prompts(2, 16, (0, 4), seed=2)
    with torch.no_grad():
        out = m.generate(ids, attention_mask=am, max_length=22, eos_token_id=None, num_beams=2)
    assert out.shape == (2, 22)
    assert sum(c[0] == "decode_attn" for c in recorder.calls) == 2 * 5


@pytest.mark.parametrize("padded", [False, True], ids=["unpadded", "left_padded"])
@pytest.mark.parametrize("n_head", [16, 8], ids=["d64", "d128"])
def test_teacher_forced_cached_logits_match_fp32_uncached(recorder, n_head, padded):
    """Prefill, four single steps, a 16-token chunk (the decode kernel's largest) and a 20-token chunk (the flash kernel
    over the cache window).  Tolerance: the cached bf16 logits may differ from the fp32 ones by at most twice what the
    uncached bf16 forward does, or 2^-6 of the largest logit, whichever is larger (non-padded positions)."""
    fp32, bf16 = _bloom(n_head)
    S = 60
    ids, am = _prompts(3, S, (0, 7, 13) if padded else (0, 0, 0), seed=3 + padded)
    mask = am if padded else None
    with torch.no_grad():
        want = fp32(ids, attention_mask=mask)["logits"].double()
        uncached = bf16(ids, attention_mask=mask)["logits"].double()
        bf16.allocate_kv_cache(3, S)
        got = []
        for lo, hi in [(0, 20), (20, 21), (21, 22), (22, 23), (23, 24), (24, 40), (40, 60)]:
            got.append(bf16(ids[:, lo:hi], attention_mask=am[:, :hi] if padded else None, use_cache=True)["logits"])
        got = torch.cat(got, dim=1).double()
    keep = am.bool()
    err_uncached = (uncached - want)[keep].abs().max().item()
    err = (got - want)[keep].abs().max().item()
    tol = max(2 * err_uncached, 2.0 ** -6 * want[keep].abs().max().item())
    assert err <= tol, (err, err_uncached, tol)
    names = [c[0] for c in recorder.calls]
    assert names.count("decode_attn") == 2 * 5                            # four single steps and the 16-token chunk
