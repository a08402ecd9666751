"""T5's relative-position bias and the non-causal key window in the split-KV decode kernel on the H100: the kernel
against fp64 element by element (tests/attention_ref.py states the bound), its determinism, CUDA-graph replay and the
binding's rejections; then a bf16 mT5 running the native append and decode kernels in every decoder layer, for greedy
and beam search, and its teacher-forced cached logits against the fp32 uncached model."""
import copy

import pytest
import torch

from libai_b200.config import DictConfig
from libai_b200.layers._param import param_defaults
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from projects.MT5.mt5_model import MAX_DISTANCE, MT5Model
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


def rel_table(A, R_, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(A, R_, device=DEV, generator=g) * 2


def i32(xs):
    return torch.tensor(xs, dtype=torch.int32, device=DEV)


def dense_rel(rel, lens, Sq, C):
    """The kernel's relative bias as a dense per-sample bias [B, A, Sq, C]: rel[h, min(lens[b] + i − j, R − 1)]."""
    j = torch.arange(C, device=DEV)[None, None, :]
    i = torch.arange(Sq, device=DEV)[None, :, None]
    dist_ = (lens.long()[:, None, None] + i - j).clamp(0, rel.shape[1] - 1)       # [B, Sq, C]
    return rel.double()[:, dist_].permute(1, 0, 2, 3)


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("splits", [1, 0])
@pytest.mark.parametrize("Sq", [1, 7, 16])
@pytest.mark.parametrize("R_", [5, 129, 2000], ids=["R5", "R129", "R2000"])
def test_decode_relative_bias_per_element(ext, D, splits, Sq, R_):
    """R below the window (the last column covers every longer distance) and above it (never clamped)."""
    A, B, C = 4, 3, 1100
    lens = i32([1000, 37, 0])                   # the last sample holds no row yet
    kv_start = i32([0, 5, 0])                   # left padding of the second
    seed = 3 * D + splits * 7 + Sq + R_
    q, kc, vc = rand(B, Sq, A, D, seed=seed), rand(B, A, C, D, seed=seed + 1), rand(B, A, C, D, seed=seed + 2)
    rel = rel_table(A, R_, seed + 3)
    o = ext.decode_attn(q, kc, vc, lens, kv_start, 1.0 / D ** 0.5, splits, None, rel, True)
    j = torch.arange(C, device=DEV)[None, None, :]
    i = torch.arange(Sq, device=DEV)[None, :, None]
    vis = (j >= kv_start.long()[:, None, None]) & (j <= lens.long()[:, None, None] + i)
    (ref, bnd), _ = R.attention_fwd_ref(q.permute(0, 2, 1, 3), kc, vc, scale=1.0 / D ** 0.5, vis=vis[:, None],
                                        bias=dense_rel(rel, lens, Sq, C), tile=64)
    check(o.permute(0, 2, 1, 3), ref, bnd, f"decode rel_bias D={D} splits={splits} Sq={Sq} R={R_}")
    want = OF.decode_attention_ref(q.double(), kc.double(), vc.double(), lens, kv_start, scale=1.0 / D ** 0.5,
                                   rel_bias=rel.double())
    assert (o.double() - want).abs().max().item() < 2e-2


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("splits", [1, 0])
@pytest.mark.parametrize("Sq", [1, 7, 16])
def test_decode_non_causal_window_per_element(ext, D, splits, Sq):
    A, B, C = 6, 4, 1100
    lens = i32([1100, 512, 40, 3])               # the encoder ends
    kv_start = i32([0, 7, 40, 0])                # left padding; the third window is empty
    seed = 5 * D + splits * 11 + Sq
    q, kc, vc = rand(B, Sq, A, D, seed=seed), rand(B, A, C, D, seed=seed + 1), rand(B, A, C, D, seed=seed + 2)
    o = ext.decode_attn(q, kc, vc, lens, kv_start, 1.0, splits, None, None, False)
    j = torch.arange(C, device=DEV)[None, None, :]
    vis = ((j >= kv_start.long()[:, None, None]) & (j < lens.long()[:, None, None])).expand(B, Sq, C)
    (ref, bnd), _ = R.attention_fwd_ref(q.permute(0, 2, 1, 3), kc, vc, scale=1.0, vis=vis[:, None], tile=64)
    check(o.permute(0, 2, 1, 3), ref, bnd, f"decode window D={D} splits={splits} Sq={Sq}")
    assert torch.equal(o[2], torch.zeros_like(o[2]))
    want = OF.decode_attention_ref(q.double(), kc.double(), vc.double(), lens, kv_start, scale=1.0, causal=False)
    assert (o.double() - want).abs().max().item() < 2e-2


def test_two_calls_are_bit_identical(ext):
    q, kc, vc = rand(4, 2, 16, 128, seed=4), rand(4, 16, 2048, 128, seed=5), rand(4, 16, 2048, 128, seed=6)
    lens, kv_start, rel = i32([2000, 1500, 17, 900]), i32([0, 40, 3, 0]), rel_table(16, 129, 7)
    for args in ((None, rel, True), (None, None, False)):
        a = ext.decode_attn(q, kc, vc, lens, kv_start, 1.0, 0, *args)
        b = ext.decode_attn(q, kc, vc, lens, kv_start, 1.0, 0, *args)
        assert torch.equal(a, b)


@pytest.mark.parametrize("causal", [True, False])
def test_graph_replay_after_lengths_bump_matches_eager(ext, causal):
    B, A, D, C = 3, 16, 64, 1024
    q, kc, vc = rand(B, 1, A, D, seed=7), rand(B, A, C, D, seed=8), rand(B, A, C, D, seed=9)
    lens, kv_start, rel = i32([100, 400, 7]), i32([0, 12, 2]), rel_table(A, 129, 10)

    def step():
        return OF.decode_attention(q, kc, vc, lens, kv_start, scale=1.0, rel_bias=rel if causal else None,
                                   causal=causal)

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


def test_binding_rejects_bad_rel_bias_and_combinations(ext):
    from projects.BLOOM.modeling.bloom_model import alibi_slopes

    q, kc, vc = rand(2, 1, 4, 64, seed=10), rand(2, 4, 64, 64, seed=11), rand(2, 4, 64, 64, seed=12)
    lens, kv_start = i32([3, 3]), i32([0, 0])
    good = rel_table(4, 129, 13)
    for bad in (good.double(), good.bfloat16(), good[:3], good.repeat(2, 1), good.view(-1), good.cpu(),
                good.t().contiguous().t(), good[:, :0], good[:, ::2]):
        with pytest.raises(RuntimeError, match="decode_attn: rel_bias: contiguous fp32 \\[A, R\\] with R >= 1"):
            ext.decode_attn(q, kc, vc, lens, kv_start, 1.0, 0, None, bad, True)
    slopes = alibi_slopes(4).to(DEV)
    with pytest.raises(RuntimeError, match="decode_attn: alibi_slopes or rel_bias, not both"):
        ext.decode_attn(q, kc, vc, lens, kv_start, 1.0, 0, slopes, good, True)
    for s_, r_ in ((slopes, None), (None, good)):
        with pytest.raises(RuntimeError, match="decode_attn: causal=False takes no score bias"):
            ext.decode_attn(q, kc, vc, lens, kv_start, 1.0, 0, s_, r_, False)


# ------------------------------------------------------------------------------------------------ mT5
@pytest.fixture(autouse=True)
def _topo():
    """A one-GPU topology; the tests after these see the global random state they would have seen without them."""
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    with torch.random.fork_rng(devices=[0]):
        yield


def _mt5(layers=2):
    """Weights at 0.02, where the bf16 model stays close to the fp32 one (T5 does not scale its scores, and larger
    random weights make the attention nearly hard and the two precisions part), and relative-bias tables of unit scale,
    so that the bias moves the logits far more than bf16 rounding does."""
    cfg = DictConfig(dict(vocab_size=512, hidden_size=512, hidden_layers=layers, num_attention_heads=8, head_size=64,
                          intermediate_size=1024, embedding_dropout_prob=0.0, hidden_dropout_prob=0.0,
                          attention_probs_dropout_prob=0.0, relative_attention_num_buckets=32, initializer_range=0.02,
                          layernorm_eps=1e-6, amp_enabled=False, model_type="mt5", padding_idx=0,
                          is_encoder_decoder=True, tie_word_embeddings=False, eos_token_id=1, pad_token_id=0,
                          decoder_start_token_id=0, max_length=20, use_cache=True))
    with param_defaults(dtype=torch.float32, device=DEV, seed=3):
        fp32 = MT5Model(cfg).eval()
    g = torch.Generator(device=DEV).manual_seed(9)
    with torch.no_grad():
        for stack in (fp32.encoder, fp32.decoder):
            table = stack.layers[0].self_attention.relative_attention_bias
            table.copy_(torch.randn(table.shape, device=DEV, generator=g))
    return fp32, copy.deepcopy(fp32).to(torch.bfloat16)


class _Recorder:
    """The extension, with the calls of the decode ops recorded (decode_attn: rel_bias and causal)."""

    def __init__(self, ext):
        self.ext, self.calls = ext, []

    def __getattr__(self, name):
        fn = getattr(self.ext, name)
        if name in ("kv_append", "decode_attn", "attn_fwd"):
            def wrapped(*a, **k):
                self.calls.append((name, a[8] if name == "decode_attn" and len(a) > 8 else None,
                                   a[9] if name == "decode_attn" and len(a) > 9 else True))
                return fn(*a, **k)
            return wrapped
        return fn


@pytest.fixture
def recorder(ext, monkeypatch):
    rec = _Recorder(ext)
    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: rec)
    monkeypatch.setattr(OF, "decode_attention_ref", lambda *a, **k: pytest.fail("the decode reference ran"))
    return rec


def _encoder_batch(b, s, pads, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, 512, (b, s), generator=g)
    am = torch.ones_like(ids)
    for i, p in enumerate(pads):
        if p:
            ids[i, s - p:], am[i, s - p:] = 0, 0
    return ids.to(DEV), am.to(DEV)


@pytest.mark.parametrize("beams", [1, 3])
def test_generate_runs_the_native_decode_kernels_in_every_layer(recorder, beams):
    _, m = _mt5()
    enc, am = _encoder_batch(3, 40, (0, 9, 17), seed=1)
    new = 6
    with torch.no_grad():
        out = m.generate(enc, encoder_attn_mask=am, max_length=1 + new, eos_token_id=None, num_beams=beams)
    assert out.shape == (3, 1 + new)
    names = [c[0] for c in recorder.calls]
    assert names.count("kv_append") == 2 * new
    self_steps = [c for c in recorder.calls if c[0] == "decode_attn" and c[2]]
    cross_steps = [c for c in recorder.calls if c[0] == "decode_attn" and not c[2]]
    assert len(self_steps) == len(cross_steps) == 2 * new
    assert all(c[1] is not None and c[1].shape == (8, MAX_DISTANCE + 1) and c[1].is_cuda for c in self_steps)
    assert names.count("attn_fwd") == 2                                  # the encoder


@pytest.mark.parametrize("padded", [False, True], ids=["unpadded", "right_padded"])
def test_teacher_forced_cached_logits_match_fp32_uncached(recorder, padded):
    """Four single steps, a 16-token chunk (the decode kernel's largest) and a 20-token chunk (the flash kernel over the
    cache window with the expanded relative bias).  Tolerance: the cached bf16 logits may differ from the fp32 ones by
    at most twice what the uncached bf16 forward does, or 2^-6 of the largest logit, whichever is larger.  So that the
    rule cannot pass a wrong model: the uncached bf16 error must be a small part of the logits, and the same fp32 model
    with the decoder's relative bias moved by one bucket, or (padded) without the encoder mask, must miss by far more."""
    fp32, bf16 = _mt5()
    enc, am = _encoder_batch(3, 64, (0, 11, 30) if padded else (0, 0, 0), seed=3)
    mask = am if padded else None
    dec = torch.randint(2, 512, (3, 40), generator=torch.Generator().manual_seed(4)).to(DEV)
    with torch.no_grad():
        want = fp32(enc, dec, mask)["logits"].double()
        uncached = bf16(enc, dec, mask)["logits"].double()
        bf16.allocate_kv_cache(3, 40)
        got = [bf16(enc, dec[:, lo:hi], mask, use_cache=True)["logits"]
               for lo, hi in [(0, 1), (1, 2), (2, 3), (3, 4), (4, 20), (20, 40)]]
        got = torch.cat(got, dim=1).double()
        shifted = copy.deepcopy(fp32)
        table = shifted.decoder.layers[0].self_attention.relative_attention_bias
        table.copy_(torch.roll(table, 1, dims=0))
        wrong = [shifted(enc, dec, mask)["logits"].double()] + ([fp32(enc, dec, None)["logits"].double()] if padded else [])
    largest = want.abs().max().item()
    err_uncached = (uncached - want).abs().max().item()
    err = (got - want).abs().max().item()
    tol = max(2 * err_uncached, 2.0 ** -6 * largest)
    assert err_uncached <= 0.05 * largest, (err_uncached, largest)
    assert all((w - want).abs().max().item() > 4 * tol for w in wrong), [(w - want).abs().max().item() for w in wrong]
    assert err <= tol, (err, err_uncached, tol)
    names = [c for c in recorder.calls if c[0] == "decode_attn"]
    assert len(names) == 2 * 2 * 5          # self and cross, four single steps and the 16-token chunk, in both layers
