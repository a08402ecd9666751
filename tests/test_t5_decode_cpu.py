"""T5 / mT5 on the preallocated KV caches, without a GPU: the relative-bias vector against ``compute_bias``, the decode
reference's relative-bias and non-causal semantics against the dense reference, cached greedy / beam generation against
``transformers.T5ForConditionalGeneration``, cached teacher-forced logits against the uncached forward, which kernels a
bf16 model reaches with the native path selected, tensor parallelism, and the ptxas figures of the decode instances."""
import os
import re
import subprocess
import sys

import pytest
import torch

from libai_b200.config import DictConfig
from libai_b200.inference.kv_cache import StaticKVCache, padding_window
from libai_b200.layers._param import param_defaults
from libai_b200.ops import build as ops_build
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from projects.MT5.mt5_model import MAX_DISTANCE, MT5Model, relative_position_bucket
from tests.dist_utils import run_distributed


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cpu")))


GEN = dict(is_encoder_decoder=True, max_length=12, min_length=0, do_sample=False, early_stopping=False, num_beams=1,
           num_beam_groups=1, diversity_penalty=0.0, temperature=1.0, top_k=50, top_p=1.0, typical_p=1.0,
           repetition_penalty=1.0, length_penalty=1.0, no_repeat_ngram_size=0, encoder_no_repeat_ngram_size=0,
           num_return_sequences=1, chunk_size_feed_forward=0, output_scores=False, use_cache=True, eos_token_id=1,
           pad_token_id=0, decoder_start_token_id=0)


def _cfg(**kw):
    return DictConfig(dict(dict(GEN, vocab_size=96, hidden_size=64, hidden_layers=2, num_attention_heads=4, head_size=16,
                                intermediate_size=128, embedding_dropout_prob=0.0, hidden_dropout_prob=0.0,
                                attention_probs_dropout_prob=0.0, relative_attention_num_buckets=8,
                                initializer_range=0.5, layernorm_eps=1e-6, amp_enabled=False, model_type="mt5",
                                padding_idx=0, tie_word_embeddings=False), **kw))


def _model(dtype=torch.float32, seed=0, **kw):
    with param_defaults(dtype=dtype, device="cpu", seed=seed):
        return MT5Model(_cfg(**kw)).eval()


def _encoder_batch(pads, side, s=12, seed=1):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(2, 96, (len(pads), s), generator=g)
    am = torch.ones_like(ids)
    for i, p in enumerate(pads):
        if p:
            sl = slice(0, p) if side == "left" else slice(s - p, s)
            ids[i, sl], am[i, sl] = 0, 0
    return ids, am


# ------------------------------------------------------------------------------------------------ relative bias
@pytest.mark.parametrize("num_buckets,max_distance", [(32, 128), (8, 20)])
def test_relative_vector_reproduces_the_bucketed_bias(num_buckets, max_distance):
    """rel[h, min(p − j, R − 1)] with R = max_distance + 1 is the decoder's bucketed bias for every 0 <= j <= p."""
    table = torch.randn(num_buckets, 3, generator=torch.Generator().manual_seed(num_buckets))
    R = max_distance + 1
    rel = table[relative_position_bucket(-torch.arange(R), bidirectional=False, num_buckets=num_buckets,
                                         max_distance=max_distance)].t()                             # [a, R]
    n = 4 * max_distance
    p, j = torch.arange(n)[:, None], torch.arange(n)[None, :]
    want = table[relative_position_bucket(j - p, bidirectional=False, num_buckets=num_buckets,
                                          max_distance=max_distance)]                                 # [n, n, a]
    got = rel[:, (p - j).clamp(0, R - 1)].permute(1, 2, 0)
    low = (j <= p).expand(n, n)
    assert torch.equal(got[low], want[low])


def test_model_relative_vector_equals_compute_bias():
    attn = _model(relative_attention_num_buckets=32).decoder.layers[0].self_attention
    rel = attn.relative_bias_vector()
    assert rel.shape == (4, MAX_DISTANCE + 1) and rel.dtype == torch.float32 and rel.is_contiguous()
    n = 4 * MAX_DISTANCE
    dense = attn.compute_bias(n, n, "cpu")[0]                                                          # [a, n, n]
    p, j = torch.arange(n)[:, None], torch.arange(n)[None, :]
    low = (j <= p).expand(n, n)
    assert torch.equal(rel[:, (p - j).clamp(0, MAX_DISTANCE)][:, low], dense.float()[:, low])


# ------------------------------------------------------------------------------------------------ reference math
def test_decode_reference_relative_bias_equals_dense_bias():
    attn = _model().decoder.layers[0].self_attention
    g = torch.Generator().manual_seed(0)
    b, a, d, past, s, cap = 3, 4, 16, 9, 5, 20
    kv_start = torch.tensor([0, 3, 7], dtype=torch.int32)
    q = torch.randn(b, s, a, d, generator=g, dtype=torch.float64)
    k_cache = torch.randn(b, a, cap, d, generator=g, dtype=torch.float64)
    v_cache = torch.randn(b, a, cap, d, generator=g, dtype=torch.float64)
    lens = torch.full((b,), past, dtype=torch.int32)
    with torch.no_grad():
        rel = attn.relative_bias_vector().double()
        dense = attn.compute_bias(s, past + s, "cpu").double()                                        # [1, a, s, L]
    got = OF.decode_attention_ref(q, k_cache, v_cache, lens, kv_start, scale=1.0, rel_bias=rel)
    L = past + s
    mask = (torch.arange(L)[None, :] >= kv_start.long()[:, None])[:, None, None, :]
    want = OF.attention_ref(q.transpose(1, 2), k_cache[:, :, :L], v_cache[:, :, :L], causal=True, scale=1.0,
                            mask=mask, bias=dense).transpose(1, 2)
    torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(OF.decode_attention(q, k_cache, v_cache, lens, kv_start, scale=1.0, rel_bias=rel), got,
                               rtol=0, atol=0)


def test_decode_reference_non_causal_window():
    g = torch.Generator().manual_seed(1)
    b, a, d, s, cap = 4, 2, 8, 3, 16
    kv_start = torch.tensor([0, 4, 2, 5], dtype=torch.int32)
    lens = torch.tensor([16, 11, 2, 5], dtype=torch.int32)          # the last two windows are empty
    q = torch.randn(b, s, a, d, generator=g, dtype=torch.float64)
    k_cache = torch.randn(b, a, cap, d, generator=g, dtype=torch.float64)
    v_cache = torch.randn(b, a, cap, d, generator=g, dtype=torch.float64)
    got = OF.decode_attention_ref(q, k_cache, v_cache, lens, kv_start, scale=0.3, causal=False)
    j = torch.arange(cap)[None, :]
    mask = ((j >= kv_start.long()[:, None]) & (j < lens.long()[:, None]))[:, None, None, :]
    want = OF.attention_ref(q.transpose(1, 2), k_cache, v_cache, causal=False, scale=0.3, mask=mask).transpose(1, 2)
    torch.testing.assert_close(got[:2], want[:2], rtol=1e-6, atol=1e-6)
    assert torch.equal(got[2:], torch.zeros_like(got[2:]))


def test_padding_window():
    m = torch.tensor([[1, 1, 0, 0], [0, 0, 1, 1], [1, 1, 1, 1], [0, 1, 1, 0]])
    start, end = padding_window(m)
    assert start.tolist() == [0, 2, 0, 1] and end.tolist() == [2, 4, 4, 3] and start.dtype == torch.int32
    assert padding_window(torch.tensor([[1, 0, 1, 1]])) is None          # a hole
    assert padding_window(torch.tensor([[1, 1], [0, 0]])) is None        # a row without a token


# ------------------------------------------------------------------------------------------------ HF parity
def _hf_pair(tmp_path, model_type, init=1.0):
    transformers = pytest.importorskip("transformers")
    from projects.MT5.utils.mt5_loader import T5LoaderHuggerFace

    torch.manual_seed(0)
    ff, tie = ("relu", True) if model_type == "t5" else ("gated-gelu", False)
    hf = transformers.T5ForConditionalGeneration(transformers.T5Config(
        vocab_size=96, d_model=64, d_kv=16, d_ff=128, num_layers=2, num_heads=4, relative_attention_num_buckets=8,
        dropout_rate=0.0, feed_forward_proj=ff, tie_word_embeddings=tie, scale_decoder_outputs=tie,
        decoder_start_token_id=0, eos_token_id=1, pad_token_id=0, initializer_factor=init)).eval()
    d = str(tmp_path / model_type)
    hf.save_pretrained(d)
    m = T5LoaderHuggerFace(MT5Model, _cfg(), d, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                           embedding_dropout_prob=0.0).load().eval()
    assert m.model_type == model_type
    return hf, m


@pytest.mark.parametrize("side", ["right", "left"])
@pytest.mark.parametrize("model_type", ["t5", "mt5"])
def test_cached_generate_matches_hf(tmp_path, model_type, side, monkeypatch):
    hf, m = _hf_pair(tmp_path, model_type)
    reordered = []
    reorder = StaticKVCache.reorder_
    monkeypatch.setattr(StaticKVCache, "reorder_", lambda c, idx: (reordered.append(c), reorder(c, idx)))
    enc, am = _encoder_batch((0, 3, 5), side)
    for beams in (1, 3):
        reordered.clear()
        ours = m.generate(enc, encoder_attn_mask=am, max_length=12, num_beams=beams)
        theirs = hf.generate(enc, attention_mask=am, max_length=12, do_sample=False, num_beams=beams,
                             early_stopping=False)
        assert ours.tolist() == theirs[:, :ours.shape[1]].tolist(), (beams, ours, theirs)
        assert isinstance(m.kv_cache, StaticKVCache) and isinstance(m.cross_cache, StaticKVCache)
        assert not m.cross_cache.dense_mask
        # beam search gathers the self-attention cache in place, never the cross cache
        assert (len(reordered) > 0) == (beams > 1)
        assert all(c is m.kv_cache for c in reordered)


def test_beam_search_with_a_sample_finishing_early_matches_hf(tmp_path):
    """With these weights and eos token 12, every beam of the first sample has ended after two tokens, eleven steps
    before the others: its rows then take row 0's self cache (as in HF) and keep their own cross rows.  After its eos
    the generator (``BeamSearchScorer.finalize``) fills a finished row with pad_token_id where HF repeats the eos, so
    that row is compared with HF up to its eos; the whole output, fill included, must equal ``use_cache=False``, which
    runs the uncached forward with no cache at all."""
    hf, m = _hf_pair(tmp_path, "mt5", init=4.0)
    enc, am = _encoder_batch((0, 2, 4), "right", seed=1)
    n, beams, eos = 14, 3, 12
    theirs = hf.generate(enc, attention_mask=am, max_length=n, do_sample=False, num_beams=beams, eos_token_id=eos,
                         pad_token_id=0, early_stopping=False)
    # the case this test is about: sample 0 ends at step 2, the others run to the last step on varied tokens
    assert theirs.shape[1] == n and theirs[0, 2] == eos and not (theirs[0, :2] == eos).any()
    assert not (theirs[1:] == eos).any() and all(len(set(row.tolist())) >= 4 for row in theirs[1:])
    ours = m.generate(enc, encoder_attn_mask=am, max_length=n, num_beams=beams, eos_token_id=eos)
    assert ours[0, :3].tolist() == theirs[0, :3].tolist() and (ours[0, 3:] == 0).all()
    assert ours[1:].tolist() == theirs[1:].tolist()
    uncached = m.generate(enc, encoder_attn_mask=am, max_length=n, num_beams=beams, eos_token_id=eos, use_cache=False)
    assert ours.tolist() == uncached.tolist()


# ------------------------------------------------------------------------------------------------ cached vs uncached
@pytest.mark.parametrize("mask", ["none", "right", "holes"])
def test_teacher_forced_cached_logits_equal_uncached(mask):
    """Single steps, a 16-token chunk (the decode kernel's largest) and a 20-token chunk through the caches give the
    uncached forward's logits, to 1e-5 of the largest one (fp32: the two paths sum in different orders)."""
    m = _model(relative_attention_num_buckets=32)
    enc, am = _encoder_batch((0, 3, 6), "right", s=20)
    if mask == "holes":
        am[0, 4] = 0
    am = None if mask == "none" else am
    dec = torch.randint(2, 96, (3, 40), generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        want = m(enc, dec, am)["logits"]
        m.allocate_kv_cache(3, 40)
        got = [m(enc, dec[:, lo:hi], am, use_cache=True)["logits"]
               for lo, hi in [(0, 1), (1, 2), (2, 3), (3, 4), (4, 20), (20, 40)]]
    assert m.kv_cache.length == 40 and m.cross_cache.dense_mask == (mask == "holes")
    err = (torch.cat(got, dim=1) - want).abs().max().item()
    assert err <= 1e-5 * want.abs().max().item(), (err, want.abs().max().item())


# ------------------------------------------------------------------------------------------------ dispatch
class _StubExt:
    """The extension's decode and flash ops, computed with the reference math; records every call."""

    def __init__(self, ref):
        self.calls, self.ref = [], ref

    def kv_append(self, qkv, k_cache, v_cache, seqlens, cos, sin, write_q):
        self.calls.append(("kv_append", None, True))
        return OF.kv_cache_append_ref(qkv, k_cache, v_cache, seqlens)

    def decode_attn(self, q, k_cache, v_cache, seqlens, kv_start, scale, splits, alibi_slopes=None, rel_bias=None,
                    causal=True):
        self.calls.append(("decode_attn", rel_bias, causal))
        return self.ref(q, k_cache, v_cache, seqlens, kv_start, scale=scale, rel_bias=rel_bias, causal=causal)

    def attn_fwd(self, q, k, v, causal, scale, kv_lens, bias, alibi_slopes, p_drop, salt, kv_start=None,
                 doc_start=None):
        self.calls.append(("attn_fwd", bias, causal))
        vis = OF.visible_keys(q.shape[-2], k.shape[-2], causal=causal, kv_start=kv_start, kv_lens=kv_lens)
        o = OF.attention_ref(q, k, v, causal=False, scale=scale, mask=vis, bias=bias)
        return o.masked_fill(~vis.any(-1, keepdim=True), 0), torch.empty(0), torch.empty(0)


@pytest.fixture
def native_attention(monkeypatch):
    """As if on the GPU for the attention ops only (the GEMMs and norms keep the PyTorch path); any call of the decode
    reference outside the stub, and any concatenation of 4-D tensors (a K/V history), is recorded."""
    ext = _StubExt(OF.decode_attention_ref)
    attention_checks = {"_decode_native", "attention_supported", "attention_qkvpacked_supported"}
    monkeypatch.setattr(OF, "use_native", lambda *t: sys._getframe(1).f_code.co_name in attention_checks)
    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: ext)
    monkeypatch.setattr(OF, "decode_attention_ref", lambda *a, **k: ext.calls.append(("decode_attention_ref",)))
    cat = torch.cat
    monkeypatch.setattr(torch, "cat", lambda ts, *a, **k: (
        ext.calls.append(("cat",)) if any(t.dim() == 4 for t in ts) else None, cat(ts, *a, **k))[1])
    return ext


@pytest.mark.parametrize("holes", [False, True])
def test_bf16_decodes_natively_in_every_layer(native_attention, holes):
    m = _model(torch.bfloat16, hidden_size=256, head_size=64)                 # head dim 64
    enc, am = _encoder_batch((0, 2, 5), "right")
    if holes:
        am[0, 3] = 0
    new = 5
    m.generate(enc, encoder_attn_mask=am, max_length=1 + new, eos_token_id=None)
    calls, layers = native_attention.calls, 2
    assert not [c for c in calls if c[0] in ("decode_attention_ref", "cat")]
    assert sum(c[0] == "kv_append" for c in calls) == layers * new
    self_steps = [c for c in calls if c[0] == "decode_attn" and c[2]]
    cross_steps = [c for c in calls if c[0] == "decode_attn" and not c[2]]
    assert len(self_steps) == layers * new
    assert all(c[1] is not None and c[1].dtype == torch.float32 and c[1].shape == (4, MAX_DISTANCE + 1)
               for c in self_steps)
    flash = [c for c in calls if c[0] == "attn_fwd"]
    if holes:   # cross-attention keeps the folded dense bias, through the flash kernel
        assert cross_steps == [] and len(flash) == layers + layers * new     # encoder + every cross step
    else:
        assert len(cross_steps) == layers * new and all(c[1] is None for c in cross_steps)
        assert len(flash) == layers                                           # the encoder only


# ------------------------------------------------------------------------------------------------ tensor parallel
def _generate_tp(rank, world):
    from libai_b200.utils import distributed as dutil

    dutil.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=world, pipeline_parallel_size=1,
                                          device_type="cpu")))
    m = _model(seed=7)
    enc, am = _encoder_batch((0, 3, 5), "left")
    return m.generate(enc, encoder_attn_mask=am, max_length=12, num_beams=2)


def test_tensor_parallel_generation_matches_one_rank():
    one = run_distributed(_generate_tp, 1)[0]
    two = run_distributed(_generate_tp, 2)
    assert (two[0] == one).all() and (two[1] == one).all()


# ------------------------------------------------------------------------------------------------ build
def _ptxas(src, tmp_path):
    res = subprocess.run([ops_build.NVCC, *ops_build.NVCC_FLAGS, "-I", ops_build.CSRC, "-c",
                          os.path.join(ops_build.CSRC, src), "-o", str(tmp_path / (src + ".o"))],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert res.returncode == 0, res.stdout
    regs = dict(re.findall(r"Compiling entry function '(\S+)'.*?Used (\d+) registers", res.stdout, re.S))
    spills = re.findall(r"Function properties for (\S+)\n.*?(\d+) bytes spill stores, (\d+) bytes spill loads",
                        res.stdout)
    return regs, spills


@pytest.mark.skipif(not os.path.exists(ops_build.NVCC), reason="needs nvcc")
def test_t5_decode_kernels_compile_without_spills(tmp_path):
    src = "decode_attention_t5_sm90.cu"
    assert src in ops_build.CU_SOURCES
    regs, spills = _ptxas(src, tmp_path)
    # exactly the relative-bias (Score 2) and non-causal window (Score 3) instances at head dims 64 and 128
    assert sorted(regs) == sorted(f"_ZN2lb3dec21decode_attn_t5_kernelILi{d}ELNS0_5ScoreE{s}EEEvNS0_6ParamsE"
                                  for d in (64, 128) for s in (2, 3))
    assert len(spills) == 4 and all(st == "0" and ld == "0" for _, st, ld in spills), spills


@pytest.mark.skipif(not os.path.exists(ops_build.NVCC), reason="needs nvcc")
def test_existing_decode_kernels_keep_their_registers(tmp_path):
    regs, _ = _ptxas("decode_attention_sm90.cu", tmp_path)
    alibi, _ = _ptxas("decode_attention_alibi_sm90.cu", tmp_path)
    regs.update(alibi)
    name = "_ZN2lb3dec18decode_attn_kernelILi{}ELb{}EEEvNS0_6ParamsE"
    assert {(d, a): int(regs[name.format(d, a)]) for d in (64, 128) for a in (0, 1)} == {
        (64, 0): 94, (64, 1): 96, (128, 0): 142, (128, 1): 145}
