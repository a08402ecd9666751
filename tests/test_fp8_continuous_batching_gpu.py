"""Continuous batching on FP8 (E4M3) pools on the GPU: the FP8 ragged paged flash prefill bit for bit against the bf16
ragged prefill over the dequantized pools (with 0x7F bytes and NaN scales outside every window, and products that are
fp32 subnormals), the ragged FP8 append bit for bit against the per-sequence paged FP8 append, and the engine's tokens,
decode graphs, prefix caching and ``generate()`` around an FP8 engine."""
import copy

import pytest
import torch

from libai_b200.inference import GenerationEngine
from libai_b200.models.llama_model import rotary_tables
from libai_b200.ops import functional as OF
from tests.test_continuous_batching_gpu import CASES, DEV, MODELS, WORK, _ids, _llama, _pools, _run
from tests.test_continuous_batching_gpu import _topo  # noqa: F401

pytestmark = pytest.mark.gpu
FP8 = torch.float8_e4m3fn


def _fp8_pools(q_lens, past, G, D, seed, share=True):
    """The pools of ``_pools`` quantized, with the E4M3 byte 0x7F (NaN) and NaN scales in every row outside the windows;
    the rows of every third page of each window get scales near 2^-120, so that many of their products float(e)·s are
    fp32 subnormals."""
    table, k, v, cu, pa = _pools(q_lens, past, G, D, seed, share)
    out = []
    for x in (k, v):
        window = ~torch.isnan(x).any(dim=-1)                   # [P, G, 64]
        e, s = OF.kv_cache_quantize_ref(torch.nan_to_num(x))
        tiny = torch.zeros_like(window)
        tiny[::3] = True
        s = torch.where(tiny, s * 2.0 ** -120, s)
        e = torch.where(window[..., None], e.view(torch.uint8), torch.full_like(e.view(torch.uint8), 0x7F))
        s = torch.where(window, s, torch.full_like(s, float("nan")))
        out += [e.view(FP8), s]
    return table, out[0], out[2], out[1], out[3], cu, pa


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("G,A", [(4, 4), (2, 8)])
@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_fp8_ragged_prefill_bit_identical_to_bf16_over_dequantized_pools(D, G, A, alibi, case):
    q_lens, past = CASES[case]
    table, k, v, ks, vs, cu, pa = _fp8_pools(q_lens, past, G, D, seed=case)
    # table entries outside the pool read as zero rows: one inside the last sequence's window, one past the first's
    table[-1, 0] = k.shape[0] + 5
    need0 = -(-(q_lens[0] + past[0]) // 64)
    if need0 < table.shape[1]:
        table[0, need0] = k.shape[0] + 7
    kd, vd = OF.kv_cache_dequant(k, ks), OF.kv_cache_dequant(v, vs)
    window = ~torch.isnan(ks)
    sub = (kd.float().abs() < torch.finfo(torch.float32).tiny) & (kd != 0) & window[..., None]
    assert int(sub.sum()) > 0   # subnormal products reach the tiles
    q = torch.randn(sum(q_lens), A, D, device=DEV).to(torch.bfloat16)
    slopes = torch.linspace(0.5, 0.01, A, device=DEV) if alibi else None
    o = OF.attention_paged_varlen(q, k, v, table, cu, pa, scale=D ** -0.5, alibi_slopes=slopes, k_scale=ks,
                                  v_scale=vs)
    ref = OF.attention_paged_varlen(q, kd, vd, table, cu, pa, scale=D ** -0.5, alibi_slopes=slopes)
    assert torch.isfinite(o).all()
    assert torch.equal(o, ref)


@pytest.mark.parametrize("grouped", [False, True])
@pytest.mark.parametrize("D", [64, 128])
def test_fp8_ragged_append_bit_identical_to_per_sequence_paged(grouped, D):
    q_lens, past = [1, 70, 3, 130], [0, 64, 100, 5]
    G = 2
    table, k, v, ks, vs, cu, pa = _fp8_pools(q_lens, past, G, D, seed=7, share=False)
    T = sum(q_lens)
    qkv = (torch.randn(1, T, G, 4, D, device=DEV) if grouped else torch.randn(1, T, G, 3 * D, device=DEV))
    qkv = qkv.to(torch.bfloat16)
    cos, sin = rotary_tables(D, 1024, device=DEV)
    before = [t.clone() for t in (k, v, ks, vs)]
    k2, v2, ks2, vs2 = (t.clone() for t in (k, v, ks, vs))
    q = OF.kv_cache_append_paged_varlen(qkv, k, v, table, cu, pa, cos, sin, k_scale=ks, v_scale=vs)
    c = cu.tolist()
    written = torch.zeros(ks.shape, dtype=torch.bool, device=DEV)
    for n in range(len(q_lens)):
        qn = OF.kv_cache_append(qkv[:, c[n] : c[n + 1]].contiguous(), k2, v2, pa[n : n + 1], cos, sin, k_scale=ks2,
                                v_scale=vs2, block_table=table[n : n + 1])
        assert torch.equal(q[:, c[n] : c[n + 1]], qn)
        for j in range(past[n], past[n] + q_lens[n]):
            written[int(table[n, j // 64]), :, j % 64] = True
    bits = lambda t: t.view(torch.uint8) if t.dtype == FP8 else t.view(torch.int32)   # noqa: E731
    for got, want, old in zip((k, v, ks, vs), (k2, v2, ks2, vs2), before):
        assert torch.equal(bits(got), bits(want))   # every byte and scale, NaN included
        keep = ~written if got.dim() == 3 else ~written[..., None].expand_as(got)
        assert torch.equal(bits(got)[keep], bits(old)[keep])   # what no sequence writes stays as it was
    assert int(written.sum()) == T * G


def test_fp8_varlen_ops_argument_cases():
    from tests import op_args_cases as C
    from tests.test_fp8_continuous_batching_cpu import fp8_varlen_cases

    ext = __import__("libai_b200.ops", fromlist=["load_ext"]).load_ext(required=True)
    for case in fp8_varlen_cases(DEV):
        out = getattr(ext, case.op)(*case.values())
        torch.cuda.synchronize()
        assert tuple(out.shape) == case.outputs[0] and out.device == torch.device(DEV)
        for name, kind, fragment in case.mutations:
            with pytest.raises(RuntimeError, match=fragment):
                getattr(ext, case.op)(*C.mutated(case, name, kind, "cpu"))


# ---- the engine ------------------------------------------------------------------------------------------------------

def _fp8_prefill_logits(model, toks):
    """The logits of a forward over ``toks`` through an FP8 cache (teacher-forced: every position attends over the
    dequantized rows of the tokens before it, as the engine does)."""
    model.kv_cache_dtype = FP8
    try:
        model.allocate_kv_cache(1, toks.shape[1])
        return model(toks, use_cache=True)["logits"][0].float()
    finally:
        model.kv_cache_dtype = None
        model.set_cache(None)


def _near_argmax_fp8(model, e, ids):
    """The near-argmax rule of the bf16 engine's test, against the fp32 model's FP8-cache forward: ``err`` is the bf16
    model's FP8-cache forward against it over the same tokens, and every emitted token trails the fp32 maximum by at
    most ``3 err``; at least 90 % are its exact argmax."""
    ref_model = copy.deepcopy(model).float()
    exact = total = 0
    with torch.no_grad():
        for rid in ids:
            r = e.requests[rid]
            toks = torch.tensor([r.tokens[:-1]], device=DEV)
            logits = _fp8_prefill_logits(ref_model, toks)[r.prompt_len - 1 :]
            err = float((_fp8_prefill_logits(model, toks)[r.prompt_len - 1 :] - logits).abs().max())
            got = logits.gather(1, torch.tensor(r.generated, device=DEV)[:, None])[:, 0]
            gap = logits.max(dim=1).values - got
            assert float(gap.max()) <= 3 * err, (rid, float(gap.max()), err)
            exact += int((gap == 0).sum())
            total += gap.numel()
    assert exact >= 0.9 * total, (exact, total)


@pytest.mark.parametrize("name", list(MODELS))
def test_fp8_engine_greedy_is_near_argmax_of_fp32_over_fp8_rows(name):
    model = MODELS[name]()
    e = GenerationEngine(model, max_batch=4, max_tokens_per_step=4 + 96, num_pages=40, kv_cache_dtype="fp8")
    ids = _run(e, WORK)
    assert all(e.requests[i].finish_reason == "length" for i in ids)
    assert sorted(e.cache.free) == list(range(40))
    _near_argmax_fp8(model, e, ids)


def test_fp8_engine_decode_graphs_match_eager_with_one_capture():
    model = _llama(num_key_value_heads=2)
    outs = []
    for graphs in (False, True):
        e = GenerationEngine(model, max_batch=4, max_tokens_per_step=4 + 96, num_pages=40, decode_graphs=graphs,
                             kv_cache_dtype="fp8")
        ids = _run(e, WORK)
        outs.append([e.requests[i].generated for i in ids])
        if graphs:
            assert e.graph_captures == 1
    assert outs[0] == outs[1]


def test_fp8_engine_prefix_caching_reuses_as_many_pages_as_bf16():
    model = _llama()
    system = _ids(200, 99)
    work = [[(system + _ids(10, i), 5) for i in range(3)], [(system + _ids(30, 10 + i), 8) for i in range(4)]]
    reused = {}
    for kv in (None, "fp8"):
        e = GenerationEngine(model, max_batch=4, max_tokens_per_step=4 + 256, num_pages=48, prefix_caching=True,
                             kv_cache_dtype=kv)
        ids = _run(e, work[0]) + _run(e, work[1])
        reused[kv] = e.reused_pages
    assert reused["fp8"] == reused[None] >= 4 * 3
    _near_argmax_fp8(model, e, ids)


@pytest.mark.parametrize("name", ["llama", "bloom"])
def test_generate_unchanged_around_an_fp8_engine(name):
    model = MODELS[name]()
    ids = torch.tensor([_ids(40, 0), _ids(40, 1)], device=DEV)
    kw = dict(max_length=60, do_sample=False, use_cache=True)
    before = model.generate(ids, **kw)
    GenerationEngine(model, max_batch=4, max_tokens_per_step=4 + 96, num_pages=40, kv_cache_dtype="fp8").generate(
        [w[0] for w in WORK[:3]], max_new_tokens=5)
    assert torch.equal(before, model.generate(ids, **kw))
