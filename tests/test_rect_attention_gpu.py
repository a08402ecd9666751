"""Rectangular flash attention on the H100: forward and backward with independent query and key lengths, per-sample key
windows (kv_start / kv_lens), bottom-right causal alignment, rectangular dense bias and ALiBi against fp32 autograd;
exact zeros outside the windows, determinism and the identities with the square path; left-padded and chunked Llama
prefill on the kernels, the memory of a long left-padded prefill, and MT5 cross-attention on the kernels."""
import pytest
import torch

from libai_b200 import ops
from libai_b200.config import DictConfig
from libai_b200.ops import functional as OF

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def rel_err(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-6))


def _inputs(B, A, G, sq, sk, D, seed, bias_shape=None):
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = torch.randn(B, A, sq, D, device=DEV, generator=g).bfloat16().requires_grad_()
    k = torch.randn(B, G, sk, D, device=DEV, generator=g).bfloat16().requires_grad_()
    v = torch.randn(B, G, sk, D, device=DEV, generator=g).bfloat16().requires_grad_()
    go = torch.randn(B, A, sq, D, device=DEV, generator=g).bfloat16()
    bias = None
    if bias_shape is not None:
        bias = torch.randn(*bias_shape, sq, sk, device=DEV, generator=g).requires_grad_()
    return q, k, v, go, bias


def _ref(q, k, v, go, causal, scale, kv_start=None, kv_lens=None, bias=None, slopes=None):
    """fp32 autograd through attention_ref with the explicit visibility mask; rows without a visible key are zero."""
    sq, sk = q.shape[2], k.shape[2]
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    bf = None if bias is None else bias.detach().float().requires_grad_()
    vis = OF.visible_keys(sq, sk, causal=causal, kv_start=kv_start, kv_lens=kv_lens, device=DEV)
    b = bf
    if slopes is not None:
        rel = torch.arange(sk, device=DEV)[None, :] - (torch.arange(sq, device=DEV)[:, None] + sk - sq)
        b = slopes[None, :, None, None] * rel[None, None].float()
    o = OF.attention_ref(qf, kf, vf, causal=False, scale=scale, mask=vis, bias=b)
    o = o.masked_fill(~vis.any(-1, keepdim=True), 0)
    o.backward(go.float())
    return o.detach(), qf.grad, kf.grad, vf.grad, (None if bf is None else bf.grad)


def _native(q, k, v, go, causal, scale, **kw):
    for t in (q, k, v):
        t.grad = None
    bias = kw.get("bias")
    if bias is not None:
        bias.grad = None
    o = OF.attention(q, k, v, causal=causal, scale=scale, **kw)
    o.backward(go)
    return o.detach(), q.grad, k.grad, v.grad, (None if bias is None else bias.grad)


SHAPES = [(1, 300), (77, 203), (203, 77), (128, 1000), (300, 300)]
GROUPS = [(8, 8), (8, 2), (8, 1)]


def _windows(B, sk):
    yield "none", None, None
    yield "lens", None, torch.tensor([sk, max(1, sk - 37)], dtype=torch.int32, device=DEV)
    yield ("start+lens", torch.tensor([min(5, sk - 1), sk // 3], dtype=torch.int32, device=DEV),
           torch.tensor([sk, max(1, sk - 7)], dtype=torch.int32, device=DEV))


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal", [True, False])
def test_rect_attention_matches_fp32_autograd(D, causal):
    B, scale = 2, D ** -0.5
    errs = {}
    for sq, sk in SHAPES:
        for A, G in GROUPS:
            q, k, v, go, _ = _inputs(B, A, G, sq, sk, D, seed=sq * 7 + sk + G)
            for name, kv_start, kv_lens in _windows(B, sk):
                ref = _ref(q, k, v, go, causal, scale, kv_start, kv_lens)
                got = _native(q, k, v, go, causal, scale, kv_start=kv_start, kv_lens=kv_lens)
                assert all(torch.isfinite(t).all() for t in got[:4])
                errs[(sq, sk, A, G, name)] = [rel_err(a, b) for a, b in zip(got[:4], ref[:4])]
    bad = {key: e for key, e in errs.items() if not max(e) < 3e-2}
    assert not bad, bad


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal", [True, False])
def test_rect_attention_bias_and_alibi(D, causal):
    B, A, G, scale = 2, 8, 2, D ** -0.5
    errs = {}
    for sq, sk in [(77, 203), (203, 77), (64, 129)]:
        kv_start = torch.tensor([3, sk // 4], dtype=torch.int32, device=DEV)
        for bshape in [(1, A), (B, 1)]:   # dense bias with its gradient; sk odd or not a multiple of 8
            q, k, v, go, bias = _inputs(B, A, G, sq, sk, D, seed=sq + sk, bias_shape=bshape)
            ref = _ref(q, k, v, go, causal, scale, kv_start, bias=bias)
            got = _native(q, k, v, go, causal, scale, kv_start=kv_start, bias=bias)
            errs[(sq, sk, "bias", bshape)] = [rel_err(a, b) for a, b in zip(got, ref)]
        q, k, v, go, _ = _inputs(B, A, G, sq, sk, D, seed=sq + sk + 1)
        slopes = torch.tensor([2.0 ** (-(i + 1)) for i in range(A)], device=DEV)
        ref = _ref(q, k, v, go, causal, scale, kv_start, slopes=slopes)
        got = _native(q, k, v, go, causal, scale, kv_start=kv_start, alibi_slopes=slopes)
        errs[(sq, sk, "alibi")] = [rel_err(a, b) for a, b in zip(got[:4], ref[:4])]
    bad = {key: e for key, e in errs.items() if not max(e) < 3e-2}
    assert not bad, bad


def test_rows_and_keys_outside_the_window_are_exact_zeros():
    B, A, G, D, sq, sk = 2, 4, 2, 64, 200, 77
    q, k, v, go, _ = _inputs(B, A, G, sq, sk, D, seed=5)
    kv_start = torch.tensor([10, 70], dtype=torch.int32, device=DEV)
    kv_lens = torch.tensor([60, 77], dtype=torch.int32, device=DEV)
    o, dq, dk, dv, _ = _native(q, k, v, go, True, 0.125, kv_start=kv_start, kv_lens=kv_lens)
    off = sk - sq   # causal: query i sees keys j <= i + off
    for b, (beg, end) in enumerate([(10, 60), (70, 77)]):
        empty = beg - off   # rows i < beg - off see no key
        assert (o[b, :, :empty] == 0).all() and (dq[b, :, :empty] == 0).all()
        assert o[b, :, empty:].abs().sum() > 0
        hidden = torch.ones(sk, dtype=torch.bool, device=DEV)
        hidden[beg:end] = False
        assert (dk[b][:, hidden] == 0).all() and (dv[b][:, hidden] == 0).all()
    assert all(torch.isfinite(t).all() for t in (o, dq, dk, dv))
    _, lse, _ = ops.load_ext().attn_fwd(q.detach(), k.detach(), v.detach(), True, 0.125, kv_lens, None, None, 0.0, 0,
                                        kv_start)
    assert torch.isfinite(lse).all()


def _run(q, k, v, go, causal, **kw):
    return _native(q, k, v, go, causal, 0.1, **kw)[:4]


def test_rect_attention_is_bit_identical_run_to_run_with_dropout_and_kv_start():
    B, A, G, D, sq, sk = 2, 8, 2, 128, 333, 1000
    q, k, v, go, _ = _inputs(B, A, G, sq, sk, D, seed=9)
    kv_start = torch.tensor([17, 400], dtype=torch.int32, device=DEV)
    outs = []
    for _ in range(2):
        torch.manual_seed(0)
        outs.append(_run(q, k, v, go, True, kv_start=kv_start, dropout_p=0.1, training=True))
    assert all(torch.equal(a, b) for a, b in zip(*outs))


@pytest.mark.parametrize("sq,sk", [(77, 203), (256, 256), (200, 77)])
def test_zero_kv_start_and_full_kv_lens_are_bit_identical_to_none(sq, sk):
    B, A, G, D = 2, 8, 2, 64
    q, k, v, go, _ = _inputs(B, A, G, sq, sk, D, seed=sq + sk)
    for causal in (True, False):
        base = _run(q, k, v, go, causal)
        zero_start = _run(q, k, v, go, causal, kv_start=torch.zeros(B, dtype=torch.int32, device=DEV))
        full_lens = _run(q, k, v, go, causal, kv_lens=torch.full((B,), sk, dtype=torch.int32, device=DEV))
        assert all(torch.equal(a, b) for a, b in zip(base, zero_start))
        assert all(torch.equal(a, b) for a, b in zip(base, full_lens))


def test_kv_start_is_checked():
    q = torch.randn(2, 4, 8, 64, device=DEV).bfloat16()
    for bad in (torch.zeros(2, dtype=torch.int64, device=DEV), torch.zeros(3, dtype=torch.int32, device=DEV),
                torch.zeros(2, dtype=torch.int32)):
        with pytest.raises(RuntimeError, match="kv_start"):
            OF.attention(q, q, q, causal=True, kv_start=bad)


# ------------------------------------------------------------------------------------------------ Llama
def _llama(max_pos=1024, **kw):
    from libai_b200.layers._param import param_defaults
    from libai_b200.models import LlamaForCausalLM

    cfg = DictConfig(dict(dict(hidden_layers=2, vocab_size=512, hidden_size=256, intermediate_size=512,
                               num_attention_heads=4, max_position_embeddings=max_pos, rms_norm_eps=1e-5,
                               initializer_range=0.02, use_scaled_init_for_output_weights=True,
                               scale_mask_softmax_fusion=False, amp_enabled=True, bos_token_id=1, eos_token_id=2,
                               pad_token_id=0), **kw))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
        return LlamaForCausalLM(cfg).eval()


def _count_ref(monkeypatch):
    calls = []
    real = OF.attention_ref

    def counting(*a, **k):
        calls.append(a[0].shape)
        return real(*a, **k)

    monkeypatch.setattr(OF, "attention_ref", counting)
    monkeypatch.setattr(OF, "decode_attention_ref", lambda *a, **k: pytest.fail("reference decode attention ran"))
    return calls


def test_llama_left_padded_prefill_matches_unpadded_prompts(monkeypatch):
    model = _llama()
    torch.manual_seed(0)
    lens, S = [37, 200, 511, 512], 512
    prompts = [torch.randint(3, 512, (n,), device=DEV) for n in lens]
    ids = torch.zeros(len(lens), S, dtype=torch.long, device=DEV)
    am = torch.zeros_like(ids)
    for b, p in enumerate(prompts):
        ids[b, S - len(p):], am[b, S - len(p):] = p, 1
    calls = _count_ref(monkeypatch)
    with torch.no_grad():
        model.set_cache(None)
        batched = model(ids, attention_mask=am, use_cache=True)["logits"].float()
        assert calls == [], calls   # the prefill ran the flash kernel with kv_start, not the dense-mask reference
        # a decode step after it reads the same cache
        step = model(torch.full((len(lens), 1), 7, dtype=torch.long, device=DEV),
                     attention_mask=torch.cat([am, torch.ones_like(am[:, :1])], 1), use_cache=True)["logits"].float()
        monkeypatch.undo()
        for b, p in enumerate(prompts):
            model.set_cache(None)
            alone = model(p[None], use_cache=True)["logits"].float()
            alone_step = model(torch.full((1, 1), 7, dtype=torch.long, device=DEV), use_cache=True)["logits"].float()
            err = rel_err(batched[b, S - len(p):], alone[0])
            assert err < 3e-2, (len(p), err)
            assert rel_err(step[b], alone_step[0]) < 3e-2
    assert torch.isfinite(batched).all()


def test_llama_chunked_prefill_matches_one_piece(monkeypatch):
    model = _llama()
    torch.manual_seed(1)
    ids = torch.randint(3, 512, (2, 1000), device=DEV)
    runs = {}
    with torch.no_grad():
        for name, cuts in [("one", [1000]), ("600+400", [600, 400]), ("100s", [100] * 10)]:
            calls = _count_ref(monkeypatch)
            model.set_cache(None)
            logits, pos = [], 0
            for n in cuts:
                logits.append(model(ids[:, pos:pos + n], use_cache=True)["logits"].float())
                pos += n
            monkeypatch.undo()
            assert calls == [], (name, calls)
            c = model.kv_cache
            runs[name] = (torch.cat(logits, 1), [c.k[i][:, :, :1000].clone() for i in c.owned],
                          [c.v[i][:, :, :1000].clone() for i in c.owned])
    one = runs["one"]
    for name in ("600+400", "100s"):
        got = runs[name]
        assert rel_err(got[0], one[0]) < 3e-2, name
        for a, b in zip(got[1] + got[2], one[1] + one[2]):
            assert rel_err(a, b) < 3e-2, name


def test_llama_7b_layer_left_padded_prefill_memory():
    """One Llama-7B-shaped attention layer prefilling a left-padded 4 x 4096 batch: the reference would hold
    4 * 32 * 4096^2 fp32 scores (8.6 GB) alone."""
    from libai_b200.inference.kv_cache import StaticKVCache

    model = _llama(max_pos=4096, hidden_layers=1, hidden_size=4096, intermediate_size=256, num_attention_heads=32,
                   vocab_size=64)
    attn = model.model.layers[0].self_attn
    B, S = 4, 4096
    cache = StaticKVCache(1, B, 32, 128, S, torch.bfloat16, DEV)
    cache.kv_start.copy_(torch.tensor([0, 1000, 2000, 4000], dtype=torch.int32))
    cos, sin = model.model.cos_cached.to(DEV), model.model.sin_cached.to(DEV)
    hidden = torch.randn(B, S, 4096, device=DEV).bfloat16()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    with torch.no_grad():
        out = attn(hidden, None, cache.layer(0), cos, sin)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    assert extra < 2 * 2 ** 30, extra / 2 ** 30
    assert torch.isfinite(out).all()


# ------------------------------------------------------------------------------------------------ MT5
def _mt5():
    from libai_b200.layers._param import param_defaults
    from projects.MT5.mt5_model import MT5Model

    cfg = DictConfig(dict(vocab_size=256, hidden_size=256, hidden_layers=2, num_attention_heads=4, head_size=64,
                          intermediate_size=512, embedding_dropout_prob=0.0, hidden_dropout_prob=0.0,
                          attention_probs_dropout_prob=0.0, relative_attention_num_buckets=32, initializer_range=0.02,
                          layernorm_eps=1e-6, amp_enabled=True, model_type="mt5", padding_idx=0,
                          is_encoder_decoder=True, tie_word_embeddings=False))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=4321):
        return MT5Model(cfg)


def test_mt5_cross_attention_runs_the_kernel_and_matches_ref(monkeypatch):
    """Native against the same model with only the attention on the reference math (same GEMMs and norms), and against
    LIBAI_B200_IMPL=ref (every operator on PyTorch: bf16 GEMM and norm differences add up over the layers)."""
    model = _mt5()
    torch.manual_seed(2)
    enc, dec = torch.randint(2, 256, (2, 77), device=DEV), torch.randint(2, 256, (2, 30), device=DEV)
    am = torch.ones(2, 77, dtype=torch.long, device=DEV)
    am[1, 50:] = 0
    results = {}
    real_supported = OF.attention_supported
    for arm in ("native", "attention_ref", "ref"):
        monkeypatch.setenv("LIBAI_B200_IMPL", "ref" if arm == "ref" else "native")
        if arm == "attention_ref":
            monkeypatch.setattr(OF, "attention_supported", lambda *a, **k: False)
        calls = _count_ref(monkeypatch)
        model.zero_grad(set_to_none=True)
        logits = model(enc, dec, am)["logits"].float()
        logits.square().mean().backward()
        # native: encoder, decoder and cross-attention all on the flash kernels; otherwise all on the reference math
        assert (calls == []) if arm == "native" else len(calls) == 3 * 2, (arm, calls)
        results[arm] = (logits.detach(), {n: p.grad.float().clone() for n, p in model.named_parameters()
                                          if p.grad is not None})
        monkeypatch.undo()
    assert OF.attention_supported is real_supported
    errs = {}
    for arm in ("attention_ref", "ref"):
        (ln, gn), (lr, gr) = results["native"], results[arm]
        errs[arm] = {"logits": rel_err(ln, lr), **{n: rel_err(gn[n], gr[n]) for n in gr}}
    print({arm: max(e.values()) for arm, e in errs.items()}, errs["attention_ref"]["logits"], errs["ref"]["logits"])
    assert max(errs["attention_ref"].values()) < 5e-2, errs["attention_ref"]
    assert max(errs["ref"].values()) < 1e-1, errs["ref"]
