"""Flash attention at every head dim the kernels take (multiples of 8 up to 128) on the H100, per element against fp64
(tests/attention_ref.py states the bounds): O, lse, dQ, dK, dV over ragged and rectangular shapes, grouped heads and key
windows; dense bias with dbias, ALiBi and dropout on both tile widths; the packed 4-D and grouped 5-D projections with
every element of the packed gradient checked (a store past d would land in the neighbouring slot); q/k/v read as
column views of a wider buffer without touching its other columns; run-to-run and CUDA-graph determinism; and GPT-2,
BERT, MT5 and ViT at the recipes' head dims on the kernels, against the same models on the reference attention."""
import pytest
import torch

from libai_b200.config import DictConfig
from libai_b200.ops import functional as OF
from tests import attention_ref as R
from tests.dense_ref import check
from tests.test_attention_fp64_gpu import check_flash, rand, run_flash, windows

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

DIMS = [8, 16, 24, 32, 40, 48, 56, 72, 80, 88, 96, 104, 112, 120]
SHAPES = [(203, 203), (65, 129), (1000, 77), (77, 203), (1, 300), (129, 65)]
HEADS = [(4, 4), (4, 2), (4, 1)]
WINDOWS = ["none", "lens", "start_lens", "empty"]
TILE_DIMS = [24, 80]   # one head dim on the 64-wide tile, one on the 128-wide tile


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


def inputs(B, A, G, Sq, Sk, d, seed):
    return rand(B, A, Sq, d, seed=seed), rand(B, G, Sk, d, seed=seed + 1), rand(B, G, Sk, d, seed=seed + 2), \
        rand(B, A, Sq, d, seed=seed + 3)


# ------------------------------------------------------------------------------------------------ per element, every d
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("d", DIMS)
def test_flash_head_dim_per_element(ext, d, causal):
    # the (d, causal) pairs walk through the shapes, head groupings and key windows so that each d meets two of each
    n = 2 * DIMS.index(d) + causal
    Sq, Sk = SHAPES[n % len(SHAPES)]
    A, G = HEADS[n % len(HEADS)]
    wk = WINDOWS[n % len(WINDOWS)]
    B = 2
    q, k, v, do = inputs(B, A, G, Sq, Sk, d, seed=100 * d + causal)
    kv_start, kv_lens = windows(wk, B, Sq, Sk, causal)
    check_flash(ext, q, k, v, do, causal=causal, scale=d ** -0.5, kv_start=kv_start, kv_lens=kv_lens,
                what=f"d={d} Sq={Sq} Sk={Sk} causal={causal} A/G={A}/{G} window={wk}")


@pytest.mark.parametrize("d", TILE_DIMS)
@pytest.mark.parametrize("causal", [False, True])
def test_rows_without_a_visible_key_are_exact_zeros(ext, d, causal):
    B, A, G, Sq, Sk = 2, 4, 2, 77, 203
    q, k, v, do = inputs(B, A, G, Sq, Sk, d, seed=7 + d)
    kv_start, kv_lens = windows("empty", B, Sq, Sk, causal)
    got, _ = check_flash(ext, q, k, v, do, causal=causal, scale=d ** -0.5, kv_start=kv_start, kv_lens=kv_lens,
                         what=f"empty rows d={d} causal={causal}")
    vis = OF.visible_keys(Sq, Sk, causal=causal, kv_start=kv_start, kv_lens=kv_lens, device=DEV)
    empty = ~vis.any(-1)[:, 0]                                          # [B, Sq]
    assert empty.any()
    for name in ("o", "dq"):
        rows = got[name].reshape(B, A, Sq, d).permute(0, 2, 1, 3)[empty]
        assert rows.numel() and torch.equal(rows, torch.zeros_like(rows)), name
    lse = got["lse"].permute(0, 2, 1)[empty]
    assert torch.equal(lse, torch.zeros_like(lse))


# ------------------------------------------------------------------------------------------------ features at both tiles
@pytest.mark.parametrize("case", ["bias_1_a", "bias_b_1", "alibi", "dropout", "dropout_bias", "gqa", "mqa"])
@pytest.mark.parametrize("d", TILE_DIMS)
def test_flash_features_per_element(ext, d, case):
    B, A, G, Sq, Sk = 2, 8, 8, 203, 203
    if case in ("gqa", "mqa", "bias_1_a"):
        G = {"gqa": 2, "mqa": 1, "bias_1_a": 2}[case]
    if case.startswith("bias"):
        Sq, Sk = 77, 203
    q, k, v, do = inputs(B, A, G, Sq, Sk, d, seed=300 + d)
    kw = {}
    if case.startswith("bias") or case == "dropout_bias":
        bshape = {"bias_1_a": (1, A), "bias_b_1": (B, 1), "dropout_bias": (1, A)}[case]
        kw["bias"] = OF._prep_bias(rand(*bshape, Sq, Sk, seed=5, scale=2.0), q)
    if case == "alibi":
        kw["alibi"] = torch.tensor([2.0 ** (-8 * (h + 1) / A) for h in range(A)], device=DEV)
    if case.startswith("dropout"):
        kw["p"], kw["salt"] = 0.1, 3
    if case in ("gqa", "mqa"):
        kw["kv_start"], kw["kv_lens"] = windows("start_lens", B, Sq, Sk, True)
    for causal in (False, True):
        check_flash(ext, q, k, v, do, causal=causal, scale=d ** -0.5, what=f"{case} d={d} causal={causal}", **kw)


# ------------------------------------------------------------------------------------------------ packed projections
def _packed_expectation(ref, B, S, G, r, d):
    """{dq, dk, dv} references (value, bound) laid out as the packed gradient [B, S, G, r + 2, d]."""
    out = []
    for i in range(2):
        t = torch.empty(B, S, G, r + 2, d, dtype=torch.float64, device=DEV)
        t[:, :, :, :r] = ref["dq"][i].reshape(B, G, r, S, d).permute(0, 3, 1, 2, 4)
        t[:, :, :, r] = ref["dk"][i].permute(0, 2, 1, 3)
        t[:, :, :, r + 1] = ref["dv"][i].permute(0, 2, 1, 3)
        out.append(t)
    return out


@pytest.mark.parametrize("layout", ["4d", "grouped"])
@pytest.mark.parametrize("d", TILE_DIMS)
def test_packed_projection_gradient_every_element(ext, d, layout):
    B, S, A = 2, 203, 8
    G = A if layout == "4d" else 2
    r = A // G
    qkv_shape = (B, S, A, 3 * d) if layout == "4d" else (B, S, G, r + 2, d)
    qkv = rand(*qkv_shape, seed=11 + d)
    do = rand(B, S, A, d, seed=12 + d)
    scale = d ** -0.5
    q, k, v = OF._packed_views(qkv)
    q4 = q if q.dim() == 4 else q.reshape(B, A, S, d)
    for causal in (False, True):
        what = f"packed {layout} d={d} causal={causal}"
        o, lse, _ = ext.attn_fwd(q, k, v, causal, scale, None, None, None, 0.0, 0, None)
        _, _, _, dqkv = ext.attn_bwd(do.permute(0, 2, 1, 3), q, k, v, o, lse, causal, scale, None, None, None, None, 0.0,
                                     None, None)
        vis = OF.visible_keys(S, S, causal=causal, device=DEV)
        (ro, rob), (rl, rlb) = R.attention_fwd_ref(q4, k, v, scale=scale, vis=vis, tile=128)
        check(o, ro, rob, what + " o")
        check(lse, rl, rlb, what + " lse")
        ref = R.attention_bwd_ref(q4, k, v, do.permute(0, 2, 1, 3), o, lse, scale=scale, vis=vis)
        want, bound = _packed_expectation(ref, B, S, G, r, d)
        check(dqkv.view(B, S, G, r + 2, d), want, bound, what + " dqkv")
        # the public autograd path returns the same packed gradient, bit for bit
        x = qkv.detach().clone().requires_grad_()
        ctx = OF.attention_qkvpacked(x, causal=causal, scale=scale)
        assert torch.equal(ctx, o.permute(0, 2, 1, 3)), what
        ctx.backward(do)
        assert torch.equal(x.grad, dqkv.view(qkv.shape)), what


# ------------------------------------------------------------------------------------------------ strided views
@pytest.mark.parametrize("d", TILE_DIMS)
def test_column_views_do_not_read_neighbouring_columns(ext, d):
    """q, k, v are the first d columns of wider rows; the other columns hold sentinels.  The result passes the fp64
    check and is bit-identical when the sentinels change (to huge values and to NaN)."""
    B, A, G, Sq, Sk, extra = 2, 4, 2, 129, 203, 40
    q, k, v, do = inputs(B, A, G, Sq, Sk, d, seed=500 + d)
    results = []
    for sentinel in (0.0, 3e38, float("nan")):
        bufs = []
        for t in (q, k, v):
            w = torch.full((*t.shape[:-1], d + extra), sentinel, dtype=torch.bfloat16, device=DEV)
            w[..., :d] = t
            bufs.append(w[..., :d])
        assert bufs[0].stride(2) == d + extra
        for causal in (False, True):
            if sentinel == 0.0:
                got, _ = check_flash(ext, *bufs, do, causal=causal, scale=d ** -0.5, what=f"views d={d} causal={causal}")
            else:
                got, _ = run_flash(ext, *bufs, do, causal=causal, scale=d ** -0.5)
            results.append((sentinel, causal, got))
    for sentinel, causal, got in results[2:]:
        base = results[int(causal)][2]
        for name in ("o", "lse", "dq", "dk", "dv"):
            assert torch.equal(got[name].reshape(base[name].shape), base[name]), (sentinel, causal, name)


# ------------------------------------------------------------------------------------------------ determinism
@pytest.mark.parametrize("d", TILE_DIMS)
def test_bit_identical_across_runs_and_cuda_graph_replay(ext, d):
    B, A, G, Sq, Sk = 2, 8, 2, 1000, 1000
    q, k, v, do = inputs(B, A, G, Sq, Sk, d, seed=900 + d)
    bias = OF._prep_bias(rand(1, A, Sq, Sk, seed=901, scale=2.0), q)

    def step():
        got, _ = run_flash(ext, q, k, v, do, causal=True, scale=d ** -0.5, bias=bias, want_dbias=True)
        return got

    first, second = step(), step()
    for name in first:
        assert torch.equal(first[name], second[name]), name
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for name in first:
            assert torch.equal(captured[name], first[name]), name
    del graph


def test_unsupported_head_dims_are_refused(ext):
    for d in (20, 136):
        q = rand(1, 2, 16, d, seed=d)
        with pytest.raises(RuntimeError, match="multiple of 8 in"):
            ext.attn_fwd(q, q, q, True, 0.1, None, None, None, 0.0, 0, None)


# ------------------------------------------------------------------------------------------------ models
def rel_err(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-6))


def _gpt2():
    from libai_b200.models import GPTModel

    cfg = DictConfig(dict(
        hidden_layers=2, vocab_size=512, hidden_size=384, ffn_hidden_size=1536, num_attention_heads=16,
        max_seq_length=256, embedding_dropout_prob=0.0, attention_dropout_prob=0.0, output_dropout_prob=0.0,
        layernorm_epsilon=1e-5, initializer_range=0.02, use_scaled_init_for_output_weights=True, bias_gelu_fusion=True,
        bias_dropout_fusion=True, scale_mask_softmax_fusion=True, apply_query_key_layer_scaling=True,
        apply_residual_post_layernorm=False, amp_enabled=True))
    model = GPTModel(cfg)
    ids = torch.randint(0, 512, (2, 256), device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    return model, lambda: model(ids)


def _bert():
    from libai_b200.models import BertModel

    cfg = DictConfig(dict(
        vocab_size=512, hidden_size=768, hidden_layers=2, num_attention_heads=16, intermediate_size=1024,
        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, max_position_embeddings=512, num_tokentypes=2,
        add_pooling_layer=True, initializer_range=0.02, layernorm_eps=1e-5, bias_gelu_fusion=True,
        bias_dropout_fusion=True, scale_mask_softmax_fusion=True, apply_query_key_layer_scaling=True,
        apply_residual_post_layernorm=False, amp_enabled=True))
    model = BertModel(cfg)
    ids = torch.randint(1, 512, (2, 200), device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    am = torch.ones(2, 200, dtype=torch.long, device=DEV)
    am[1, 137:] = 0                                                   # right padding: kv_lens in the kernel
    # only the tokens: a padded query row sees its sample's keys in the kernel but every key under the dense mask of
    # the reference math, and a loss never reads it.  The final layer norm makes the sum of squares of its output
    # nearly constant, so the output is projected first (a test loss that depends on it)
    proj = torch.randn(768, 64, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5)).bfloat16()
    return model, lambda: model(ids, am)[0][am.bool()] @ proj


def _mt5():
    from projects.MT5.mt5_model import MT5Model

    cfg = DictConfig(dict(vocab_size=256, hidden_size=384, hidden_layers=2, num_attention_heads=12, head_size=32,
                          intermediate_size=768, embedding_dropout_prob=0.0, hidden_dropout_prob=0.0,
                          attention_probs_dropout_prob=0.0, relative_attention_num_buckets=32, initializer_range=0.02,
                          layernorm_eps=1e-6, amp_enabled=True, model_type="mt5", padding_idx=0,
                          is_encoder_decoder=True, tie_word_embeddings=False))
    model = MT5Model(cfg)
    g = torch.Generator(device=DEV).manual_seed(3)
    enc = torch.randint(2, 256, (2, 77), device=DEV, generator=g)
    dec = torch.randint(2, 256, (2, 30), device=DEV, generator=g)
    am = torch.ones(2, 77, dtype=torch.long, device=DEV)
    am[1, 50:] = 0
    return model, lambda: model(enc, dec, am)["logits"]


def _vit():
    from libai_b200.models import VisionTransformer

    model = VisionTransformer(img_size=224, patch_size=14, embed_dim=1280, depth=2, num_heads=16, num_classes=16)
    images = torch.randn(2, 3, 224, 224, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4)).bfloat16()
    return model, lambda: model(images)["prediction_scores"]


MODELS = {"gpt2_d24": _gpt2, "bert_d48": _bert, "mt5_d32": _mt5, "vit_d80": _vit}


@pytest.mark.parametrize("name", list(MODELS))
def test_model_runs_the_kernels_and_matches_reference_attention(monkeypatch, name):
    from libai_b200.layers._param import param_defaults

    monkeypatch.setenv("LIBAI_B200_IMPL", "native")
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
        model, run = MODELS[name]()
    model.train()
    results = {}
    real_ref = OF.attention_ref
    for arm in ("native", "attention_ref"):
        with monkeypatch.context() as m:
            if arm == "native":
                m.setattr(OF, "attention_ref", lambda *a, **k: pytest.fail("reference attention ran"))
            else:
                m.setattr(OF, "attention_supported", lambda *a, **k: False)
                m.setattr(OF, "attention_qkvpacked_supported", lambda *a, **k: False)
            model.zero_grad(set_to_none=True)
            out = run().float()
            out.square().mean().backward()
            results[arm] = (out.detach(), {n: p.grad.float().clone() for n, p in model.named_parameters()
                                           if p.grad is not None})
    assert OF.attention_ref is real_ref
    (ln, gn), (lr, gr) = results["native"], results["attention_ref"]
    assert gn.keys() == gr.keys() and gr
    errs = {"out": rel_err(ln, lr), **{n: rel_err(gn[n], gr[n]) for n in gr}}
    assert max(errs.values()) < 3e-2, errs
