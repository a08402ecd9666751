"""Grouped-query attention on the H100: the grouped flash-attention forward and backward against fp32 autograd on
expanded K/V, their determinism and the r = 1 identity with the MHA path, the grouped decode kernel and cache append,
and generation / training of a GQA Llama on the native kernels."""
import pytest
import torch

from libai_b200.config import DictConfig
from libai_b200.ops import functional as OF

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def rel_err(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-6))


def _kv_mask(kv_lens, s):
    return None if kv_lens is None else (torch.arange(s, device=DEV)[None, :] < kv_lens[:, None].long())[:, None, None, :]


def _ref_grads(q, k, v, go, causal, scale, kv_lens):
    """fp32 autograd through attention_ref, K/V repeated to the query heads inside it (dK/dV = the group sums)."""
    qf, kf, vf = (t.detach().float().requires_grad_() for t in (q, k, v))
    o = OF.attention_ref(qf, kf, vf, causal=causal, scale=scale, mask=_kv_mask(kv_lens, q.shape[2]))
    o = o.float() if o.dtype != torch.float32 else o
    o.backward(go.float())
    return o.detach(), qf.grad, kf.grad, vf.grad


CASES = [(8, 8), (8, 4), (8, 2), (8, 1), (14, 2)]


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("padded", [False, True])
def test_grouped_attention_matches_fp32_autograd(D, causal, padded):
    B, S, scale = 2, 200, D ** -0.5
    errs = {}
    for A, G in CASES:
        g = torch.Generator(device=DEV).manual_seed(A * 100 + G)
        kv_lens = torch.tensor([S, 131], dtype=torch.int32, device=DEV) if padded else None
        q = torch.randn(B, A, S, D, device=DEV, generator=g).bfloat16().requires_grad_()
        k = torch.randn(B, G, S, D, device=DEV, generator=g).bfloat16().requires_grad_()
        v = torch.randn(B, G, S, D, device=DEV, generator=g).bfloat16().requires_grad_()
        go = torch.randn(B, A, S, D, device=DEV, generator=g).bfloat16()
        o_ref, dq_ref, dk_ref, dv_ref = _ref_grads(q, k, v, go, causal, scale, kv_lens)

        o = OF.attention(q, k, v, causal=causal, scale=scale, kv_lens=kv_lens)
        o.backward(go)
        errs[("4d", A, G)] = [rel_err(o, o_ref), rel_err(q.grad, dq_ref), rel_err(k.grad, dk_ref), rel_err(v.grad, dv_ref)]

        # the same problem through the grouped packed projection [B, S, G, r + 2, D]
        r = A // G
        qkv = torch.cat([q.detach().view(B, G, r, S, D), k.detach()[:, :, None], v.detach()[:, :, None]], 2)
        qkv = qkv.permute(0, 3, 1, 2, 4).contiguous().requires_grad_()
        ctx = OF.attention_qkvpacked(qkv, causal=causal, scale=scale, kv_lens=kv_lens)
        assert ctx.shape == (B, S, A, D)
        ctx.backward(go.permute(0, 2, 1, 3))
        dg = qkv.grad.permute(0, 2, 3, 1, 4)   # [B, G, r + 2, S, D]
        errs[("packed", A, G)] = [rel_err(ctx.permute(0, 2, 1, 3), o_ref), rel_err(dg[:, :, :r].reshape(B, A, S, D), dq_ref),
                                  rel_err(dg[:, :, r], dk_ref), rel_err(dg[:, :, r + 1], dv_ref)]
    bad = {key: e for key, e in errs.items() if not max(e) < 3e-2}
    assert not bad, bad


def test_grouped_backward_is_bit_identical_run_to_run():
    B, A, G, S, D = 2, 8, 2, 384, 128
    g = torch.Generator(device=DEV).manual_seed(0)
    qkv = torch.randn(B, S, G, A // G + 2, D, device=DEV, generator=g).bfloat16()
    go = torch.randn(B, S, A, D, device=DEV, generator=g).bfloat16()
    outs = []
    for _ in range(2):
        x = qkv.clone().requires_grad_()
        y = OF.attention_qkvpacked(x, causal=True, scale=0.1)
        y.backward(go)
        outs.append((y.detach(), x.grad))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("D", [64, 128])
def test_r1_grouped_path_is_bit_identical_to_mha(D):
    B, A, S = 2, 6, 320
    g = torch.Generator(device=DEV).manual_seed(1)
    qkv = torch.randn(B, S, A, 3 * D, device=DEV, generator=g).bfloat16()
    go = torch.randn(B, S, A, D, device=DEV, generator=g).bfloat16()
    res = []
    for x in (qkv.clone(), qkv.clone().view(B, S, A, 3, D)):
        x.requires_grad_()
        y = OF.attention_qkvpacked(x, causal=True, scale=D ** -0.5)
        y.backward(go)
        res.append((y.detach(), x.grad.reshape(B, S, A, 3 * D)))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


# ------------------------------------------------------------------------------------------------ decode
def _case(B, G, r, D, sq, L, cap_extra=37, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    C = L + sq + cap_extra
    k = torch.randn(B, G, C, D, device=DEV, generator=g).bfloat16()
    v = torch.randn(B, G, C, D, device=DEV, generator=g).bfloat16()
    q = torch.randn(B, sq, G * r, D, device=DEV, generator=g).bfloat16()
    lens = torch.tensor([max(L - 5 * b, 1) for b in range(B)], dtype=torch.int32, device=DEV)
    start = torch.tensor([(7 * b) % max(int(lens[b]), 1) if b % 2 else 0 for b in range(B)], dtype=torch.int32,
                         device=DEV)
    return q, k, v, lens, start


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("r", [1, 2, 4, 7, 8])
@pytest.mark.parametrize("sq", [1, 4, 16])
def test_grouped_decode_matches_reference(D, r, sq):
    errs = {}
    for L in (63, 1000):
        for splits in (1, 3, 0):
            q, k, v, lens, start = _case(3, 2, r, D, sq, L, seed=r * 1000 + L)
            got = OF.decode_attention(q, k, v, lens, start, scale=D ** -0.5, splits=splits)
            want = OF.decode_attention_ref(q, k, v, lens, start, scale=D ** -0.5)
            assert got.shape == (3, sq, 2 * r, D)
            errs[(L, splits)] = rel_err(got, want)
    bad = {key: e for key, e in errs.items() if not e < 3e-2}
    assert not bad, bad


def test_grouped_decode_no_visible_key_writes_zeros():
    q, k, v, lens, _ = _case(2, 2, 4, 64, 4, 100)
    start = lens + 4
    for splits in (0, 1):
        o = OF.decode_attention(q, k, v, lens, start.contiguous(), scale=0.125, splits=splits)
        assert torch.equal(o, torch.zeros_like(o))


def test_grouped_decode_graph_replay_after_lengths_bump():
    q, k, v, lens, start = _case(2, 2, 8, 128, 4, 500, cap_extra=300)
    OF.decode_attention(q, k, v, lens, start, scale=0.1)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = OF.decode_attention(q, k, v, lens, start, scale=0.1)
    lens.add_(200)
    graph.replay()
    eager = OF.decode_attention(q, k, v, lens, start, scale=0.1)
    assert torch.equal(out, eager)
    assert rel_err(out, OF.decode_attention_ref(q, k, v, lens, start, scale=0.1)) < 3e-2


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("r", [2, 4])
def test_grouped_kv_append_bit_identical_to_rope_qkv(D, r):
    from libai_b200.models.llama_model import rotary_tables

    B, sq, G, C = 3, 5, 2, 64
    cos, sin = rotary_tables(D, 128, device=DEV)
    qkv = torch.randn(B, sq, G, r + 2, D, device=DEV).bfloat16()
    k = torch.zeros(B, G, C, D, device=DEV, dtype=torch.bfloat16)
    v = torch.zeros_like(k)
    lens = torch.tensor([0, 7, 40], dtype=torch.int32, device=DEV)
    q = OF.kv_cache_append(qkv, k, v, lens, cos, sin)
    assert q.shape == (B, sq, G * r, D)
    for b in range(B):
        p = int(lens[b])
        want = OF.apply_rotary_qkv(qkv[b : b + 1].contiguous(), cos, sin, p)[0]     # the rope_qkv kernel
        assert torch.equal(q[b], want[:, :, :r].reshape(sq, G * r, D))
        assert torch.equal(k[b, :, p : p + sq], want[:, :, r].transpose(0, 1))
        assert torch.equal(v[b, :, p : p + sq], want[:, :, r + 1].transpose(0, 1))


# ------------------------------------------------------------------------------------------------ models
def _gqa_llama(head_dim, kv_heads=2):
    from libai_b200.layers._param import param_defaults
    from libai_b200.models import LlamaForCausalLM

    cfg = DictConfig(dict(hidden_layers=2, vocab_size=512, hidden_size=512, intermediate_size=1024,
                          num_attention_heads=512 // head_dim, num_key_value_heads=kv_heads, max_position_embeddings=256,
                          rms_norm_eps=1e-5, initializer_range=0.02, use_scaled_init_for_output_weights=True,
                          scale_mask_softmax_fusion=False, amp_enabled=True, bos_token_id=1, eos_token_id=2,
                          pad_token_id=0))
    with param_defaults(dtype=torch.bfloat16, device=DEV, seed=1234):
        return LlamaForCausalLM(cfg)


@pytest.mark.parametrize("head_dim", [64, 128])
def test_gqa_llama_generate_runs_native_decode(head_dim, monkeypatch):
    from tests.test_decode_gpu import _native_decoding, _teacher_forced

    model = _gqa_llama(head_dim).eval()
    torch.manual_seed(0)
    ids = torch.randint(3, 512, (3, 16), device=DEV)
    seqs, steps = _native_decoding(model, monkeypatch, ids)
    assert model.kv_cache.heads == 2
    ref = _teacher_forced(model, seqs, 16)
    assert rel_err(steps, ref) < 3e-2, rel_err(steps, ref)
    am = torch.ones_like(ids)
    ids[1, :5], am[1, :5] = 0, 0
    seqs, steps = _native_decoding(model, monkeypatch, ids, attention_mask=am)
    full_mask = torch.cat([am, torch.ones_like(seqs[:, 16:])], 1)
    ref = _teacher_forced(model, seqs, 16, full_mask)
    assert rel_err(steps, ref) < 3e-2, rel_err(steps, ref)


def test_llama_built_on_the_gpu_trains_through_forward_stage(monkeypatch):
    """A model built under ``param_defaults(device=...)`` holds its rotary tables on that device, so a training step
    through ``forward_stage`` (the blocks' path in the trainer and the pipeline schedules) rotates on the native
    kernel without being moved first."""
    from libai_b200 import ops

    def refuse(*a, **k):
        raise AssertionError("the reference rotary must not run on the native path")

    monkeypatch.setenv("LIBAI_B200_IMPL", "native")
    monkeypatch.setattr(OF, "rotate_half", refuse)
    model = _gqa_llama(128).train()
    ids = torch.randint(3, 512, (2, 128), device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    ops.reset_launch_count()
    loss = model.forward_stage({"input_ids": ids, "labels": ids})["lm_loss"]
    loss.backward()
    assert ops.launch_count() > 0
    assert torch.isfinite(loss)
    assert all(torch.isfinite(p.grad).all() for p in model.parameters())


def test_gqa_llama_training_is_bit_identical_run_to_run():
    def run():
        model = _gqa_llama(128).train()
        opt = torch.optim.SGD(model.parameters(), lr=0.05)
        g = torch.Generator(device=DEV).manual_seed(7)
        losses = []
        for _ in range(3):
            ids = torch.randint(3, 512, (4, 192), device=DEV, generator=g)
            loss = model(ids, labels=ids)["lm_loss"]
            loss.backward()
            opt.step()
            opt.zero_grad(set_to_none=True)
            losses.append(loss.detach().float())
        return torch.stack(losses), [p.detach().clone() for p in model.parameters()]

    l1, p1 = run()
    l2, p2 = run()
    assert torch.isfinite(l1).all()
    assert torch.equal(l1, l2)
    assert all(torch.equal(a, b) for a, b in zip(p1, p2))
