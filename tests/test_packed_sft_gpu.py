"""Packed sequences on the H100: the flash kernels with ``doc_start`` against fp64 per element, their identity with the
plain causal kernels when every row is one document, rope_qkv with per-token positions, determinism and CUDA-graph
replay with a new packing, and a packed Llama / Qwen2-style training step against the same samples one per row."""
import random

import pytest
import torch

from libai_b200.ops import functional as OF
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


def doc_starts(kind, B, S, seed):
    """int32 [B, S] doc_start of a layout kind."""
    rng = random.Random(seed)
    rows = []
    for b in range(B):
        if kind == "one":
            ds = [0] * S
        elif kind == "short":      # many short documents
            ds, at = [], 0
            while at < S:
                n = rng.randint(1, 9)
                ds += [at] * min(n, S - at)
                at += n
        elif kind == "edges":      # lengths 1, tile - 1, tile, tile + 1 for both tile widths (64 and 128)
            ds, at, lens = [], 0, [1, 63, 64, 65, 127, 128, 129, 1]
            while at < S:
                n = lens[rng.randrange(len(lens))]
                ds += [at] * min(n, S - at)
                at += n
        else:                      # arbitrary: non-monotone, out of range
            ds = [i - rng.randint(-3, 150) if rng.random() < 0.8 else rng.randint(-10, S + 10) for i in range(S)]
        rows.append(ds)
    return torch.tensor(rows, dtype=torch.int32, device=DEV)


def packed_qkv(B, S, G, r, D, seed):
    """[B, S, A, 3D] (r = 1 and G = A: MHA) or grouped [B, S, G, r + 2, D]."""
    if r == 1:
        return rand(B, S, G, 3 * D, seed=seed)
    return rand(B, S, G, r + 2, D, seed=seed)


def run(ext, qkv, do, doc_start, scale):
    q, k, v = OF._packed_views(qkv)
    o, lse, _ = ext.attn_fwd(q, k, v, True, scale, None, None, None, 0.0, 0, None, doc_start)
    dq, dk, dv, dqkv = ext.attn_bwd(do, q, k, v, o, lse, True, scale, None, None, None, None, 0.0, None, None, doc_start)
    return dict(o=o, lse=lse, dq=dq, dk=dk, dv=dv, dqkv=dqkv)


CASES = [  # (D, G, r, S, kind)
    (64, 4, 1, 300, "short"), (64, 2, 3, 517, "edges"), (64, 4, 1, 256, "random"), (64, 2, 2, 200, "one"),
    (128, 2, 1, 300, "edges"), (128, 1, 4, 257, "short"), (128, 2, 2, 384, "random"),
    (24, 3, 1, 333, "edges"), (80, 1, 2, 211, "random"), (80, 2, 1, 129, "short"),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "D{}-G{}-r{}-S{}-{}".format(*c))
def test_doc_start_per_element(ext, case):
    D, G, r, S, kind = case
    B, A = 2, G * r
    seed = D * 1000 + S
    qkv = packed_qkv(B, S, G, r, D, seed)
    do = rand(B, A, S, D, seed=seed + 1)
    ds = doc_starts(kind, B, S, seed)
    got = run(ext, qkv, do, ds, D ** -0.5)
    q, k, v = OF._packed_views(qkv)
    q4 = q if q.dim() == 4 else q.reshape(B, A, S, D)
    vis = OF.visible_keys(S, S, causal=True, doc_start=ds, device=DEV)
    (o, ob), (lse, lseb) = R.attention_fwd_ref(q4, k, v, scale=D ** -0.5, vis=vis, tile=128)
    what = f"D={D} G={G} r={r} S={S} {kind}"
    check(got["o"], o, ob, what + " o")
    check(got["lse"], lse, lseb, what + " lse")
    ref = R.attention_bwd_ref(q4, k, v, do, got["o"], got["lse"], scale=D ** -0.5, vis=vis)
    R.check_all({"dq": got["dq"].reshape(B, A, S, D), "dk": got["dk"], "dv": got["dv"]}, ref, what)


@pytest.mark.parametrize("D,G,r", [(64, 4, 1), (128, 2, 2), (80, 1, 3)])
def test_zero_doc_start_is_bit_identical_to_plain_causal(ext, D, G, r):
    B, S = 2, 389
    qkv = packed_qkv(B, S, G, r, D, 7)
    do = rand(B, G * r, S, D, seed=8)
    a = run(ext, qkv, do, torch.zeros(B, S, dtype=torch.int32, device=DEV), D ** -0.5)
    q, k, v = OF._packed_views(qkv)
    o, lse, _ = ext.attn_fwd(q, k, v, True, D ** -0.5, None)
    dq, dk, dv, dqkv = ext.attn_bwd(do, q, k, v, o, lse, True, D ** -0.5, None)
    for name, x in (("o", o), ("lse", lse), ("dqkv", dqkv)):
        assert torch.equal(a[name], x), name
    # and repeated runs with a packing are bit-identical (ordered dQ sums, skipped visits included)
    ds = doc_starts("short", B, S, 3)
    first, second = run(ext, qkv, do, ds, D ** -0.5), run(ext, qkv, do, ds, D ** -0.5)
    for name in ("o", "lse", "dqkv"):
        assert torch.equal(first[name], second[name]), name


def test_doc_start_arguments_are_validated(ext):
    B, S, D = 2, 64, 64
    qkv = packed_qkv(B, S, 2, 1, D, 1)
    q, k, v = OF._packed_views(qkv)
    good = torch.zeros(B, S, dtype=torch.int32, device=DEV)
    for bad in (good.long(), good[:, :-1], good.t().contiguous().t(), good.cpu()):
        with pytest.raises(RuntimeError, match="doc_start"):
            ext.attn_fwd(q, k, v, True, 0.125, None, None, None, 0.0, 0, None, bad)
    with pytest.raises(RuntimeError, match="causal self-attention"):
        ext.attn_fwd(q, k, v, False, 0.125, None, None, None, 0.0, 0, None, good)
    with pytest.raises(RuntimeError, match="causal self-attention"):
        ext.attn_fwd(q, k, v, True, 0.125, torch.full((B,), S, dtype=torch.int32, device=DEV), None, None, 0.0, 0,
                     None, good)


@pytest.mark.parametrize("shape", [(2, 37, 4, 3 * 64), (2, 37, 2, 5, 128), (1, 20, 3, 3 * 24)])
def test_rope_positions(ext, shape):
    from libai_b200.models.llama_model import rotary_tables

    D = shape[-1] // 3 if len(shape) == 4 else shape[-1]
    cos, sin = (t.to(DEV) for t in rotary_tables(D, 128))
    qkv = rand(*shape, seed=5)
    B, S = shape[:2]
    pos = (torch.arange(S, device=DEV, dtype=torch.int32) + 11)[None].expand(B, S).contiguous()
    for bwd in (False, True):
        assert torch.equal(ext.rope_qkv(qkv, cos, sin, 11, bwd, False, None), ext.rope_qkv(qkv, cos, sin, 0, bwd, False, pos))
    # arbitrary positions against the reference gather
    pos = torch.randint(0, 128, (B, S), device=DEV, dtype=torch.int32)
    got = ext.rope_qkv(qkv, cos, sin, 0, False, False, pos)
    q5 = qkv.float()
    idx = pos.long()
    c, s = cos[idx], sin[idx]
    if len(shape) == 4:
        c, s = c[:, :, None], s[:, :, None]
        parts = [q5[..., :D], q5[..., D : 2 * D]]
        want = torch.cat([p * c + OF.rotate_half(p) * s for p in parts] + [q5[..., 2 * D :]], -1)
    else:
        c, s = c[:, :, None, None], s[:, :, None, None]
        r = shape[3] - 2
        want = torch.cat([q5[..., : r + 1, :] * c + OF.rotate_half(q5[..., : r + 1, :]) * s, q5[..., r + 1 :, :]], 3)
    torch.testing.assert_close(got.float(), want, rtol=2 ** -7, atol=2 ** -7)


def test_graph_replay_with_new_packing_matches_eager(ext):
    B, S, G, r, D = 2, 300, 2, 2, 64
    qkv = packed_qkv(B, S, G, r, D, 11)
    do = rand(B, G * r, S, D, seed=12)
    static_ds = doc_starts("short", B, S, 1)
    run(ext, qkv, do, static_ds, 0.125)   # warm-up (one-time kernel attributes)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = run(ext, qkv, do, static_ds, 0.125)
    for kind, seed in (("edges", 2), ("random", 3), ("one", 4)):
        ds = doc_starts(kind, B, S, seed)
        static_ds.copy_(ds)
        g.replay()
        eager = run(ext, qkv, do, ds, 0.125)
        for name in ("o", "lse", "dqkv"):
            assert torch.equal(out[name], eager[name]), (kind, name)


# ------------------------------------------------------------------------------------------------ model
def _model(g, qkv_bias, dtype):
    from libai_b200.layers._param import param_defaults
    from libai_b200.models.llama_model import LlamaForCausalLM

    with param_defaults(dtype=dtype, device=DEV, seed=1234):
        return LlamaForCausalLM(hidden_layers=2, vocab_size=256, hidden_size=256, intermediate_size=512,
                                num_attention_heads=4, max_position_embeddings=512, qkv_bias=qkv_bias,
                                num_key_value_heads=g, amp_enabled=dtype == torch.bfloat16).to(DEV)


def _batches(L=256, seed=0):
    g = torch.Generator().manual_seed(seed)
    lens = [int(x) for x in torch.randint(2, 120, (9,), generator=g)]
    docs = []
    for n in lens:
        ids = torch.randint(1, 256, (n,), generator=g)
        lab = torch.full((n,), -1)
        lab[n // 4 : n - 1] = ids[n // 4 + 1 :]
        docs.append((ids, lab))
    rows, cur, used = [], [], 0
    for d in docs:
        if used + len(d[0]) > L:
            rows.append(cur)
            cur, used = [], 0
        cur.append(d)
        used += len(d[0])
    rows.append(cur)

    def row(ds):
        ids, lab, pos = torch.zeros(L, dtype=torch.long), torch.full((L,), -1), torch.zeros(L, dtype=torch.long)
        at = 0
        for i, l in ds:
            n = len(i)
            ids[at : at + n], lab[at : at + n], pos[at : at + n] = i, l, torch.arange(n)
            at += n
        pos[at:] = torch.arange(L - at)
        return ids, lab, pos

    packed = [row(r) for r in rows]
    padded = [row([d]) for d in docs]
    mk = lambda rs, with_pos: dict(input_ids=torch.stack([x[0] for x in rs]).to(DEV),
                                   labels=torch.stack([x[1] for x in rs]).to(DEV),
                                   **({"position_ids": torch.stack([x[2] for x in rs]).to(DEV)} if with_pos else {}))
    return mk(packed, True), mk(padded, False)


def _step(model, batch):
    model.zero_grad()
    loss = model(**batch)["lm_loss"]
    loss.backward()
    grads = {n: (p.grad if p.grad is not None else p.main_grad).detach().float().clone()
             for n, p in model.named_parameters()}
    for p in model.parameters():
        if getattr(p, "main_grad", None) is not None:
            p.main_grad.zero_()
    return loss.detach().float(), grads


@pytest.mark.parametrize("g,qkv_bias", [(4, False), (2, True)], ids=["llama", "qwen2-gqa"])
def test_packed_training_step_runs_native_and_matches_padded(monkeypatch, g, qkv_bias):
    packed, padded = _batches()
    fp32 = _model(g, qkv_bias, torch.float32)
    ref = _step(fp32, padded)    # fp32 reference (reference math on fp32)
    model = _model(g, qkv_bias, torch.bfloat16)
    model.load_state_dict(fp32.state_dict())

    def boom(*a, **k):
        raise AssertionError("attention_ref must not run on the native path")

    monkeypatch.setattr(OF, "attention_ref", boom)
    got_pad = _step(model, padded)
    got_pk = _step(model, packed)
    # the packed run may be no further from fp32 than twice the padded run, plus 5 % of each quantity's largest element
    for name in ["loss"] + list(ref[1]):
        r = ref[0] if name == "loss" else ref[1][name]
        p = got_pad[0] if name == "loss" else got_pad[1][name]
        k = got_pk[0] if name == "loss" else got_pk[1][name]
        dist_pad = float((p - r).abs().max())
        dist_pk = float((k - r).abs().max())
        assert dist_pk <= 2 * dist_pad + 0.05 * float(r.abs().max()) + 1e-6, (name, dist_pk, dist_pad)


# ------------------------------------------------------------------------------------------------ trainer + CUDA graphs
def _sft_corpus(n, L, seed):
    g = torch.Generator().manual_seed(seed)
    data = []
    for _ in range(n):
        full = int(torch.randint(4, L // 2, (1,), generator=g))
        prompt = int(torch.randint(1, full - 1, (1,), generator=g))
        ids = torch.cat([torch.randint(3, 256, (full,), generator=g), torch.zeros(L - full, dtype=torch.long)])
        labels = torch.full((L,), -1)
        labels[prompt - 1 : full - 1] = ids[prompt:full]
        data.append({"input_ids": ids, "labels": labels})
    return data


def test_trainer_steps_with_packed_dataset_and_cuda_graphs_match_eager():
    """StepTrainer.train_on_batches (the step DefaultTrainer runs) on PackedSFTDataset rows: with CUDA graphs on, the
    blocks are captured through engine/cuda_graphs with position_ids / doc_start as graph inputs and replayed with a
    different packing at every step; losses and parameters follow the eager steps."""
    import os

    from libai_b200.config import DictConfig
    from libai_b200.engine.trainer import StepTrainer
    from libai_b200.layers._param import param_defaults
    from libai_b200.models.llama_model import LlamaForCausalLM
    from libai_b200.optim import AdamW, get_default_optimizer_params
    from libai_b200.utils import distributed as dutil
    from projects.common.sft import PackedSFTDataset

    os.environ["LIBAI_B200_IMPL"] = "native"
    L = 256
    ds = PackedSFTDataset(_sft_corpus(120, L, seed=5), L)
    rows = [{k: ds[i].get(k).tensor for k in ("input_ids", "labels", "position_ids")} for i in range(len(ds))]
    steps = []
    for s in range(4):      # 2 micro-batches of 2 packed rows per step
        mbs = []
        for m in range(2):
            part = rows[(4 * s + 2 * m) % len(rows):][:2]
            mbs.append({k: torch.stack([r[k] for r in part]).to(DEV) for k in part[0]})
        steps.append(mbs)
    assert not torch.equal(steps[0][0]["position_ids"], steps[1][0]["position_ids"])
    runs = {}
    for graphed in (False, True):
        dutil.reset_dist_util()
        dutil.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1)))
        with param_defaults(dtype=torch.bfloat16, device=DEV, seed=3):
            model = LlamaForCausalLM(hidden_layers=2, vocab_size=256, hidden_size=256, intermediate_size=512,
                                     num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=L,
                                     amp_enabled=True).to(DEV).train()
        opt = AdamW(get_default_optimizer_params(model, clip_grad_max_norm=1.0, clip_grad_norm_type=2.0), lr=1e-3)
        opt.configure(param_names={id(p): n for n, p in model.named_parameters()})
        opt.setup()
        trainer = StepTrainer(model, [], opt, grad_acc_steps=2)
        trainer.cuda_graphs = graphed
        losses = [float(trainer.train_on_batches(mbs)["lm_loss"]) for mbs in steps]
        assert trainer.graphs_enabled == graphed
        runs[graphed] = (losses, {n: p.detach().float().clone() for n, p in model.named_parameters()})
    (eager, pe), (graph, pg) = runs[False], runs[True]
    assert all(abs(a - b) < 1e-2 for a, b in zip(eager, graph)), (eager, graph)
    for n in pe:
        assert torch.allclose(pe[n], pg[n], rtol=2e-2, atol=2e-3), (n, float((pe[n] - pg[n]).abs().max()))
