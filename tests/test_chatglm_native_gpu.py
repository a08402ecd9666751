"""ChatGLM2/3 on the H100: the GLM rotary packing kernel against the PyTorch rotary (bit for bit) and fp64 autograd, the
model's native forward against the rotary + ``repeat_interleave`` composition it replaces, a training step, and cached
generation running the decode kernels in every layer."""
import pytest
import torch

from libai_b200 import ops
from libai_b200.config import LazyConfig, instantiate
from libai_b200.ops import functional as OF
from tests.test_chatglm_native_cpu import _old_attention_forward

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _own_rng():
    """These tests seed and draw from the global generators; the tests after them see the state they would have seen
    without them."""
    with torch.random.fork_rng(devices=[0]):
        yield


def rel_err(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-6))


def _positions(b, s, P, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randperm(P, generator=g)[:s] for _ in range(b)]).to(DEV)


def _rotate64(x, rope):
    """fp64 GLM rotary of x ``[b, s, h, d]`` by ``rope`` ``[s, d/4, 2]``."""
    b, s, h, d = x.shape
    rot = rope.shape[-2] * 2
    xr = x[..., :rot].reshape(b, s, h, rot // 2, 2)
    c = rope.double()[None, :, None]
    out = torch.stack([xr[..., 0] * c[..., 0] - xr[..., 1] * c[..., 1], xr[..., 1] * c[..., 0] + xr[..., 0] * c[..., 1]], -1)
    return torch.cat([out.flatten(3), x[..., rot:]], dim=-1)


def _pack64(mixed, a, g, rope, grouped):
    b, s, _ = mixed.shape
    d = mixed.shape[-1] // (a + 2 * g)
    q, k, v = mixed.split([a * d, g * d, g * d], dim=-1)
    q, k, v = _rotate64(q.view(b, s, a, d), rope), _rotate64(k.view(b, s, g, d), rope), v.reshape(b, s, g, d)
    if grouped:
        return torch.cat([q.view(b, s, g, a // g, d), k.unsqueeze(3), v.unsqueeze(3)], dim=3)
    return torch.cat([q, k.repeat_interleave(a // g, dim=2), v.repeat_interleave(a // g, dim=2)], dim=-1)


CASES = [(0, False), (45, False), (0, True)]   # (pos_offset, with position_ids)


@pytest.mark.parametrize("grouped", [False, True])
@pytest.mark.parametrize("d", [64, 128])
def test_packing_forward_is_bit_identical_to_pytorch_rotary(d, grouped):
    torch.manual_seed(0)
    b, s, a, g, P = 2, 37, 8, 2, 96
    table = OF.glm_rope_table(P, d // 2, device=DEV)
    mixed = (torch.randn(b, s, (a + 2 * g) * d, device=DEV) * 3).to(torch.bfloat16)
    for offset, with_pos in CASES:
        pos = _positions(b, s, P, seed=offset + d) if with_pos else None
        before = ops.launch_count()
        out = OF.apply_glm_rotary_qkv(mixed, heads=a, kv_heads=g, table=table, pos_offset=offset, position_ids=pos,
                                      grouped=grouped)
        assert ops.launch_count() > before, "the packing kernel did not run"
        # the PyTorch rotary on the GPU (fp32 ops), stacked and repeated: every q/k slot, every K/V copy, v and the
        # unrotated halves
        ref = OF.apply_glm_rotary_qkv_ref(mixed, heads=a, kv_heads=g, table=table, pos_offset=offset, position_ids=pos,
                                          grouped=grouped)
        assert out.shape == ref.shape and torch.equal(out, ref), (offset, with_pos)


@pytest.mark.parametrize("grouped", [False, True])
@pytest.mark.parametrize("d", [64, 128])
def test_packing_backward_matches_fp64_and_is_deterministic(d, grouped):
    torch.manual_seed(1)
    b, s, a, g, P = 2, 29, 8, 2, 64
    table = OF.glm_rope_table(P, d // 2, device=DEV)
    mixed = torch.randn(b, s, (a + 2 * g) * d, device=DEV).to(torch.bfloat16)
    for offset, with_pos in ((0, False), (30, False), (0, True)):
        pos = _positions(b, s, P, seed=d) if with_pos else None
        rope = table[pos[0]] if with_pos else table[offset : offset + s]
        grads = []
        for _ in range(2):
            x = mixed.clone().requires_grad_()
            out = OF.apply_glm_rotary_qkv(x, heads=a, kv_heads=g, table=table, pos_offset=offset, position_ids=pos,
                                          grouped=grouped)
            if not grads:
                gy = torch.randn(out.shape, device=DEV).to(torch.bfloat16)
            out.backward(gy)
            grads.append(x.grad)
        assert torch.equal(grads[0], grads[1])
        x64 = mixed.double().requires_grad_()
        _pack64(x64, a, g, rope, grouped).backward(gy.double())
        err = (grads[0].double() - x64.grad).abs()
        assert bool((err <= 2.0 ** -8 * x64.grad.abs() + 1e-4).all()), float(err.max())


def test_binding_rejects_bad_arguments():
    ext = ops.load_ext()
    table = OF.glm_rope_table(16, 32, device=DEV)
    mixed = torch.randn(1, 8, 8 * 64, device=DEV).to(torch.bfloat16)
    with pytest.raises(RuntimeError, match="glm_rotary_qkv: bf16"):
        ext.glm_rotary_qkv(mixed.float(), 4, 2, table, 0, None, False)
    with pytest.raises(RuntimeError, match="glm_rotary_qkv: heads"):
        ext.glm_rotary_qkv(torch.randn(1, 8, 7 * 64, device=DEV).to(torch.bfloat16), 3, 2, table, 0, None, False)
    with pytest.raises(RuntimeError, match="glm_rotary_qkv: head dim"):
        ext.glm_rotary_qkv(torch.randn(1, 8, 8 * 6, device=DEV).to(torch.bfloat16), 4, 2, table, 0, None, False)
    with pytest.raises(RuntimeError, match="glm_rotary_qkv: table"):
        ext.glm_rotary_qkv(mixed, 4, 2, table.double(), 0, None, False)
    with pytest.raises(RuntimeError, match="glm_rotary_qkv: positions"):
        ext.glm_rotary_qkv(mixed, 4, 2, table, 9, None, False)
    with pytest.raises(RuntimeError, match="glm_rotary_qkv: position_ids must lie"):
        ext.glm_rotary_qkv(mixed, 4, 2, table, 0, torch.full((1, 8), 16, dtype=torch.int32, device=DEV), False)
    with pytest.raises(RuntimeError, match="glm_rotary_qkv: int32"):
        ext.glm_rotary_qkv(mixed, 4, 2, table, 0, torch.zeros(1, 8, dtype=torch.long, device=DEV), False)
    with pytest.raises(RuntimeError, match="glm_rotary_qkv_bwd: contiguous"):
        ext.glm_rotary_qkv_bwd(torch.randn(1, 8, 4, 6 * 64, device=DEV).to(torch.bfloat16)[..., : 3 * 64], 4, 2,
                               table, 0, None)


# ------------------------------------------------------------------------------------------------ the model
def _glm(d, dtype=torch.bfloat16, **over):
    c = LazyConfig.load("projects/ChatGLM/configs/chatglm_config.py")
    tiny = dict(num_layers=2, hidden_size=256, ffn_hidden_size=512, num_attention_heads=4, kv_channels=d,
                multi_query_group_num=2, padded_vocab_size=512, seq_length=256, pad_token_id=0)
    tiny.update(over)
    c = LazyConfig.apply_overrides(c, [f"cfg.{k}={v}" for k, v in tiny.items()])
    c.model.cfg = c.cfg
    torch.manual_seed(1234)
    m = instantiate(c.model).to(DEV, dtype)
    if c.cfg.lora_enable:   # nonzero adapters, so that the LoRA branch changes the function
        with torch.no_grad():
            for n, p in m.named_parameters():
                if "lora_B" in n:
                    p.normal_(std=0.05)
    return m


@pytest.mark.parametrize("d", [64, 128])
def test_native_forward_equals_old_composition(d, monkeypatch):
    from projects.ChatGLM.chatglm import SelfAttention

    m = _glm(d).eval()
    ids = torch.randint(3, 512, (2, 100), device=DEV)
    with torch.no_grad():
        new = m(ids)["logits"]
        monkeypatch.setattr(SelfAttention, "forward", _old_attention_forward)
        old = m(ids)["logits"]
    # the same values reach the same MHA flash kernel, through strided views of the packed projection instead of
    # repeated K/V tensors
    assert torch.equal(new, old)


@pytest.mark.parametrize("d", [64, 128])
def test_training_step_matches_fp32_and_is_deterministic(d):
    ids = torch.randint(3, 512, (2, 128), device=DEV)
    m = _glm(d).train()
    grads = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        m(ids, labels=ids)["loss"].backward()
        grads.append({n: p.grad.clone() for n, p in m.named_parameters()})
    for n in grads[0]:
        assert torch.equal(grads[0][n], grads[1][n]), n
    ref = _glm(d, torch.float32).train()   # the same weights in fp32: the reference math throughout
    ref.load_state_dict({k: v.float() for k, v in m.state_dict().items()})
    ref(ids, labels=ids)["loss"].backward()
    for n, p in ref.named_parameters():
        g, r = grads[0][n].float(), p.grad
        assert float((g - r).norm() / (r.norm() + 1e-12)) < 3e-2, n


def _native_generate(model, monkeypatch, ids, **kw):
    """Greedy cached generation (or beam search) in which every step after the prompt is written runs the native
    cache append and decode attention: the reference attention raises once the cache holds rows."""
    real_ref = OF.attention_ref

    def guarded(*a, **k):
        if model.kv_cache is not None and model.kv_cache.length > 0:
            raise AssertionError("a cached step fell back to the reference attention")
        return real_ref(*a, **k)

    def refuse(*a, **k):
        raise AssertionError("a cached step ran a reference op")

    launches = {"decode_attention": [], "kv_cache_append": []}

    def counting(name):
        real = getattr(OF, name)

        def fn(*a, **k):
            before = ops.launch_count()
            out = real(*a, **k)
            launches[name].append(ops.launch_count() - before)
            return out
        return fn

    monkeypatch.setattr(OF, "attention_ref", guarded)
    for name in ("decode_attention_ref", "kv_cache_append_ref", "apply_glm_rotary_qkv_ref"):
        monkeypatch.setattr(OF, name, refuse)
    for name in launches:
        monkeypatch.setattr(OF, name, counting(name))
    out = model.generate(ids, max_length=ids.shape[1] + 12, eos_token_id=None, pad_token_id=0, output_scores=True,
                         use_cache=True, **kw)
    monkeypatch.undo()
    dec, app = launches["decode_attention"], launches["kv_cache_append"]
    assert dec and all(c > 0 for c in dec) and app and all(c > 0 for c in app), (dec, app)
    assert len(app) == 12 * 2 and len(dec) >= 11 * 2   # two layers; every step after the prefill decodes
    return out


@pytest.mark.parametrize("case", ["plain", "left_padded", "prefix", "lora"])
@pytest.mark.parametrize("d", [64, 128])
def test_cached_generate_runs_native_decoding(d, case, monkeypatch):
    over = dict(pre_seq_len=6, prefix_projection=False) if case == "prefix" else \
        dict(lora_enable=True) if case == "lora" else {}
    m = _glm(d, **over).eval()
    torch.manual_seed(0)
    ids = torch.randint(3, 512, (3, 20), device=DEV)
    kw = {}
    if case == "left_padded":
        am = torch.ones_like(ids)
        ids[1, :5], am[1, :5] = 0, 0
        kw["attention_mask"] = am
    seqs, scores = _native_generate(m, monkeypatch, ids, **kw)
    steps = torch.stack(scores, 1)
    with torch.no_grad():   # teacher-forced, uncached
        if "attention_mask" in kw:
            full = torch.cat([kw["attention_mask"], torch.ones_like(seqs[:, 20:])], 1)
            logits = m(seqs[:, :-1], attention_mask=full[:, :-1])["logits"]
        else:
            logits = m(seqs[:, :-1])["logits"]
    ref = logits[:, 19:].float()
    assert rel_err(steps, ref) < 3e-2, rel_err(steps, ref)
    assert m.kv_cache.heads == 2


def test_beam_search_runs_on_the_cache(monkeypatch):
    m = _glm(128).eval()
    ids = torch.randint(3, 512, (2, 20), device=DEV)
    seqs = _native_generate(m, monkeypatch, ids, num_beams=2)[0]   # (sequences, sequence scores, step scores)
    assert seqs.shape == (2, 32) and m.kv_cache.batch == 4
