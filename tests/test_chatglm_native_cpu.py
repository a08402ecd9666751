"""ChatGLM2/3 on the native attention path, checked on the CPU: the GLM rotary packing reference against the rotary +
``repeat_interleave`` composition it replaces, the attention block's loss and gradients against that composition, and
cached generation (the preallocated ``StaticKVCache``) against uncached generation."""
import math

import pytest
import torch

from libai_b200.config import DictConfig, LazyConfig, instantiate
from libai_b200.inference.kv_cache import StaticKVCache
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cpu")))


@pytest.fixture(autouse=True)
def _own_rng():
    """These tests seed and draw from the global generators; the tests after them see the state they would have seen
    without them."""
    with torch.random.fork_rng(devices=[torch.cuda.current_device()] if torch.cuda.is_available() else []):
        yield


def _old_rotary(x, cache):
    """The rotary ChatGLM applied before the packing kernel, verbatim."""
    b, s, h, d = x.shape
    rot = cache.shape[-2] * 2
    xr, xp = x[..., :rot], x[..., rot:]
    xr = xr.float().reshape(b, s, h, rot // 2, 2)
    c = cache[:s].view(1, s, 1, rot // 2, 2)
    out = torch.stack([xr[..., 0] * c[..., 0] - xr[..., 1] * c[..., 1], xr[..., 1] * c[..., 0] + xr[..., 0] * c[..., 1]], -1)
    return torch.cat([out.flatten(3).to(x.dtype), xp], dim=-1)


def _old_qkv(mixed, a, g, rope):
    """q ``[b, a, s, d]`` and k, v ``[b, g, s, d]`` as the old attention block computed them."""
    b, s, _ = mixed.shape
    d = mixed.shape[-1] // (a + 2 * g)
    q, k, v = mixed.split([a * d, g * d, g * d], dim=-1)
    q, k, v = q.view(b, s, a, d), k.view(b, s, g, d), v.view(b, s, g, d)
    q, k = _old_rotary(q, rope), _old_rotary(k, rope)
    return q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("d", [16, 64])
def test_reference_packing_equals_old_composition(dtype, d):
    torch.manual_seed(0)
    b, s, a, g = 2, 7, 6, 2
    r = a // g
    table = OF.glm_rope_table(40, d // 2)
    mixed = torch.randn(b, s, (a + 2 * g) * d).to(dtype)
    pos = torch.stack([torch.randperm(40)[:s], torch.randperm(40)[:s]])
    for offset, position_ids in ((0, None), (9, None), (0, pos)):
        rope = table[position_ids[0]] if position_ids is not None else table[offset : offset + s]
        q, k, v = _old_qkv(mixed, a, g, rope)
        k_rep, v_rep = k.repeat_interleave(r, dim=1), v.repeat_interleave(r, dim=1)
        per_head = OF.apply_glm_rotary_qkv(mixed, heads=a, kv_heads=g, table=table, pos_offset=offset,
                                           position_ids=position_ids)
        assert per_head.shape == (b, s, a, 3 * d)
        assert torch.equal(per_head[..., :d], q.transpose(1, 2))
        assert torch.equal(per_head[..., d : 2 * d], k_rep.transpose(1, 2))
        assert torch.equal(per_head[..., 2 * d :], v_rep.transpose(1, 2))
        grouped = OF.apply_glm_rotary_qkv(mixed, heads=a, kv_heads=g, table=table, pos_offset=offset,
                                          position_ids=position_ids, grouped=True)
        assert grouped.shape == (b, s, g, r + 2, d)
        assert torch.equal(grouped[:, :, :, :r].reshape(b, s, a, d), q.transpose(1, 2))
        assert torch.equal(grouped[:, :, :, r], k.transpose(1, 2))
        assert torch.equal(grouped[:, :, :, r + 1], v.transpose(1, 2))


def _cfg(**over):
    c = LazyConfig.load("projects/ChatGLM/configs/chatglm_config.py")
    tiny = ["cfg.num_layers=2", "cfg.hidden_size=64", "cfg.ffn_hidden_size=96", "cfg.num_attention_heads=4",
            "cfg.kv_channels=16", "cfg.multi_query_group_num=2", "cfg.padded_vocab_size=128", "cfg.seq_length=48",
            "cfg.max_length=20", "cfg.pad_token_id=0"]
    c = LazyConfig.apply_overrides(c, tiny + [f"cfg.{k}={v}" for k, v in over.items()])
    c.model.cfg = c.cfg
    return c


def _model(seed=0, **over):
    torch.manual_seed(seed)
    return instantiate(_cfg(**over).model)


def _old_attention_forward(self, hidden, inputs, kv_cache=None):
    """The attention block before the packing kernel: PyTorch rotary, the prefix concatenated, K/V repeated."""
    b, s, _ = hidden.shape
    a, g, d = self.heads, self.groups, self.d
    rope = inputs.table[inputs.position_ids[0]] if inputs.position_ids is not None else \
        inputs.table[inputs.pos_offset : inputs.pos_offset + s]
    q, k, v = _old_qkv(self.query_key_value(hidden), a, g, rope)
    if kv_cache is not None:
        k = torch.cat((kv_cache[0].type_as(k), k), dim=2)
        v = torch.cat((kv_cache[1].type_as(v), v), dim=2)
    k, v = k.repeat_interleave(a // g, dim=1), v.repeat_interleave(a // g, dim=1)
    ctx = OF.attention(q, k, v, causal=inputs.mask is None and q.shape[2] == k.shape[2], scale=1.0 / math.sqrt(d),
                       mask=inputs.mask)
    return self.dense(ctx.transpose(1, 2).reshape(b, s, a * d))


@pytest.mark.parametrize("prefix", [None, 3])
def test_attention_block_matches_old_composition(prefix, monkeypatch):
    from projects.ChatGLM.chatglm import SelfAttention

    over = {} if prefix is None else dict(pre_seq_len=prefix, prefix_projection=False)
    ids = torch.randint(1, 128, (2, 10))
    m = _model(**over).train()

    def loss_and_grads():
        m.zero_grad(set_to_none=True)
        torch.manual_seed(3)   # the same dropout mask on the P-tuning prefix
        loss = m(ids, labels=ids)["loss"]
        loss.backward()
        return loss, {n: p.grad for n, p in m.named_parameters() if p.grad is not None}

    new_loss, new_grads = loss_and_grads()
    monkeypatch.setattr(SelfAttention, "forward", _old_attention_forward)
    old_loss, old_grads = loss_and_grads()
    assert new_grads and new_grads.keys() == old_grads.keys()
    if prefix is not None:
        assert all(n.startswith("transformer.prefix_encoder") for n in new_grads)
    torch.testing.assert_close(new_loss, old_loss, rtol=1e-6, atol=1e-6)
    for n in new_grads:
        torch.testing.assert_close(new_grads[n], old_grads[n], rtol=1e-5, atol=1e-6, msg=n)


def _generate_both(m, ids, **kw):
    m.eval()
    cached = m.generate(ids, max_length=ids.shape[1] + 6, eos_token_id=None, use_cache=True, **kw)
    assert isinstance(m.kv_cache, StaticKVCache)
    uncached = m.generate(ids, max_length=ids.shape[1] + 6, eos_token_id=None, use_cache=False, **kw)
    return cached, uncached


@pytest.mark.parametrize("case", ["plain", "left_padded", "prefix", "beams", "lora"])
def test_cached_generation_equals_uncached(case):
    over = dict(pre_seq_len=4, prefix_projection=False) if case == "prefix" else \
        dict(lora_enable=True) if case == "lora" else {}
    m = _model(seed=1, **over)
    if case == "lora":   # nonzero adapters, so that the LoRA path changes the function
        with torch.no_grad():
            for n, p in m.named_parameters():
                if "lora_B" in n:
                    p.normal_(std=0.05)
    torch.manual_seed(2)
    ids = torch.randint(3, 128, (3, 8))
    kw = {}
    if case == "left_padded":
        am = torch.ones_like(ids)
        ids[1, :3], am[1, :3] = 0, 0
        ids[2, :1], am[2, :1] = 0, 0
        kw["attention_mask"] = am
    if case == "beams":
        kw["num_beams"] = 2
    cached, uncached = _generate_both(m, ids, **kw)
    assert cached.shape == (3, 14)
    assert torch.equal(cached, uncached)


def test_cache_holds_the_key_value_groups():
    m = _model(pre_seq_len=2, prefix_projection=False).eval()
    ids = torch.randint(3, 128, (2, 5))
    m.generate(ids, max_length=9, eos_token_id=None, use_cache=True)
    c = m.kv_cache
    assert c.heads == 2 and c.head_dim == 16 and c.k[0].shape[:2] == (2, 2)
    assert c.capacity >= 2 + 9   # the prefix rows and the longest sequence
