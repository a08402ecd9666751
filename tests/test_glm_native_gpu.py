"""GLM on the H100: bf16 models at head dim 64 whose prefill runs the prefix-LM flash instance in every layer and whose
decode steps run kv_append + decode_attn with no reference-math call, against the fp32 uncached model; one GLMLoss
training step through the prefix forward and backward kernels; and the FP8 cache and FP8 weights."""
import copy

import pytest
import torch

from libai_b200.config import DictConfig
from libai_b200.layers._param import param_defaults
from libai_b200.ops import functional as OF
from libai_b200.utils import distributed as dist
from projects.GLM.modeling_glm import GLMForConditionalGeneration
from tests.test_glm_native_cpu import Tok, tiny_cfg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LAYERS = 2


@pytest.fixture(autouse=True)
def _topo():
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=1, tensor_parallel_size=1, pipeline_parallel_size=1,
                                         device_type="cuda")))
    with torch.random.fork_rng(devices=[0]):
        yield


@pytest.fixture(scope="module")
def ext():
    from libai_b200 import ops

    return ops.load_ext(required=True)


def _glm():
    cfg = tiny_cfg()
    cfg.update(dict(vocab_size=256, hidden_size=256, num_attention_heads=4, num_layers=LAYERS, max_sequence_length=128))
    with param_defaults(dtype=torch.float32, device=DEV, seed=5):
        fp32 = GLMForConditionalGeneration(cfg).eval()
    return fp32, copy.deepcopy(fp32).to(torch.bfloat16)


class _Recorder:
    def __init__(self, ext):
        self.ext, self.calls = ext, []

    def __getattr__(self, name):
        fn = getattr(self.ext, name)
        if name in ("attn_fwd", "attn_bwd", "kv_append", "kv_append_fp8", "decode_attn", "linear_fp8w"):
            def wrapped(*a, **k):
                self.calls.append((name, k.get("prefix_lens") is not None))
                if name == "decode_attn":
                    self.kv_start = a[4].tolist()   # (the generator empties the cache when it ends)
                return fn(*a, **k)
            return wrapped
        return fn


def _refuse(*a, **k):
    raise AssertionError("the reference attention ran")


@pytest.fixture
def recorder(ext, monkeypatch):
    rec = _Recorder(ext)
    monkeypatch.setattr(OF, "load_ext", lambda *a, **k: rec)
    return rec


def _inputs(gen=12):
    """Three contexts of different lengths, right-padded by the tokenizer's own layout, on the GPU."""
    ids = torch.tensor([[11, 12, 13, 7, 14, 15, 16, 17, 18, 19], [31, 7, 33, 0, 0, 0, 0, 0, 0, 0],
                        [41, 42, 7, 43, 44, 45, 0, 0, 0, 0]])
    inp = Tok().build_inputs_for_generation({"input_ids": ids, "attention_mask": (ids != 0).long()}, max_gen_length=gen)
    return {k: v.to(DEV) for k, v in inp.items()}, (ids != 0).to(DEV)


def test_generate_runs_prefix_prefill_and_native_steps(recorder, monkeypatch):
    _, m = _glm()
    inp, _ = _inputs()
    monkeypatch.setattr(OF, "attention_ref", _refuse)
    monkeypatch.setattr(OF, "decode_attention_ref", _refuse)
    monkeypatch.setattr(OF, "kv_cache_append_ref", _refuse)
    S, new = inp["input_ids"].shape[1], 8
    with torch.no_grad():
        out = m.generate(inp["input_ids"], position_ids=inp["position_ids"],
                         generation_attention_mask=inp["generation_attention_mask"], max_length=S + new,
                         eos_token_id=None, use_cache=True)
    assert out.shape == (3, S + new)
    assert recorder.kv_start == [0, 7, 4]   # the right padding moved in front of each context
    assert recorder.calls.count(("attn_fwd", True)) == LAYERS and ("attn_fwd", False) not in recorder.calls
    assert recorder.calls.count(("kv_append", False)) == LAYERS * new
    assert recorder.calls.count(("decode_attn", False)) == LAYERS * (new - 1)


def _sequence(fp32, inp, steps):
    """The fp32 model's greedy continuation (uncached, recomputed each step) and its full-sequence inputs."""
    ids, pos, mask = inp["input_ids"], inp["position_ids"], inp["generation_attention_mask"]
    with torch.no_grad():
        for _ in range(steps):
            L = ids.shape[1]
            logits = fp32(ids, pos[:, :, :L], mask[:, :, :L, :L])["logits"]
            ids = torch.cat([ids, logits[:, -1].argmax(-1, keepdim=True)], 1)
    L = ids.shape[1]
    return ids, pos[:, :, :L], mask[:, :, :L, :L]


def _cached_logits(m, ids, pos, mask, s, kv_cache_dtype=None):
    m.kv_cache_dtype = kv_cache_dtype
    m.allocate_kv_cache(ids.shape[0], ids.shape[1])
    with torch.no_grad():
        out = [m(ids[:, :s], pos[:, :, :s], mask[:, :, :s, :s], use_cache=True)["logits"]]
        for L in range(s + 1, ids.shape[1] + 1):
            out.append(m(ids[:, L - 1 : L], pos[:, :, L - 1 : L], mask[:, :, L - 1 : L, :L], use_cache=True)["logits"])
    m.kv_cache_dtype = None
    m.set_cache(None)
    return torch.cat(out, 1).double()


def test_teacher_forced_cached_logits_match_fp32_uncached(recorder):
    """Tolerance as in the BLOOM test: the cached bf16 logits may differ from the fp32 ones by at most twice what the
    uncached bf16 forward does, or 2^-6 of the largest logit, whichever is larger (rows that are not padding)."""
    fp32, bf16 = _glm()
    inp, ctx = _inputs()
    s = inp["input_ids"].shape[1]
    ids, pos, mask = _sequence(fp32, inp, 8)
    with torch.no_grad():
        want = fp32(ids, pos, mask)["logits"].double()
        uncached = bf16(ids, pos, mask)["logits"].double()
    got = _cached_logits(bf16, ids, pos, mask, s)
    keep = torch.cat([ctx, torch.ones(3, ids.shape[1] - ctx.shape[1], dtype=torch.bool, device=DEV)], 1)
    err_uncached = (uncached - want)[keep].abs().max().item()
    err = (got - want)[keep].abs().max().item()
    tol = max(2 * err_uncached, 2.0 ** -6 * want[keep].abs().max().item())
    assert err <= tol, (err, err_uncached, tol)
    # greedy: the cached model's tokens are the fp32 model's wherever the fp32 choice is not a tie within tol
    with torch.no_grad():
        out = bf16.generate(inp["input_ids"], position_ids=inp["position_ids"],
                            generation_attention_mask=inp["generation_attention_mask"], max_length=s + 8,
                            eos_token_id=None, use_cache=True)
        ref = fp32(out, pos, mask)["logits"].double()
    chosen = ref[:, s - 1 : -1].gather(-1, out[:, s:, None])[..., 0]
    best = ref[:, s - 1 : -1].amax(-1)
    assert bool((chosen >= best - tol).all()), (out[:, s:], ids[:, s:])
    assert ("attn_fwd", True) in recorder.calls


def test_glm_loss_step_matches_reference_gradients(recorder, monkeypatch):
    """One GLMLoss step on the tokenizer's right-padded training layout: the prefix forward and backward kernels
    against the same bf16 model on the dense mask and the reference math."""
    _, m = _glm()
    m.train()
    ids = torch.tensor([[11, 12, 13, 7, 14, 15, 16], [31, 7, 33, 0, 0, 0, 0]])
    tr = Tok().build_inputs_for_generation({"input_ids": ids, "attention_mask": (ids != 0).long()},
                                           targets=["x", "y"], max_gen_length=6)
    tr = {k: v.to(DEV) for k, v in tr.items()}

    def step():
        m.zero_grad()
        loss = m(**tr)["lm_loss"]
        loss.backward()
        return loss.detach(), {n: p.grad.float().clone() for n, p in m.named_parameters()}

    loss, grads = step()
    assert ("attn_fwd", True) in recorder.calls and ("attn_bwd", True) in recorder.calls
    from projects.GLM import modeling_glm
    monkeypatch.setattr(modeling_glm, "_native_attention", lambda x, d: False)
    ref_loss, ref_grads = step()
    assert abs(float(loss) - float(ref_loss)) <= 2e-2 * abs(float(ref_loss))
    for n, g in ref_grads.items():
        rel = float((grads[n] - g).norm() / (g.norm() + 1e-12))
        assert rel < 3e-2, (n, rel)


def rel_err(a, b):
    return float((a - b).abs().max() / (b.abs().max() + 1e-6))


def test_fp8_cache_matches_dequantized_reference(recorder, monkeypatch):
    """The native kernels on an FP8 cache against the reference attention over the same format (FP8 tests' bound)."""
    _, m = _glm()
    inp, _ = _inputs()
    s = inp["input_ids"].shape[1]
    ids = torch.cat([inp["input_ids"], torch.randint(20, 200, (3, 6), device=DEV)], 1)
    pos, mask = inp["position_ids"][:, :, : s + 6], inp["generation_attention_mask"][:, :, : s + 6, : s + 6]
    got = _cached_logits(m, ids, pos, mask, s, kv_cache_dtype=torch.float8_e4m3fn)
    assert ("kv_append_fp8", False) in recorder.calls and ("decode_attn", False) in recorder.calls
    monkeypatch.setattr(OF, "_decode_native", lambda *a: False)
    want = _cached_logits(m, ids, pos, mask, s, kv_cache_dtype=torch.float8_e4m3fn)
    assert rel_err(got, want) < 3e-2, rel_err(got, want)


def test_fp8_weights_match_dequantized_bf16_model(recorder):
    """Generation with FP8 weights runs the weight-streaming kernel; its cached logits match the bf16 model holding the
    dequantized weights (FP8 tests' bound)."""
    from libai_b200.inference import quantize_weights_fp8_

    _, m = _glm()
    deq = copy.deepcopy(m)
    quantize_weights_fp8_(m)
    with torch.no_grad():
        mods = dict(m.named_modules())
        for name, mod in deq.named_modules():
            q = mods.get(name)
            if q is not None and getattr(q, "weight_scale", None) is not None:
                mod.weight.copy_((q.weight.float() * q.weight_scale[:, None]).to(torch.bfloat16))
    inp, _ = _inputs()
    s = inp["input_ids"].shape[1]
    ids = torch.cat([inp["input_ids"], torch.randint(20, 200, (3, 6), device=DEV)], 1)
    pos, mask = inp["position_ids"][:, :, : s + 6], inp["generation_attention_mask"][:, :, : s + 6, : s + 6]
    got = _cached_logits(m, ids, pos, mask, s)
    assert any(c[0] == "linear_fp8w" for c in recorder.calls)
    want = _cached_logits(deq, ids, pos, mask, s)
    assert rel_err(got, want) < 3e-2, rel_err(got, want)
    with torch.no_grad():
        out = m.generate(inp["input_ids"], position_ids=inp["position_ids"],
                         generation_attention_mask=inp["generation_attention_mask"], max_length=s + 4,
                         eos_token_id=None, use_cache=True, kv_cache_dtype="fp8")
    assert out.shape == (3, s + 4)
