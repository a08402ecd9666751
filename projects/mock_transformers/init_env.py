"""Tensor-parallel inference for stock HuggingFace ``transformers`` models.

Spec: reference projects/mock_transformers/init_env.py + dist_infer_*.py — the reference monkey-patches torch →
oneflow and swaps a HF model's Linear/Conv1D modules for LiBai's column/row-parallel layers so the unmodified HF
modelling code (and ``model.generate``) runs tensor-parallel.

Here the HF model already is a torch model, so nothing needs mocking.  What remains is the real feature: *rewrite a
loaded HF model in place into a tensor-parallel one*.  ``parallelize`` walks a plan of
``(module-name regex → "col" | "row")`` rules, replaces each matched ``nn.Linear``/``Conv1D`` by this framework's
:class:`Linear1D` (so the GEMM runs on the wgmma kernels, and — with ``fused_tp_comm`` — the all-gather /
reduce-scatter runs inside the GEMM), copies this rank's shard of the checkpoint weights into it, and divides the
per-module head counts by the TP size.  Fused QKV projections are sharded per section so every rank gets whole heads
of q, k and v.
"""
from __future__ import annotations

import re
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch
from torch import nn

from libai_b200.layers import Linear
from libai_b200.utils import distributed as dist


def _is_conv1d(m) -> bool:
    return m.__class__.__name__ == "Conv1D" and hasattr(m, "nf")


def _weight_out_in(m) -> torch.Tensor:
    """Weight as [out, in] regardless of the module flavour (HF ``Conv1D`` stores [in, out])."""
    return m.weight.data.t() if _is_conv1d(m) else m.weight.data


def _shard_rows(w: torch.Tensor, rank: int, world: int, sections: int, interleave: Optional[int]):
    """Rows (output features) of ``w`` owned by ``rank``.

    ``sections``: the output is a concatenation of that many equal blocks (q|k|v) and each is sharded separately.
    ``interleave``: the output is laid out [heads, interleave, head_dim] (BLOOM/NeoX fused qkv): shard over heads."""
    if interleave:
        assert w.shape[0] % world == 0
        return w.chunk(world, dim=0)[rank]          # heads are the outermost factor → a plain row split is per-head
    blocks = w.chunk(sections, dim=0)
    return torch.cat([b.chunk(world, dim=0)[rank] for b in blocks], dim=0)


def shard_linear(module, parallel: str, *, sections: int = 1, interleave: Optional[int] = None, layer_idx: int = 0,
                 dtype: Optional[torch.dtype] = None) -> Linear:
    """Build the tensor-parallel replacement of ``module`` holding this rank's shard of its weights."""
    assert parallel in ("col", "row", "data")
    topo = dist.get_dist_util()
    world, rank = topo.tensor_parallel_size, topo.tp_rank
    w = _weight_out_in(module)
    out_features, in_features = w.shape
    dtype = dtype or w.dtype
    new = Linear(in_features, out_features, bias=module.bias is not None, parallel=parallel, init_method=None,
                 dtype=dtype, layer_idx=layer_idx)
    with torch.no_grad():
        if parallel == "col":
            new.weight.copy_(_shard_rows(w, rank, world, sections, interleave).to(dtype))
            if module.bias is not None:
                new.bias.copy_(_shard_rows(module.bias.data[:, None], rank, world, sections, interleave)[:, 0].to(dtype))
        elif parallel == "row":
            new.weight.copy_(w.chunk(world, dim=1)[rank].to(dtype))
            if module.bias is not None:
                new.bias.copy_(module.bias.data.to(dtype))
        else:
            new.weight.copy_(w.to(dtype))
            if module.bias is not None:
                new.bias.copy_(module.bias.data.to(dtype))
    return new.to(w.device)


@dataclass
class Rule:
    pattern: str                       # regex on the qualified module name (``re.search``)
    parallel: str                      # "col" | "row"
    sections: int = 1
    interleave: Optional[int] = None


@dataclass
class Plan:
    rules: List[Rule]
    # (regex on module name, attribute names to divide by the TP size) — head counts / split sizes the HF
    # ``forward`` uses to reshape the now-narrower projections
    divide: List[Tuple[str, Sequence[str]]] = field(default_factory=list)
    # (regex, hook(module, tp_rank, tp_world)) for anything else (e.g. slicing BLOOM's alibi per rank)
    hooks: List[Tuple[str, Callable]] = field(default_factory=list)


def parallelize(model: nn.Module, plan: Plan, dtype: Optional[torch.dtype] = None) -> nn.Module:
    topo = dist.get_dist_util()
    world = topo.tensor_parallel_size
    replaced: Dict[str, str] = {}
    for name, module in list(model.named_modules()):
        if not (isinstance(module, nn.Linear) or _is_conv1d(module)):
            continue
        for rule in plan.rules:
            if re.search(rule.pattern, name):
                parent_name, _, child = name.rpartition(".")
                parent = model.get_submodule(parent_name) if parent_name else model
                setattr(parent, child, shard_linear(module, rule.parallel, sections=rule.sections,
                                                    interleave=rule.interleave, dtype=dtype))
                replaced[name] = rule.parallel
                break
    for name, module in model.named_modules():
        for pattern, attrs in plan.divide:
            if re.search(pattern, name):
                for a in attrs:
                    if hasattr(module, a):
                        v = getattr(module, a)
                        assert v % world == 0, f"{name}.{a}={v} is not divisible by tensor_parallel_size={world}"
                        setattr(module, a, v // world)
        for pattern, hook in plan.hooks:
            if re.search(pattern, name):
                hook(module, topo.tp_rank, world)
    model._tp_replaced = replaced
    return model


# ------------------------------------------------------------------------------------------------ model plans
GPT2_PLAN = Plan(
    rules=[Rule(r"attn\.c_attn$", "col", sections=3), Rule(r"attn\.q_attn$", "col"), Rule(r"attn\.c_proj$", "row"),
           Rule(r"mlp\.c_fc$", "col"), Rule(r"mlp\.c_proj$", "row")],
    divide=[(r"\.attn$", ("num_heads", "split_size", "embed_dim"))],
)

LLAMA_PLAN = Plan(      # also Qwen2 / Mistral / Aquila: same module names
    rules=[Rule(r"self_attn\.(q|k|v)_proj$", "col"), Rule(r"self_attn\.o_proj$", "row"),
           Rule(r"mlp\.(gate|up)_proj$", "col"), Rule(r"mlp\.down_proj$", "row")],
    divide=[(r"self_attn$", ("num_heads", "num_key_value_heads"))],
)

BAICHUAN_PLAN = Plan(   # fused W_pack = [q|k|v]
    rules=[Rule(r"self_attn\.W_pack$", "col", sections=3), Rule(r"self_attn\.o_proj$", "row"),
           Rule(r"mlp\.(gate|up)_proj$", "col"), Rule(r"mlp\.down_proj$", "row")],
    divide=[(r"self_attn$", ("num_heads", "hidden_size"))],
)

OPT_PLAN = Plan(
    rules=[Rule(r"self_attn\.(q|k|v)_proj$", "col"), Rule(r"self_attn\.out_proj$", "row"),
           Rule(r"layers\.\d+\.fc1$", "col"), Rule(r"layers\.\d+\.fc2$", "row")],
    divide=[(r"self_attn$", ("num_heads", "embed_dim"))],
)


def _bloom_alibi_hook(module, rank, world):
    """BLOOM builds alibi for all heads at the model level ([B*H, 1, kv]); each TP rank keeps its heads' slopes."""
    full_heads = module.num_heads * world     # runs after `divide`

    def pre(mod, args, kwargs):
        alibi = kwargs.get("alibi", None)
        if alibi is not None and world > 1:
            b = alibi.shape[0] // full_heads
            a = alibi.view(b, full_heads, *alibi.shape[1:])[:, rank * mod.num_heads:(rank + 1) * mod.num_heads]
            kwargs["alibi"] = a.reshape(b * mod.num_heads, *alibi.shape[1:])
        return args, kwargs

    module.register_forward_pre_hook(pre, with_kwargs=True)


BLOOM_PLAN = Plan(
    rules=[Rule(r"self_attention\.query_key_value$", "col", interleave=3), Rule(r"self_attention\.dense$", "row"),
           Rule(r"mlp\.dense_h_to_4h$", "col"), Rule(r"mlp\.dense_4h_to_h$", "row")],
    divide=[(r"self_attention$", ("num_heads", "hidden_size", "split_size"))],
    hooks=[(r"self_attention$", _bloom_alibi_hook)],
)

PLANS = {"gpt2": GPT2_PLAN, "llama": LLAMA_PLAN, "qwen2": LLAMA_PLAN, "mistral": LLAMA_PLAN, "aquila": LLAMA_PLAN,
         "baichuan": BAICHUAN_PLAN, "opt": OPT_PLAN, "bloom": BLOOM_PLAN}


def setup(tensor_parallel_size: Optional[int] = None, device_type: Optional[str] = None):
    """Initialise the topology for pure tensor-parallel inference over every launched process."""
    from libai_b200.config import DictConfig

    world = dist.get_world_size() if torch.distributed.is_initialized() else int(__import__("os").environ.get("WORLD_SIZE", 1))
    tp = tensor_parallel_size or world
    device_type = device_type or ("cuda" if torch.cuda.is_available() else "cpu")
    dist.setup_dist_util(DictConfig(dict(data_parallel_size=world // tp, tensor_parallel_size=tp,
                                         pipeline_parallel_size=1, pipeline_num_layers=None,
                                         device_type=device_type)))
    return dist.get_dist_util()


def load_parallel(model_or_path, model_type: Optional[str] = None, dtype: Optional[torch.dtype] = None,
                  device: Optional[str] = None, **from_pretrained_kwargs) -> nn.Module:
    """``AutoModelForCausalLM.from_pretrained`` (or an already built HF model) → tensor-parallel model on
    ``device``.  The full weights are materialised on the host, each rank keeps its shard."""
    if isinstance(model_or_path, nn.Module):
        model = model_or_path
    else:
        from transformers import AutoModelForCausalLM

        model = AutoModelForCausalLM.from_pretrained(model_or_path, **from_pretrained_kwargs)
    model_type = model_type or getattr(model.config, "model_type", None)
    assert model_type in PLANS, f"no tensor-parallel plan for model_type={model_type!r}; known: {sorted(PLANS)}"
    if dtype is None:
        dtype = torch.bfloat16 if (device or "").startswith("cuda") or torch.cuda.is_available() else torch.float32
    model = model.to(dtype)
    model = parallelize(model.eval(), PLANS[model_type], dtype=dtype)
    if device is None:
        device = f"cuda:{torch.cuda.current_device()}" if torch.cuda.is_available() else "cpu"
    return model.to(device)
