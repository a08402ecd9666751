"""GPT-2 with a KV cache and ``generate`` (reference projects/MagicPrompt/gpt2.py: the library GPT-2 extended with
``past_key_values`` / ``use_cache`` and the ``Generator`` mixin for prompt completion)."""
from torch import nn

from libai_b200.config import configurable
from libai_b200.inference.generator.generation_utils import Generator
from libai_b200.inference.kv_cache import KVCacheOwner
from libai_b200.models import gpt_model as core
from libai_b200.models.gpt_model import GPTEmbedding, Transformer  # noqa: F401  (building blocks, same names as the reference module)
from libai_b200.parallel import mappings
from libai_b200.utils import distributed as dutil


class GPTModel(core.GPTModel, Generator, KVCacheOwner):
    @configurable
    def __init__(self, *args, cfg=None, **kwargs):
        super().__init__(*args, **kwargs)
        self.cfg = cfg
        self.kv_cache = None
        self.past_length = 0

    @classmethod
    def from_config(cls, cfg):
        out = core.GPTModel.from_config.__func__(cls, cfg)
        out["cfg"] = cfg
        return out

    def forward(self, input_ids, use_cache=False):
        if not use_cache and self.training:
            return {"logits": super().forward(input_ids)}
        cache = self._prepare_cache(input_ids) if use_cache else None
        past_len = cache.length if use_cache else 0
        hidden = self.embeddings(input_ids, past_len)
        for i, layer in enumerate(self.transformer.layers):
            # causal prefill, then decoding steps over the cache (every cached token is visible)
            hidden = layer(hidden, None, past_key_value=cache.layer(i) if use_cache else None)
        if use_cache:
            cache.advance(input_ids.shape[1])
            self.past_length = cache.length
        logits = self.lm_head(self.transformer.layernorm_f(hidden), self.word_embeddings_weight())
        if dutil.get_dist_util().tensor_parallel_size > 1:
            logits = mappings.gather_from_tp(logits)
        return {"logits": logits}

    # ---- KV cache (KVCacheOwner) ----------------------------------------------------------------
    def _cache_attention_modules(self):
        return [layer.self_attention for layer in self.transformer.layers]

    def prepare_inputs_for_generation(self, input_ids, past=None, use_cache=None, **kwargs):
        if past is not None and use_cache:
            input_ids = input_ids[:, -1:]
        return {"input_ids": input_ids, "use_cache": bool(use_cache)}


class GPTForPreTraining(core.GPTForPreTraining):
    def __init__(self, cfg) -> None:
        nn.Module.__init__(self)
        self.GPT_model = GPTModel(cfg)
        self.loss_func = core.GPTLoss()

    def forward(self, input_ids, labels=None):
        logits = core.GPTModel.forward(self.GPT_model, input_ids)
        if labels is not None:
            return self.loss_func(logits, labels)
        return {"prediction_scores": logits}
