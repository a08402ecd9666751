"""Llama loaders (reference projects/Llama/utils/llama_loader.py): HF ``q_proj/k_proj/v_proj`` → fused per-head
interleaved ``query_key_value`` (grouped per key/value head for grouped-query checkpoints); everything else keeps its
name."""
import collections

from .base_loader import ModelLoaderHuggerFace, ModelLoaderLiBai


class LlamaLoaderHuggerFace(ModelLoaderHuggerFace):
    def __init__(self, model, libai_cfg, pretrained_model_path, **kwargs):
        super().__init__(model, libai_cfg, pretrained_model_path, **kwargs)
        self.base_model_prefix_1 = "model"
        self.base_model_prefix_2 = "model"

    def _convert_state_dict(self, sd, cfg):
        sd = collections.OrderedDict(sd)
        heads, hidden, layers = cfg.get("num_attention_heads"), cfg.get("hidden_size"), cfg.get("hidden_layers")
        kv_heads = cfg.get("num_key_value_heads") or heads
        prefix = "model." if any(k.startswith("model.") for k in sd) else ""
        for i in range(layers):
            base = f"{prefix}layers.{i}.self_attn"
            self._fuse_qkv(sd, f"{base}.q_proj", f"{base}.k_proj", f"{base}.v_proj", f"{base}.query_key_value",
                           hidden // heads, heads, num_kv_heads=kv_heads)
        out = collections.OrderedDict()
        for k, v in sd.items():
            if k.endswith("rotary_emb.inv_freq"):
                continue
            out[k if (k.startswith("model.") or k.startswith("lm_head.")) else "model." + k] = v
        if "lm_head.weight" not in out and "model.embed_tokens.weight" in out:
            out["lm_head.weight"] = out["model.embed_tokens.weight"]  # tied checkpoints
        return out

    def _load_config_from_json(self, config_file):
        cfg = self._read_config_json()
        self._map_config(cfg, {
            "num_hidden_layers": "hidden_layers", "hidden_size": "hidden_size", "num_attention_heads": "num_attention_heads",
            "max_position_embeddings": "max_position_embeddings", "intermediate_size": "intermediate_size",
            "rms_norm_eps": "rms_norm_eps", "vocab_size": "vocab_size", "initializer_range": "initializer_range",
            "rope_theta": "rope_base", "bos_token_id": "bos_token_id", "eos_token_id": "eos_token_id",
            "pad_token_id": "pad_token_id", "num_key_value_heads": "num_key_value_heads",
        })


class LlamaLoaderLiBai(ModelLoaderLiBai):
    def __init__(self, model, libai_cfg, pretrained_model_path, **kwargs):
        super().__init__(model, libai_cfg, pretrained_model_path, **kwargs)
        self.base_model_prefix_2 = "model"
