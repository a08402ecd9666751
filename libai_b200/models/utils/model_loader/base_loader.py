"""Pretrained-weight loaders: LiBai-format checkpoints and HuggingFace checkpoints → ``libai_b200`` models.

Spec: reference libai/models/utils/model_loader/base_loader.py — ``ModelLoader`` (:52-289: build the model from
``model(cfg)`` then fill it, reporting missing / unexpected / mismatched keys), ``ModelLoaderLiBai`` (:292-363),
``ModelLoaderHuggerFace`` (:366-641: read ``config.json`` → update the LiBai config, read ``pytorch_model.bin`` /
safetensors (+ sharded index), convert names, fuse q/k/v with the per-head ``[a, 3, d]`` row order
(``_fix_qkv_ordering`` :425-443), cast, load).

The reference broadcasts the rank-0 state dict and re-shards by SBP; here every rank reads the (mmap-able) files
itself and ``parallel.state.load_full_state_dict`` copies the rank's tensor-parallel slice of each logical tensor
into the parameters of the pipeline stage it owns.
"""
from __future__ import annotations

import collections
import copy
import json
import logging
import os
import re
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch

from libai_b200.config import LazyCall, instantiate, try_get_key
from libai_b200.parallel.state import load_full_state_dict
from libai_b200.utils import distributed as dutil

logger = logging.getLogger(__name__)

WEIGHTS_NAME_PT = "pytorch_model.bin"
WEIGHTS_NAME_SAFE = "model.safetensors"
CONFIG_NAME = "config.json"


class LoadPretrainedBase:
    """Shared machinery: model construction from a LiBai config and the final state-dict hand-over."""

    def __init__(self, model, libai_cfg, pretrained_model_path, **kwargs):
        self.model = model                      # class, LazyCall node or already-built nn.Module
        self.libai_cfg = libai_cfg              # the model's cfg node (updated in place from config.json / kwargs)
        self.pretrained_model_path = pretrained_model_path
        self.kwargs = kwargs
        self.output_loading_info = kwargs.pop("output_loading_info", False)
        self.base_model_prefix_1 = None         # prefix used by the checkpoint ("bert", "transformer", …)
        self.base_model_prefix_2 = None         # prefix used by the libai_b200 model ("bert", "GPT_model", …)

    # ------------------------------------------------------------------ helpers
    def _update_cfg(self, key, value):
        if isinstance(self.libai_cfg, dict) or hasattr(self.libai_cfg, "__setitem__"):
            self.libai_cfg[key] = value
        else:
            setattr(self.libai_cfg, key, value)

    def _apply_kwargs(self):
        for k, v in self.kwargs.items():
            self._update_cfg(k, v)

    def _build_model(self):
        if isinstance(self.model, torch.nn.Module):
            return self.model
        if isinstance(self.model, type):
            return self.model(self.libai_cfg)
        node = copy.copy(self.model)            # LazyCall node: {_target_: cls, cfg: …}
        if "cfg" in node:
            node["cfg"] = self.libai_cfg
        return instantiate(node)

    def _load(self, model, state_dict):
        state_dict = self._align_prefix(model, state_dict)
        missing, unexpected, mismatched = load_full_state_dict(model, state_dict, strict=False)
        if dutil.is_main_process():
            name = model.__class__.__name__
            if unexpected:
                logger.warning(f"Some weights of the checkpoint at {self.pretrained_model_path} were not used when "
                               f"initializing {name}:\n {unexpected}\n")
            if missing:
                logger.warning(f"Some weights of {name} were not initialized from the checkpoint at "
                               f"{self.pretrained_model_path}:\n {missing}\n")
            else:
                logger.info(f"All the weights of {name} were initialized from {self.pretrained_model_path}.")
        if mismatched:
            # on EVERY rank (the list is computed identically everywhere): raising on rank 0 only would leave the
            # others waiting in the next collective
            txt = "\n".join(f"- {k}: found shape {a} in the checkpoint and {b} in the model" for k, a, b in mismatched)
            raise RuntimeError(f"Error(s) in loading state_dict for {model.__class__.__name__}:\n{txt}")
        if self.output_loading_info:
            return model, {"missing_keys": missing, "unexpected_keys": unexpected, "mismatched_keys": mismatched}
        return model

    def _align_prefix(self, model, state_dict):
        """Backbone checkpoint ↔ task model (or the reverse): pick, among {as is, first segment stripped, task prefix
        added}, the key mapping that matches most of the model's own keys."""
        own = set(model.state_dict().keys())

        def score(mapping):
            return sum(1 for k in mapping if k in own)

        candidates = [collections.OrderedDict(state_dict)]
        firsts = {k.split(".", 1)[0] for k in state_dict if "." in k}
        for first in firsts:
            candidates.append(collections.OrderedDict(
                (k[len(first) + 1 :] if k.startswith(first + ".") else k, v) for k, v in state_dict.items()))
        prefixes = {k.split(".", 1)[0] for k in own if "." in k}
        if self.base_model_prefix_2:
            prefixes.add(self.base_model_prefix_2)
        for p2 in prefixes:
            candidates.append(collections.OrderedDict(
                ((p2 + "." + k) if (p2 + "." + k) in own else k, v) for k, v in state_dict.items()))
        return max(candidates, key=score)


# name used by the reference for the common base (libai/models/utils/model_loader/base_loader.py:69)
ModelLoader = LoadPretrainedBase


class ModelLoaderLiBai(LoadPretrainedBase):
    """Load a checkpoint written by ``libai_b200.utils.checkpoint.Checkpointer`` (directory with a ``model`` file,
    or the ``model_XXXXXXX`` directory itself, or a single ``torch.save`` file)."""

    def __init__(self, model, libai_cfg, pretrained_model_path, **kwargs):
        super().__init__(model, libai_cfg, pretrained_model_path, **kwargs)
        self.base_model_prefix_2 = None

    def _load_state_dict(self):
        path = self.pretrained_model_path
        if os.path.isdir(path):
            if os.path.isfile(os.path.join(path, "last_checkpoint")):
                with open(os.path.join(path, "last_checkpoint")) as f:
                    path = os.path.join(path, f.read().strip())
            if os.path.isfile(os.path.join(path, "model")):
                path = os.path.join(path, "model")
        obj = torch.load(path, map_location="cpu", weights_only=False)
        return obj["model"] if isinstance(obj, dict) and "model" in obj and isinstance(obj["model"], dict) else obj

    def load(self):
        self._apply_kwargs()
        model = self._build_model()
        return self._load(model, self._load_state_dict())


class ModelLoaderHuggerFace(LoadPretrainedBase):
    """Base of the HuggingFace converters (the class name keeps the reference's spelling)."""

    def __init__(self, model, libai_cfg, pretrained_model_path, **kwargs):
        super().__init__(model, libai_cfg, pretrained_model_path, **kwargs)
        self.base_model_prefix_2 = None

    # ------------------------------------------------------------------ file reading
    def _weight_files(self) -> List[str]:
        d = self.pretrained_model_path
        for index in (WEIGHTS_NAME_SAFE + ".index.json", WEIGHTS_NAME_PT + ".index.json"):
            fp = os.path.join(d, index)
            if os.path.isfile(fp):
                with open(fp) as f:
                    shards = sorted(set(json.load(f)["weight_map"].values()))
                return [os.path.join(d, s) for s in shards]
        for name in (WEIGHTS_NAME_SAFE, WEIGHTS_NAME_PT):
            if os.path.isfile(os.path.join(d, name)):
                return [os.path.join(d, name)]
        cands = sorted(f for f in os.listdir(d) if f.endswith((".safetensors", ".bin", ".pt", ".pth")))
        if not cands:
            raise EnvironmentError(f"no weight file ({WEIGHTS_NAME_SAFE} / {WEIGHTS_NAME_PT}) found in {d}")
        return [os.path.join(d, c) for c in cands]

    def _load_torch_state_dict(self) -> Dict[str, torch.Tensor]:
        sd: Dict[str, torch.Tensor] = collections.OrderedDict()
        for fp in self._weight_files():
            if fp.endswith(".safetensors"):
                from safetensors.torch import load_file

                sd.update(load_file(fp, device="cpu"))
            else:
                part = torch.load(fp, map_location="cpu", weights_only=True)
                sd.update(part.get("state_dict", part) if isinstance(part, dict) else part)
        return self._fix_key(sd)

    # ------------------------------------------------------------------ conversion helpers
    @staticmethod
    def _fix_key(state_dict):
        """TF-era names: ``gamma`` → ``weight``, ``beta`` → ``bias``."""
        for key in list(state_dict.keys()):
            new = key.replace("gamma", "weight") if "gamma" in key else key
            new = new.replace("beta", "bias") if "beta" in new else new
            if new != key:
                state_dict[new] = state_dict.pop(key)
        return state_dict

    @staticmethod
    def _fix_qkv_ordering(qkv, head_size, num_heads, hidden_size=None, checkpoint_version=0.0, num_kv_heads=None):
        """``[q; k; v]`` blocks (each ``[a·d, …]``) → per-head interleaved ``[a, (q|k|v), d, …]`` rows, the layout
        the fused ``query_key_value`` projection (and its tensor-parallel split over heads) expects.  With
        ``num_kv_heads`` = g < a (grouped-query attention: q ``[a·d, …]``, k and v ``[g·d, …]``) the rows are grouped
        ``[g, (q_0 .. q_{r-1}|k|v), d, …]``, ``r = a / g``."""
        if num_kv_heads is not None and num_kv_heads != num_heads:
            g, r = num_kv_heads, num_heads // num_kv_heads
            rest = tuple(qkv.shape[1:])
            q, k, v = qkv.split([num_heads * head_size, g * head_size, g * head_size])
            out = torch.cat([q.reshape(g, r, head_size, *rest), k.reshape(g, 1, head_size, *rest),
                             v.reshape(g, 1, head_size, *rest)], dim=1)
            return out.reshape(-1, *rest).contiguous()
        n = qkv.shape[0] // (head_size * num_heads)
        if qkv.dim() > 1:
            hidden_size = qkv.shape[1] if hidden_size is None else hidden_size
            return (qkv.reshape(n, num_heads, head_size, hidden_size).permute(1, 0, 2, 3).contiguous()
                    .reshape(n * num_heads * head_size, hidden_size))
        return qkv.reshape(n, num_heads, head_size).permute(1, 0, 2).contiguous().reshape(-1)

    @staticmethod
    def _convert_tensor(tensor):
        """Checkpoint tensors are kept in their stored dtype on CPU; the copy into the parameter casts."""
        return tensor.contiguous() if torch.is_tensor(tensor) else torch.as_tensor(tensor)

    def _fuse_qkv(self, sd, q, k, v, out, head_size, num_heads, transpose=False, num_kv_heads=None):
        """Pop q/k/v entries (weight + optional bias) and store the fused, re-ordered tensor under ``out``
        (``num_kv_heads``: see :meth:`_fix_qkv_ordering`)."""
        for suffix in ("weight", "bias"):
            keys = [f"{n}.{suffix}" for n in (q, k, v)]
            if not all(kk in sd for kk in keys):
                continue
            parts = [sd.pop(kk) for kk in keys]
            if transpose and suffix == "weight":
                parts = [p.t() for p in parts]
            sd[f"{out}.{suffix}"] = self._fix_qkv_ordering(torch.cat(parts, dim=0), head_size, num_heads,
                                                           num_kv_heads=num_kv_heads)

    @staticmethod
    def _rename(sd, rules: Sequence[Tuple[str, str]]):
        """Apply ``(regex, replacement)`` rules in order to every key."""
        out = collections.OrderedDict()
        for key, value in sd.items():
            new = key
            for pat, rep in rules:
                new = re.sub(pat, rep, new)
            out[new] = value
        return out

    def _convert_state_dict(self, torch_state_dict, cfg):
        raise NotImplementedError("_convert_state_dict not implemented")

    def _load_config_from_json(self, config_file):
        raise NotImplementedError("_load_config_from_json not implemented")

    def _read_config_json(self):
        fp = os.path.join(self.pretrained_model_path, CONFIG_NAME)
        if not os.path.isfile(fp):
            raise EnvironmentError(f"Can't find {CONFIG_NAME} in {self.pretrained_model_path}")
        with open(fp, encoding="utf-8") as f:
            return json.load(f)

    def _map_config(self, cfg_dict, mapping: Dict[str, str]):
        """``mapping``: HF key → LiBai key (only keys present in config.json are touched)."""
        for hf_key, libai_key in mapping.items():
            if hf_key in cfg_dict and cfg_dict[hf_key] is not None:
                self._update_cfg(libai_key, cfg_dict[hf_key])

    def load(self):
        if os.path.isdir(self.pretrained_model_path):
            self._load_config_from_json(os.path.join(self.pretrained_model_path, CONFIG_NAME))
        else:
            raise EnvironmentError(f"{self.pretrained_model_path} must be a directory")
        self._apply_kwargs()
        torch_sd = self._load_torch_state_dict()
        sd = self._convert_state_dict(torch_sd, self.libai_cfg)
        sd = collections.OrderedDict((k, self._convert_tensor(v)) for k, v in sd.items())
        model = self._build_model()
        return self._load(model, sd)
