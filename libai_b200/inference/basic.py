"""Task pipeline base class.

Spec: reference libai/inference/basic.py:32-208 — load a LazyConfig, override the parallel layout, set up the
distributed topology, build + load the model (``mode``: ``"libai"`` checkpoint, ``"huggingface"`` where the
subclass supports it, ``"random"``), build the tokenizer, then ``__call__ = preprocess → forward → postprocess``
with per-call parameter routing (``_parse_parameters``).  Results are produced on the main process (other ranks
return ``{}``), like the reference.
"""
from __future__ import annotations

import logging
from abc import ABCMeta, abstractmethod
from pathlib import Path
from typing import Any, Dict

import torch

from libai_b200.config import LazyConfig, try_get_key
from libai_b200.utils import distributed as dist

logger = logging.getLogger(__name__)


class BasePipeline(metaclass=ABCMeta):
    def __init__(self, config_file, data_parallel=None, tensor_parallel=None, pipeline_parallel=None,
                 pipeline_stage_id=None, pipeline_num_layers=None, model_path=None, mode="libai", device=None,
                 weight_dtype=None, **kwargs):
        """``weight_dtype``: None keeps the weights as placed; ``"fp8"`` converts the model's linear layers to FP8
        (E4M3) weights with per-channel scales after placing it (:func:`libai_b200.inference.quantize_weights_fp8_`),
        ``"int4"`` to INT4 weights with a scale and zero point per group of 128 input columns
        (:func:`libai_b200.inference.quantize_weights_int4_`)."""
        if weight_dtype not in (None, "fp8", "int4"):
            raise ValueError(f"weight_dtype={weight_dtype!r}: None, 'fp8' or 'int4'")
        self.cfg = LazyConfig.load(config_file) if isinstance(config_file, (str, Path)) else config_file
        self.update_cfg(data_parallel, tensor_parallel, pipeline_parallel, pipeline_stage_id, pipeline_num_layers)
        self.device = device or ("cuda" if torch.cuda.is_available() else "cpu")
        self.cfg.train.dist.device_type = self.device
        dist.setup_dist_util(self.cfg.train.dist)
        logger.info(self.cfg.train.dist)

        self.model_path = model_path
        model_cfg = try_get_key(self.cfg, "model.cfg")
        if self.model_path is not None and model_cfg is not None:
            model_cfg.pretrained_model_path = self.model_path
        elif model_cfg is not None and "pretrained_model_path" in model_cfg:
            self.model_path = model_cfg.pretrained_model_path
        else:
            assert mode == "random", "a `model_path` (or cfg.model.cfg.pretrained_model_path) is required"

        self.model = self.load_pretrain_weight(self.cfg.model, self.model_path, mode=mode)
        self.model = self._place(self.model).eval()
        if weight_dtype == "fp8":
            from libai_b200.inference import quantize_weights_fp8_

            quantize_weights_fp8_(self.model)
        elif weight_dtype == "int4":
            from libai_b200.inference import quantize_weights_int4_

            quantize_weights_int4_(self.model)
        self.tokenizer = self.build_tokenizer(self.cfg)
        self._preprocess_params, self._forward_params, self._postprocess_params = self._parse_parameters(**kwargs)

    # ------------------------------------------------------------------ setup
    def update_cfg(self, data_parallel=1, tensor_parallel=1, pipeline_parallel=1, pipeline_stage_id=None,
                   pipeline_num_layers=None):
        d = self.cfg.train.dist
        d.data_parallel_size = data_parallel or 1
        d.tensor_parallel_size = tensor_parallel or 1
        d.pipeline_parallel_size = pipeline_parallel or 1
        d.custom_pipeline_stage_id = pipeline_stage_id
        if pipeline_num_layers is not None:
            d.pipeline_num_layers = pipeline_num_layers
        if d.pipeline_parallel_size > 1:
            assert try_get_key(d, "pipeline_num_layers") is not None, (
                "cfg.train.dist.pipeline_num_layers must be set when run pipeline parallel"
            )

    def _place(self, model):
        """Parameters were created on the stage/TP layout by the layer constructors; move them to the device and
        to bf16 for inference on GPU (fp32 on CPU)."""
        if self.device.startswith("cuda"):
            return model.to(device=torch.device("cuda", torch.cuda.current_device()), dtype=torch.bfloat16)
        return model

    def load_pretrain_weight(self, libai_cfg_model, model_path, mode="libai"):
        """``mode="libai"``: checkpoint written by this framework; ``"random"``: freshly initialised weights
        (debugging); subclasses add ``"huggingface"``."""
        if mode == "libai":
            from libai_b200.models.utils.model_loader.base_loader import ModelLoaderLiBai

            loader = ModelLoaderLiBai(libai_cfg_model, libai_cfg_model.cfg, model_path)
            loader.base_model_prefix_1 = None
            loader.base_model_prefix_2 = ""
            return loader.load()
        if mode == "random":
            from libai_b200.engine import DefaultTrainer

            return DefaultTrainer.build_model(self.cfg)
        raise NotImplementedError(f"mode={mode!r}")

    def build_tokenizer(self, cfg):
        if try_get_key(cfg, "tokenization") is None:
            return None
        from libai_b200.engine import DefaultTrainer

        tokenizer_cfg = cfg.tokenization.tokenizer
        if "pretrained_model_path" not in tokenizer_cfg and self.model_path is not None:
            candidate = Path(self.model_path).joinpath("tokenizer.model")
            if candidate.exists():
                tokenizer_cfg.pretrained_model_path = str(candidate)
        return DefaultTrainer.build_tokenizer(cfg)

    # ------------------------------------------------------------------ call protocol
    @abstractmethod
    def _parse_parameters(self, **pipeline_parameters):
        raise NotImplementedError("_parse_parameters not implemented")

    def __call__(self, inputs, *args, batch_size=None, **kwargs) -> dict:
        pre, fwd, post = self._parse_parameters(**kwargs)
        pre = {**self._preprocess_params, **pre}
        fwd = {**self._forward_params, **fwd}
        post = {**self._postprocess_params, **post}
        with torch.no_grad():
            model_inputs = self.preprocess(inputs, **pre)
            model_outputs = self.to_local(self.forward(model_inputs, **fwd))
            outputs = self.postprocess(model_outputs, **post) if dist.is_main_process() else {}
            dist.synchronize()
        return outputs

    def to_device(self, tensor):
        # (parameters of other pipeline stages are `meta` placeholders: take the first materialised one)
        dev = next((p.device for p in self.model.parameters() if p.device.type != "meta"), None)
        return tensor.to(dev if dev is not None else dist.get_dist_util().device)

    def to_local(self, model_outputs_dict):
        """Outputs are replicated across the model-parallel group already; bring them to host memory."""
        out = {}
        for key, value in model_outputs_dict.items():
            out[key] = value.detach().float().cpu() if torch.is_tensor(value) and value.is_floating_point() else (
                value.detach().cpu() if torch.is_tensor(value) else value)
        return out

    @abstractmethod
    def preprocess(self, input_: Any, **preprocess_parameters: Dict) -> dict:
        raise NotImplementedError("preprocess not implemented")

    @abstractmethod
    def forward(self, **kwargs: Dict) -> dict:
        raise NotImplementedError("forward not implemented")

    @abstractmethod
    def postprocess(self, **kwargs: Dict) -> dict:
        raise NotImplementedError("postprocess not implemented")
