"""``default_setup`` and ``DefaultTrainer``.

Spec: reference libai/engine/default.py — batch-size algebra ``global = micro × acc × D``
(:62-119), ``default_setup`` (:147-201: logger, dist topology, batch check, config dump, native
helper build), ``DefaultTrainer`` (:204-848: tokenizer + padded vocab :523-544, resume :264-283 /
:377-405, loaders, ``auto_scale_hyperparams`` :695-774, model/optimizer/scheduler builders, hooks
:407-449, writers :451-478, ``get_batch`` :493-521, ``test`` :781-848).

Differences by design: there is one execution mode (an iteration is one optimizer step over
``num_accumulation_steps`` micro-batches — the reference's graph-mode accounting); the features the
reference could only enable under ``nn.Graph`` (mixed precision, ZeRO, activation checkpointing,
1F1B pipelining) are always available and configured from the same ``cfg.train`` keys.
"""
from __future__ import annotations

import logging
import math
import os
import time
from collections import OrderedDict
from typing import Callable, Optional

import torch

from libai_b200.config import LazyConfig, instantiate, try_get_key
from libai_b200.data import Instance
from libai_b200.engine import hooks
from libai_b200.engine.trainer import StepTrainer, TrainerBase
from libai_b200.evaluation import inference_on_dataset, print_csv_format
from libai_b200.layers._param import param_defaults
from libai_b200.models import build_model as _build_model
from libai_b200.optim import DynamicLossScaler, build_optimizer
from libai_b200.scheduler import build_lr_scheduler
from libai_b200.utils import distributed as dutil
from libai_b200.utils.checkpoint import Checkpointer
from libai_b200.utils.events import CommonMetricPrinter, JSONWriter, TensorboardXWriter
from libai_b200.utils.logger import colored, setup_logger

__all__ = ["default_setup", "DefaultTrainer"]


def _highlight(code, filename):
    try:
        import pygments
        from pygments.formatters import Terminal256Formatter
        from pygments.lexers import Python3Lexer, YamlLexer
    except ImportError:
        return code
    lexer = Python3Lexer() if filename.endswith(".py") else YamlLexer()
    return pygments.highlight(code, lexer, Terminal256Formatter(style="monokai"))


def _check_batch_size(cfg):
    """Derive the missing one of (micro batch, global batch, accumulation steps)."""
    D = dutil.get_data_parallel_size()
    micro = try_get_key(cfg, "train.train_micro_batch_size", default=None)
    glob = try_get_key(cfg, "train.global_batch_size", default=None)
    acc = try_get_key(cfg, "train.num_accumulation_steps", default=None)
    if micro is not None and glob is not None:
        if acc is None:
            if glob % (micro * D) != 0:
                raise ValueError(
                    f"global_batch_size {glob} must be divisible by "
                    f"train_micro_batch_size * data_parallel_size ({micro} * {D})"
                )
            cfg.train.num_accumulation_steps = glob // (micro * D)
        elif glob != micro * D * acc:
            raise ValueError(
                f"global_batch_size {glob} must equal to train_micro_batch_size * data_parallel_size * "
                f"num_accumulation_steps ({micro} * {D} * {acc})"
            )
    elif micro is not None:
        if acc is None:
            cfg.train.num_accumulation_steps = 1
        cfg.train.global_batch_size = micro * D * cfg.train.num_accumulation_steps
    elif glob is not None:
        if acc is None:
            cfg.train.num_accumulation_steps = 1
        denom = D * cfg.train.num_accumulation_steps
        if glob % denom != 0:
            raise ValueError(
                f"global_batch_size {glob} must be divisible by data_parallel_size * "
                f"num_accumulation_steps ({D} * {cfg.train.num_accumulation_steps})"
            )
        cfg.train.train_micro_batch_size = glob // denom
    else:
        raise ValueError("train_micro_batch_size and global_batch_size must be set either")
    cfg.train.samples = cfg.train.train_iter * cfg.train.global_batch_size


def _compile_dependencies():
    """Build the native pieces once per node (local rank 0), everyone else waits.

    Reference: engine/default.py:122-144 runs ``make`` for the C++ dataset helpers.  Here both the
    C++ helpers and the CUDA extension are built in-tree ahead of time (``__graft_entry__.build``);
    this only builds what is missing."""
    logger = logging.getLogger(__name__)
    if dutil.get_local_rank() == 0:
        t0 = time.time()
        try:
            from libai_b200.data.data_utils import helpers_build

            helpers_build.ensure_built()
        except Exception as e:  # the pure-python fallback remains usable
            logger.warning(f"could not build the C++ dataset helpers: {e}")
        logger.info(">>> done with dataset index builder. Compilation time: {:.3f} seconds".format(time.time() - t0))
    dutil.synchronize()


def _resolve_auto_tensor_parallel_mode(cfg):
    """``train.dist.sequence_parallel / fused_tp_comm = "auto"``: on for models that declare
    ``supports_sequence_parallel`` (GPT-2, BERT, Llama family) — their tensor-parallel blocks then run on token shards
    with the collectives inside the GEMM kernels (the H100 product path) — off for the others, which keep the
    reference's replicated-activation form (libai/layers/linear.py:123-149)."""
    d = try_get_key(cfg, "train.dist")
    if d is None:
        return
    sp, fused = try_get_key(d, "sequence_parallel", default=False), try_get_key(d, "fused_tp_comm", default=False)
    if not (isinstance(sp, str) or isinstance(fused, str)):
        return
    supported = False
    target = try_get_key(cfg, "model._target_")
    if target is not None:
        try:
            from libai_b200.config.instantiate import _resolve_callable

            cls = _resolve_callable(target) if isinstance(target, str) else target
            supported = bool(getattr(cls, "supports_sequence_parallel", False))
        except Exception:   # unknown target: stay with the conservative form
            supported = False
    if isinstance(sp, str):
        d.sequence_parallel = supported
    if isinstance(fused, str):
        d.fused_tp_comm = bool(d.sequence_parallel) and supported


def default_setup(cfg, args):
    """Common start-up: output dir + logger, distributed topology, batch sizes, config dump."""
    output_dir = try_get_key(cfg, "train.output_dir")
    if dutil.get_rank() == 0 and output_dir:
        os.makedirs(output_dir, exist_ok=True)
    cfg.train.resume = bool(getattr(args, "resume", False))
    _resolve_auto_tensor_parallel_mode(cfg)
    dutil.setup_dist_util(cfg.train.dist)
    # device RNG (dropout masks): one stream per model replica / pipeline stage, shared by its tensor-parallel ranks
    torch.manual_seed(dutil.model_parallel_seed(try_get_key(cfg, "train.seed", default=1234)))
    rank = dutil.get_rank()
    logger = setup_logger(output_dir, distributed_rank=rank)
    logger.info("Rank of current process: {}. World size: {}".format(rank, dutil.get_world_size()))
    logger.info("Command line arguments: " + str(args))
    cfg_file = getattr(args, "config_file", "")
    if cfg_file:
        try:
            with open(cfg_file, "r") as f:
                logger.info("Contents of args.config_file={}:\n{}".format(cfg_file, _highlight(f.read(), cfg_file)))
        except OSError:
            pass
    logger.info(str(dutil.get_dist_util()))
    _check_batch_size(cfg)
    if dutil.is_main_process() and output_dir:
        path = os.path.join(output_dir, "config.yaml")
        LazyConfig.save(cfg, path)
        logger.info("Full config saved to {}".format(path))
    # NCCL bucket knobs of the reference (train.nccl_fusion_threshold_mb / nccl_fusion_max_ops)
    # map to the gradient-bucket size of the flat-buffer optimizer.
    os.environ.setdefault("LIBAI_B200_BUCKET_MB", str(try_get_key(cfg, "train.nccl_fusion_threshold_mb", default=16)))
    _compile_dependencies()


class DefaultTrainer(TrainerBase):
    """Trainer with the default logic: build everything from ``cfg`` then ``train()``.

    Override points (classmethods): ``build_model, build_optimizer, build_lr_scheduler,
    build_train_loader, build_test_loader, build_tokenizer, build_evaluator, get_batch, test,
    auto_scale_hyperparams``; instance methods ``build_hooks, build_writers, run_step``."""

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        logger = logging.getLogger("libai_b200")
        if not logger.isEnabledFor(logging.INFO):
            setup_logger()
        self.tokenizer = self.build_tokenizer(cfg)

        # ---- resume bookkeeping --------------------------------------------------------------
        self.start_iter = 0
        if try_get_key(cfg, "train.resume", default=False):
            marker = os.path.join(cfg.train.output_dir, "last_checkpoint")
            try:
                with open(marker, "r") as f:
                    last = f.read().strip()
                assert last != "model_final", "model training has finished, check your model in train.output_dir"
                self.start_iter = int(last.split("_")[-1]) + 1
            except IOError:
                self.start_iter = 0
        cfg.dataloader.consumed_samples = self.start_iter * cfg.train.global_batch_size

        # ---- data ------------------------------------------------------------------------------
        self.train_loader = None
        self.test_loader = []
        train_loader, val_loader, test_loader = self.build_train_loader(cfg, self.tokenizer)
        self.train_loader = train_loader
        for extra in (val_loader, test_loader):
            if extra is not None:
                self.test_loader.append(extra)
        self.test_loader.extend(self.build_test_loader(cfg, self.tokenizer))
        self.auto_scale_hyperparams(cfg, self.train_loader)

        # ---- model / optimizer -----------------------------------------------------------------
        dutil.synchronize()
        t0 = time.time()
        logger.info("> Start building model...")
        self.model = self.build_model(cfg)
        dutil.synchronize()
        logger.info(">>> done with building model. Building time: {:.3f} seconds".format(time.time() - t0))
        self.optimizer = self.build_optimizer(cfg, self.model)
        self.lr_scheduler = self.build_lr_scheduler(cfg, self.optimizer)
        self.loss_scaler = None
        if try_get_key(cfg, "train.amp.enabled", default=False) and try_get_key(cfg, "train.amp.dtype", default="bf16") == "fp16":
            self.loss_scaler = DynamicLossScaler(init_scale=65536.0 * dutil.get_data_parallel_size())

        self._trainer = StepTrainer(
            self.model, self.train_loader, self.optimizer, cfg.train.num_accumulation_steps,
            log_period=try_get_key(cfg, "train.log_period", default=1), loss_scaler=self.loss_scaler,
        )
        # NEW: replay the transformer blocks from CUDA graphs (engine/cuda_graphs.py); captured at the first step
        self._trainer.cuda_graphs = bool(try_get_key(cfg, "train.cuda_graphs.enabled", default=False))
        if try_get_key(cfg, "train.fp8.enabled", default=False):
            from libai_b200 import ops

            ops.set_fp8(True)   # NEW: E4M3 forward GEMMs (ops/functional.py:_linear_fwd_any)
        extra = {"loss_scaler": self.loss_scaler} if self.loss_scaler is not None else {}
        self.checkpointer = Checkpointer(
            self.model, cfg.train.output_dir, optimizer=self.optimizer, lr_scheduler=self.lr_scheduler, **extra
        )
        self.resume_or_load(try_get_key(cfg, "train.resume", default=False))
        cfg.train.start_iter = self.start_iter
        self.global_batch_size = cfg.train.global_batch_size
        self.max_iter = cfg.train.train_iter
        self.register_hooks(self.build_hooks())

    # ------------------------------------------------------------------ checkpoint
    def resume_or_load(self, resume=True):
        """``resume`` and a ``last_checkpoint`` exists → restore model, optimizer, scheduler (the
        iteration comes from the directory name); otherwise load ``cfg.train.load_weight`` weights."""
        weight_path = try_get_key(self.cfg, "train.load_weight", default="")
        if resume:
            assert self.checkpointer.has_checkpoint() or not weight_path or True
            self.checkpointer.resume_or_load(weight_path, resume=True)
        elif weight_path:
            assert os.path.isdir(weight_path) or os.path.isfile(weight_path), f"'{weight_path}' must be a checkpoint"
            self.checkpointer.load(weight_path, checkpointables=[])

    # ------------------------------------------------------------------ hooks / writers
    def build_hooks(self):
        cfg = self.cfg
        ret = [hooks.IterationTimer(), hooks.LRScheduler()]
        if os.environ.get("LIBAI_B200_FAULT_INJECT"):
            ret.append(hooks.FaultInjectionHook(os.environ["LIBAI_B200_FAULT_INJECT"]))
        if try_get_key(cfg, "train.checkpointer.period", default=0):
            ret.append(
                hooks.PeriodicCheckpointer(
                    self.checkpointer, cfg.train.checkpointer.period,
                    max_to_keep=try_get_key(cfg, "train.checkpointer.max_to_keep"),
                )
            )
        if try_get_key(cfg, "train.evaluation.enabled", default=False):
            assert cfg.train.evaluation.eval_iter > 0, "run_iter must be positive number"

            def test_and_save_results():
                model = self.model
                self._last_eval_results = self.test(self.cfg, self.test_loader, model)
                return self._last_eval_results

            ret.append(hooks.EvalHook(cfg.train.evaluation.eval_period, test_and_save_results))
            ret.append(
                hooks.BestCheckpointer(
                    cfg.train.evaluation.eval_period, self.checkpointer,
                    cfg.train.evaluation.eval_metric, mode=cfg.train.evaluation.eval_mode,
                )
            )
        # NEW: preemption-safe stop (SIGTERM → checkpoint at the step boundary) and an optional profiling window
        if try_get_key(cfg, "train.emergency_checkpoint.enabled", default=False):
            ret.append(hooks.EmergencyCheckpointHook(
                self.checkpointer, check_period=try_get_key(cfg, "train.emergency_checkpoint.check_period", default=1)))
        if try_get_key(cfg, "train.profiler.enabled", default=False):
            p = cfg.train.profiler
            ret.append(hooks.ProfilerHook(p.get("start_iter", 10), p.get("num_iters", 3),
                                          os.path.join(cfg.train.output_dir, "profiler"),
                                          torch_profiler=p.get("torch_profiler", True), nvtx=p.get("nvtx", True)))
        if dutil.is_main_process():
            ret.append(hooks.PeriodicWriter(self.build_writers(), cfg.train.log_period))
        return ret

    def build_writers(self):
        out = self.cfg.train.output_dir
        tokens = try_get_key(self.cfg, "model.cfg.max_seq_length", "model.cfg.max_position_embeddings", default=None)
        writers = [
            CommonMetricPrinter(self.global_batch_size, self.max_iter, tokens_per_sample=tokens),
            JSONWriter(os.path.join(out, "metrics.json")),
        ]
        try:
            writers.append(TensorboardXWriter(out))
        except Exception as e:  # tensorboard is optional
            logging.getLogger(__name__).warning(f"TensorBoard writer disabled: {e}")
        return writers

    # ------------------------------------------------------------------ loop
    def train(self):
        super().train(self.start_iter, self.max_iter)
        if hasattr(self, "_last_eval_results") and dutil.is_main_process():
            return self._last_eval_results

    def run_step(self):
        self._trainer.iter = self.iter
        self._trainer.start_iter = self.start_iter
        self._trainer.max_iter = self.max_iter
        self._trainer.storage = self.storage
        self._trainer.run_step(self.get_batch, try_get_key(self.cfg, "train.input_placement_device", default="cuda"))

    @classmethod
    def get_batch(cls, data: Instance, input_placement_device: str = "cuda", mixup_func: Optional[Callable] = None):
        """``Instance`` of ``DistTensorData`` → ``dict`` of device tensors keyed by forward kwarg.
        Mixup/CutMix (if any) runs here, on device."""
        if mixup_func is not None:
            dev = dutil.get_device()
            images, labels = mixup_func(data.get("images").tensor.to(dev), data.get("labels").tensor.to(dev))
            data.get("images").tensor = images
            data.get("labels").tensor = labels
        out = {}
        for key, value in data.get_fields().items():
            value.to_global(device_type=input_placement_device)
            out[key] = value.tensor
        return out

    # ------------------------------------------------------------------ builders
    @classmethod
    def build_tokenizer(cls, cfg):
        tokenizer = None
        if try_get_key(cfg, "tokenization") is not None:
            from libai_b200.tokenizer import build_tokenizer

            tokenizer = build_tokenizer(cfg.tokenization)
            if try_get_key(cfg, "model.cfg.vocab_size", default=None) is not None and tokenizer is not None:
                multiple = cfg.tokenization.make_vocab_size_divisible_by * cfg.train.dist.tensor_parallel_size
                if hasattr(tokenizer, "padded_vocab_size"):
                    cfg.model.cfg.vocab_size = tokenizer.padded_vocab_size(multiple)
        return tokenizer

    @classmethod
    def param_dtype(cls, cfg) -> torch.dtype:
        """bf16 parameters (fp32 master in the optimizer) when ``train.amp.enabled`` on GPU."""
        if try_get_key(cfg, "train.amp.enabled", default=False) and dutil.get_dist_util().device_type == "cuda":
            return {"bf16": torch.bfloat16, "fp16": torch.float16}[try_get_key(cfg, "train.amp.dtype", default="bf16")]
        return torch.float32

    @classmethod
    def build_model(cls, cfg):
        assert try_get_key(cfg, "model") is not None, "cfg must contain `model` namespace"
        if try_get_key(cfg.model, "cfg.amp_enabled") is not None:
            cfg.model.cfg.amp_enabled = bool(try_get_key(cfg, "train.amp.enabled", default=False))
        with param_defaults(dtype=cls.param_dtype(cfg), seed=try_get_key(cfg, "train.seed", default=1234)):
            model = cls.construct_model(cfg)
        if try_get_key(cfg, "train.activation_checkpoint.enabled", default=False):
            setter = getattr(type(model), "set_activation_checkpoint", None)
            if setter is not None:
                setter(model)
            for m in model.modules():
                if hasattr(m, "activation_checkpoint"):
                    m.activation_checkpoint = True
        return model

    @classmethod
    def construct_model(cls, cfg):
        """Instantiate ``cfg.model`` (called under the parameter dtype / seed defaults).  Override to start from a
        pretrained checkpoint — ``build_model`` still applies the dtype and activation-checkpoint settings."""
        return _build_model(cfg.model)

    @classmethod
    def build_graph(cls, cfg, model, optimizer=None, lr_scheduler=None, is_train=True):
        """API parity: there is no graph compiler; the model itself is returned."""
        return model

    @classmethod
    def build_optimizer(cls, cfg, model):
        opt = build_optimizer(cfg.optim, model)
        if hasattr(opt, "configure"):
            zero = try_get_key(cfg, "train.zero_optimization", default=None)
            stage = int(zero.stage) if zero is not None and zero.enabled else 0
            names = {id(p): n for n, p in model.named_parameters()}
            opt.configure(zero_stage=stage, param_names=names,
                          dp_grad_reduce=getattr(model, "dp_grad_reduce", "mean"), model=model)
            opt.setup()
            if getattr(opt, "bucket_hooks", None) is not None:
                model.zero_hooks = opt.bucket_hooks    # ZeRO-2/3: forward_stage brackets every block with them
        return opt

    @classmethod
    def build_lr_scheduler(cls, cfg, optimizer):
        assert try_get_key(cfg, "train.scheduler") is not None, "cfg.train must contain `scheduler` namespace"
        return build_lr_scheduler(cfg.train.scheduler, optimizer)

    @classmethod
    def build_train_loader(cls, cfg, tokenizer=None):
        assert try_get_key(cfg, "dataloader.train") is not None, "cfg must contain `dataloader.train` namespace"
        logging.getLogger(__name__).info("Prepare training, validating, testing set")
        ds = cfg.dataloader.train.dataset
        items = ds if isinstance(ds, (list,)) or hasattr(ds, "_iter_ex") else [ds]
        if tokenizer is not None:
            for d in items:
                if try_get_key(d, "tokenizer") is not None or "tokenizer" in d:
                    d.tokenizer = tokenizer
        cfg.dataloader.train.train_batch_size = cfg.train.train_micro_batch_size
        cfg.dataloader.train.test_batch_size = cfg.train.test_micro_batch_size
        cfg.dataloader.train.seed = cfg.train.seed
        if "consumed_samples" in cfg.dataloader:
            cfg.dataloader.train.consumed_samples = cfg.dataloader.consumed_samples
        if try_get_key(cfg, "dataloader.train.train_val_test_num_samples") is not None or \
                "splits" in cfg.dataloader.train:
            eval_iters = (cfg.train.train_iter // max(1, cfg.train.evaluation.eval_period) + 1) * cfg.train.evaluation.eval_iter
            cfg.dataloader.train.train_val_test_num_samples = [
                int(cfg.train.samples),
                int(eval_iters * cfg.train.test_micro_batch_size * dutil.get_data_parallel_size()),
                int(cfg.train.evaluation.eval_iter * cfg.train.test_micro_batch_size * dutil.get_data_parallel_size()),
            ]
        return instantiate(cfg.dataloader.train, _recursive_=False)

    @classmethod
    def build_test_loader(cls, cfg, tokenizer=None):
        if not try_get_key(cfg, "train.evaluation.enabled", default=False) or try_get_key(cfg, "dataloader.test") is None:
            return []
        logging.getLogger(__name__).info("Prepare testing set")
        loaders = []
        for i in range(len(cfg.dataloader.test)):
            cfg.dataloader.test[i].test_batch_size = cfg.train.test_micro_batch_size
            cfg.dataloader.test[i].seed = cfg.train.seed
            if tokenizer is not None and "tokenizer" in cfg.dataloader.test[i].dataset:
                cfg.dataloader.test[i].dataset.tokenizer = tokenizer
            loaders.append(instantiate(cfg.dataloader.test[i], _recursive_=False))
        return loaders

    @classmethod
    def auto_scale_hyperparams(cls, cfg, data_loader):
        """epochs → iterations, warm-up ratio → warm-up iterations, milestone ratios → iterations,
        "after n epoch" periods → iteration periods; injects ``max_iter`` / ``warmup_iter`` into the
        scheduler record."""
        logger = logging.getLogger(__name__)
        train_iter = try_get_key(cfg, "train.train_iter", default=0)
        train_epoch = try_get_key(cfg, "train.train_epoch", default=0)
        warmup_ratio = try_get_key(cfg, "train.warmup_ratio", default=0)
        assert 0 <= warmup_ratio < 1, "warmup_ratio must be in [0, 1) that presents the ratio of warmup iter to the train iter"
        n_data = len(data_loader.dataset)
        cfg.train.train_iter = max(math.ceil(n_data * train_epoch / cfg.train.global_batch_size), train_iter)
        cfg.train.warmup_iter = math.ceil(cfg.train.train_iter * warmup_ratio)
        msg = "Auto-scaling the config to train.train_iter={}, train.warmup_iter={}".format(
            cfg.train.train_iter, cfg.train.warmup_iter
        )
        milestones = try_get_key(cfg, "train.scheduler.milestones")
        if milestones:
            if any(m < 0 or m >= 1 for m in milestones):
                raise ValueError("milestones should be a list of increasing ratio in [0, 1), but got {}".format(milestones))
            cfg.train.scheduler.milestones = [int(m * cfg.train.train_iter) for m in milestones]
            msg += f", scheduler milestones={cfg.train.scheduler.milestones}"
        logger.info(msg)
        cfg.train.scheduler.warmup_iter = cfg.train.warmup_iter
        cfg.train.scheduler.max_iter = cfg.train.train_iter
        cfg.train.samples = cfg.train.train_iter * cfg.train.global_batch_size
        per_epoch = n_data // cfg.train.global_batch_size
        if try_get_key(cfg, "train.evaluation.eval_after_n_epoch"):
            cfg.train.evaluation.eval_period = per_epoch * cfg.train.evaluation.eval_after_n_epoch
            logger.info(f"Auto-scaling train.evaluation.eval_period={cfg.train.evaluation.eval_period}")
        if try_get_key(cfg, "train.checkpointer.save_model_after_n_epoch"):
            cfg.train.checkpointer.period = per_epoch * cfg.train.checkpointer.save_model_after_n_epoch
            logger.info(f"Auto-scaling train.checkpointer.period={cfg.train.checkpointer.period}")

    @classmethod
    def build_evaluator(cls, cfg):
        return instantiate(cfg.train.evaluation.evaluator)

    @classmethod
    def test(cls, cfg, test_loaders, model, evaluator=None):
        """Evaluate ``model`` on every loader; returns ``{dataset_name: metrics}`` (flattened to the
        metrics dict when there is a single loader)."""
        logger = logging.getLogger(__name__)
        batch = cfg.train.test_micro_batch_size * dutil.get_data_parallel_size()
        evaluator = evaluator or cls.build_evaluator(cfg)
        results = OrderedDict()
        for loader in test_loaders:
            name = type(loader.dataset).__name__
            res = inference_on_dataset(
                model, loader, batch, cfg.train.evaluation.eval_iter, cls.get_batch,
                try_get_key(cfg, "train.input_placement_device", default="cuda"), evaluator,
            )
            results[name] = res
            if dutil.is_main_process():
                assert isinstance(res, dict), "Evaluator must return a dict on the main process. Got {} instead.".format(res)
                logger.info("Evaluation results for {} in csv format:".format(colored(name, "green")))
                print_csv_format(res)
        if len(results) == 1:
            results = list(results.values())[0]
        return results
