"""Training loop skeleton, hooks protocol and the step executors.

Spec: reference libai/engine/trainer.py — ``HookBase`` (:32-87), ``TrainerBase`` (:90-219; hook
loop, ``write_metrics``), ``EagerTrainer`` (:222-286) and ``GraphTrainer`` (:289-349).

One execution mode replaces eager/graph: :class:`StepTrainer` runs one *optimizer step* per
iteration over ``num_accumulation_steps`` micro-batches (the reference's graph-mode semantics):
plain micro-batch loop when ``pp == 1``, the 1F1B schedule (``libai_b200/parallel/pipeline.py``)
otherwise; gradients accumulate in the fp32 flat buffers, data-parallel reduction / ZeRO /
clipping / update happen in ``optimizer.step()``.  Metrics are reduced and copied to the host only
every ``log_period`` iterations (the reference synchronises every step: trainer.py:191-194).
"""
from __future__ import annotations

import logging
import os
import time
import weakref
from typing import Callable, List, Mapping, Optional

import torch

from libai_b200.utils import distributed as dutil
from libai_b200.utils.events import EventStorage, get_event_storage

__all__ = ["HookBase", "TrainerBase", "StepTrainer", "EagerTrainer", "GraphTrainer"]


class TrainingInterrupted(Exception):
    """Raised by a hook (``EmergencyCheckpointHook``) to leave the training loop cleanly at a step boundary."""


class HookBase:
    """Callbacks around the loop::

        hook.before_train()
        for iter in range(start_iter, max_iter):
            hook.before_step(); trainer.run_step(); hook.after_step()
        hook.after_train()

    ``self.trainer`` is a weak proxy to the owning trainer (set on registration)."""

    trainer: "TrainerBase" = None

    def before_train(self):
        pass

    def after_train(self):
        pass

    def before_step(self):
        pass

    def after_step(self):
        pass


class TrainerBase:
    """Iterative trainer with hooks; subclasses implement :meth:`run_step`."""

    def __init__(self):
        self._hooks: List[HookBase] = []
        self.iter: int = 0
        self.start_iter: int = 0
        self.max_iter: int = 0
        self.storage: Optional[EventStorage] = None

    def register_hooks(self, hooks):
        hooks = [h for h in hooks if h is not None]
        for h in hooks:
            assert isinstance(h, HookBase)
            h.trainer = weakref.proxy(self)  # avoid a reference cycle trainer <-> hook
        self._hooks.extend(hooks)

    def train(self, start_iter: int, max_iter: int):
        logger = logging.getLogger(__name__)
        logger.info(f"Starting training from iteration {start_iter}")
        self.iter = self.start_iter = start_iter
        self.max_iter = max_iter
        with EventStorage(start_iter) as self.storage:
            try:
                self.before_train()
                for self.iter in range(start_iter, max_iter):
                    self.before_step()
                    self.run_step()
                    self.after_step()
                # the loop variable stops at max_iter - 1; after_train hooks expect max_iter
                self.iter += 1
            except TrainingInterrupted as stop:     # graceful: emergency checkpoint already written
                logger.warning("%s", stop)
                self.interrupted = True
            except Exception:
                logger.exception("Exception during training:")
                from libai_b200.ops import spin_timeout_report

                timeout = spin_timeout_report()
                if timeout:
                    logger.error("%s", timeout)
                raise
            finally:
                self.after_train()

    def before_train(self):
        for h in self._hooks:
            h.before_train()

    def after_train(self):
        self.storage.iter = self.iter
        for h in self._hooks:
            h.after_train()

    def before_step(self):
        self.storage.iter = self.iter
        for h in self._hooks:
            h.before_step()

    def after_step(self):
        self.storage.samples = (self.iter + 1) * getattr(self, "global_batch_size", 0)
        for h in self._hooks:
            h.after_step()

    def run_step(self):
        raise NotImplementedError

    @staticmethod
    def write_metrics(loss_dict: Mapping[str, torch.Tensor], data_time: float, prefix: str = "",
                      device_time: Optional[float] = None) -> None:
        """Average the scalars over the DP group, move to host, store in the EventStorage.
        Only the ranks of the *last* pipeline stage hold losses; rank 0 receives them."""
        topo = dutil.get_dist_util()
        metrics = {k: dutil.dp_mean_to_rank0(v) for k, v in loss_dict.items()}
        if topo.pipeline_parallel_size > 1 and torch.distributed.is_initialized():
            # ship from the last stage to the first (same dp/tp coordinates) through the host
            payload = {k: float(v) for k, v in metrics.items()} if topo.is_last_stage else None
            gathered = dutil.all_gather_py_object(payload)
            src = topo.world_size - 1
            metrics = {k: torch.tensor(v) for k, v in (gathered[src] or {}).items()}
        if not dutil.is_main_process():
            return
        host = {k: float(v) for k, v in metrics.items()}
        storage = get_event_storage()
        storage.put_scalar("data_time", data_time)
        if device_time is not None:
            storage.put_scalar("device_time", device_time)
        total = sum(v for k, v in host.items() if "loss" in k)
        if not all(map(lambda x: x == x and abs(x) != float("inf"), host.values())):
            raise FloatingPointError(f"Loss became infinite or NaN at iteration={storage.iter}!\nloss_dict = {host}")
        storage.put_scalar(f"{prefix}total_loss", total)
        if len(host) > 1:
            storage.put_scalars(**host)


class StepTrainer(TrainerBase):
    """One optimizer step per iteration (micro-batch accumulation, optional 1F1B pipeline)."""

    def __init__(self, model, data_loader, optimizer, grad_acc_steps: int = 1, *, log_period: int = 1,
                 loss_scaler=None):
        super().__init__()
        model.train()
        self.model = model
        self.data_loader = data_loader
        self._data_loader_iter = iter(data_loader)
        self.optimizer = optimizer
        self.grad_acc_steps = int(grad_acc_steps)
        self.log_period = max(1, int(log_period))
        self.loss_scaler = loss_scaler
        self._pipeline = None
        self._ev = None
        self.cuda_graphs = False       # set by DefaultTrainer from cfg.train.cuda_graphs.enabled
        self._graphs_tried = False
        self.graphs_enabled = False
        # inputs of the NEXT step are fetched (loader → pinned host → device) right behind this step's kernels, before
        # the host blocks on the metrics of a logging step: the device then finds its inputs resident instead of idling
        # through the loader hand-over and the copy (matters with log_period = 1, e.g. bench.py's end-to-end loop)
        self.prefetch_inputs = os.environ.get("LIBAI_B200_INPUT_PREFETCH", "1") == "1"
        self._staged_batches = None

    def _arm_grad_overlap(self, last_micro_batch: bool):
        """Opt-in (``LIBAI_B200_OVERLAP_GRAD_SYNC=1``): overlap the data-parallel gradient reduction with the backward
        pass of the last micro-batch (the fused NVLink reduce-scatter of the already-final part of the gradient buffer
        starts at a few block boundaries).  Off by default: for a model of the benchmark's size the end-of-step
        reduction is short, while the extra side-stream kernels, their flag exchanges and the added host work are paid
        on every step.  Meant for models whose gradient volume per step is much larger."""
        if not hasattr(self, "_overlap_layers"):
            self._overlap_layers = ()
            model = self.model.module if hasattr(self.model, "module") else self.model
            opt = self.optimizer
            if (hasattr(opt, "plan_overlap") and hasattr(model, "grad_ready_layers")
                    and dutil.get_dist_util().device_type == "cuda" and dutil.get_dist_util().data_parallel_size > 1
                    and os.environ.get("LIBAI_B200_OVERLAP_GRAD_SYNC", "0") == "1"):
                self._overlap_layers = tuple(opt.plan_overlap())
            self._overlap_model = model
        if not self._overlap_layers:
            return
        m = self._overlap_model
        m.grad_ready_layers = self._overlap_layers
        m.grad_ready_callback = self.optimizer.on_grads_ready if last_micro_batch else None

    def _next_batches(self, get_batch: Callable, input_placement_device: str):
        out = []
        mixup = getattr(self.data_loader, "mixup_func", None)
        for _ in range(self.grad_acc_steps):
            data = next(self._data_loader_iter)
            out.append(get_batch(data, input_placement_device, mixup))
        return out

    def train_on_batches(self, batches):
        """One optimizer step over already staged micro-batches (dicts of device tensors): forward/backward of every
        micro-batch (1F1B schedule under pipeline parallelism), gradient sync, clipping, update.  Returns the
        micro-batch averaged loss dict (device tensors; ``None`` on non-last pipeline stages).  Public so that callers
        that stage their own data (``bench.py``) run exactly the trainer's step."""
        topo = dutil.get_dist_util()
        if self.cuda_graphs and not self._graphs_tried and topo.device_type == "cuda":
            # first step: capture forward+backward of every transformer block into CUDA graphs (engine/cuda_graphs.py)
            from libai_b200.engine.cuda_graphs import enable_for_model

            self._graphs_tried = True
            model = self.model.module if hasattr(self.model, "module") else self.model
            self.graphs_enabled = enable_for_model(model, batches[0])
        self.optimizer.zero_grad()
        if topo.pipeline_parallel_size > 1:
            if self._pipeline is None:
                from libai_b200.parallel.pipeline import PipelineSchedule1F1B

                self._pipeline = PipelineSchedule1F1B(self.model, loss_scaler=self.loss_scaler)
            loss_dict = self._pipeline.run(batches)
        else:
            loss_dict = None
            inv = 1.0 / len(batches)
            for k, batch in enumerate(batches):
                self._arm_grad_overlap(k == len(batches) - 1)
                out = self.model(**batch)
                loss = sum(v for k, v in out.items() if "loss" in k) * inv
                if self.loss_scaler is not None:
                    loss = self.loss_scaler.scale_loss(loss)
                loss.backward()
                det = {k: v.detach() * inv for k, v in out.items()}
                loss_dict = det if loss_dict is None else {k: loss_dict[k] + det[k] for k in det}
        if self.loss_scaler is not None:
            self.loss_scaler.check_and_update(self.optimizer)
        self.optimizer.step()
        return loss_dict

    def run_step(self, get_batch: Callable, input_placement_device: str = "cuda"):
        assert self.model.training, "[StepTrainer] model was changed to eval mode!"
        topo = dutil.get_dist_util()
        t0 = time.perf_counter()
        batches, self._staged_batches = self._staged_batches, None
        if batches is None:
            batches = self._next_batches(get_batch, input_placement_device)
        data_time = time.perf_counter() - t0
        use_events = topo.device_type == "cuda"
        if use_events:
            if self._ev is None:
                self._ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            self._ev[0].record()

        loss_dict = self.train_on_batches(batches)

        device_time = None
        if use_events:
            self._ev[1].record()
        logging_step = (self.iter + 1) % self.log_period == 0 or self.iter == self.start_iter
        if logging_step and self.prefetch_inputs and (self.max_iter <= 0 or self.iter + 1 < self.max_iter):
            t1 = time.perf_counter()
            try:
                self._staged_batches = self._next_batches(get_batch, input_placement_device)
            except StopIteration:
                self._staged_batches = None
            data_time += time.perf_counter() - t1
        if logging_step:
            if use_events:
                self._ev[1].synchronize()
                device_time = self._ev[0].elapsed_time(self._ev[1]) * 1e-3
            self.write_metrics(loss_dict or {}, data_time, device_time=device_time)


# reference names: both map onto the single execution mode
EagerTrainer = StepTrainer
GraphTrainer = StepTrainer
