"""Training hooks.

Spec: reference libai/engine/hooks.py — ``CallbackHook`` (:46-78), ``IterationTimer`` (:81-145;
skips the first warm-up iterations, prints the "Overall training speed" summary),
``PeriodicWriter`` (:148-174), ``PeriodicCheckpointer`` (:177-190), ``BestCheckpointer``
(:193-293; rank 0 decides, decision broadcast so every rank enters the collective save),
``EvalHook`` (:296-354), ``LRScheduler`` (:357-417).  Hook order used by ``DefaultTrainer``:
``[IterationTimer, LRScheduler, PeriodicCheckpointer, EvalHook, BestCheckpointer, PeriodicWriter]``.
"""
from __future__ import annotations

import datetime
import logging
import math
import operator
import time
from collections import Counter

from libai_b200.evaluation.utils import flatten_results_dict
from libai_b200.utils import distributed as dutil
from libai_b200.utils.checkpoint import Checkpointer
from libai_b200.utils.checkpoint import PeriodicCheckpointer as _PeriodicCheckpointer
from libai_b200.utils.timer import Timer

from .trainer import HookBase, TrainingInterrupted

logger = logging.getLogger(__name__)

__all__ = [
    "CallbackHook", "IterationTimer", "PeriodicWriter", "PeriodicCheckpointer", "BestCheckpointer",
    "EvalHook", "LRScheduler", "EmergencyCheckpointHook", "ProfilerHook", "TrainingInterrupted",
]


class CallbackHook(HookBase):
    """Build a hook from plain callables (each receives the trainer)."""

    def __init__(self, *, before_train=None, after_train=None, before_step=None, after_step=None):
        self._before_train, self._after_train = before_train, after_train
        self._before_step, self._after_step = before_step, after_step

    def before_train(self):
        if self._before_train:
            self._before_train(self.trainer)

    def after_train(self):
        if self._after_train:
            self._after_train(self.trainer)
        # drop references so closures over the trainer can be collected
        del self._before_train, self._after_train, self._before_step, self._after_step

    def before_step(self):
        if self._before_step:
            self._before_step(self.trainer)

    def after_step(self):
        if self._after_step:
            self._after_step(self.trainer)


class IterationTimer(HookBase):
    """Records wall time per iteration under ``"time"`` (excluding time spent in other hooks and
    the first ``warmup_iter`` iterations) and logs the overall speed at the end."""

    def __init__(self, warmup_iter=3):
        self._warmup_iter = warmup_iter
        self._step_timer = Timer()

    def before_train(self):
        self._start_time = time.perf_counter()
        self._total_timer = Timer()
        self._total_timer.pause()

    def after_train(self):
        total = time.perf_counter() - self._start_time
        in_steps = self._total_timer.seconds()
        n_iter = self.trainer.iter + 1 - self.trainer.start_iter - self._warmup_iter
        if n_iter > 0 and in_steps > 0:
            logger.info(
                "Overall training speed: {} iterations in {} ({:.4f} s / it)".format(
                    n_iter, str(datetime.timedelta(seconds=int(in_steps))), in_steps / n_iter
                )
            )
        logger.info(
            "Total training time: {} ({} on hooks)".format(
                str(datetime.timedelta(seconds=int(total))),
                str(datetime.timedelta(seconds=int(total - in_steps))),
            )
        )

    def before_step(self):
        self._step_timer.reset()
        self._total_timer.resume()

    def after_step(self):
        done = self.trainer.iter - self.trainer.start_iter + 1
        if done >= self._warmup_iter:
            self.trainer.storage.put_scalars(time=self._step_timer.seconds())
        else:
            self._start_time = time.perf_counter()
            self._total_timer.reset()
        self._total_timer.pause()


class PeriodicWriter(HookBase):
    """Calls every ``EventWriter`` each ``period`` iterations and after the last one."""

    def __init__(self, writers, period=20):
        self._writers = writers
        self._period = period

    def after_step(self):
        if (self.trainer.iter + 1) % self._period == 0 or self.trainer.iter == self.trainer.max_iter - 1:
            for w in self._writers:
                w.write()

    def after_train(self):
        for w in self._writers:
            w.write()
            w.close()


class PeriodicCheckpointer(_PeriodicCheckpointer, HookBase):
    """``utils.checkpoint.PeriodicCheckpointer`` driven by the trainer's iteration counter."""

    def before_train(self):
        self.max_iter = self.trainer.max_iter

    def after_step(self):
        self.step(self.trainer.iter)


class BestCheckpointer(HookBase):
    """Save ``model_best`` whenever ``val_metric`` (produced by ``EvalHook``) improves."""

    def __init__(self, eval_period: int, checkpointer: Checkpointer, val_metric: str, mode: str = "max",
                 file_prefix: str = "model_best") -> None:
        assert mode in ("max", "min"), f'Mode "{mode}" to `BestCheckpointer` is unknown. It should be one of max, min.'
        self._period = eval_period
        self._val_metric = val_metric
        self._compare = operator.gt if mode == "max" else operator.lt
        self._checkpointer = checkpointer
        self._file_prefix = file_prefix
        self.best_metric = None
        self.best_iter = None

    def _update_best(self, val, iteration) -> bool:
        if math.isnan(val) or math.isinf(val):
            return False
        self.best_metric, self.best_iter = val, iteration
        return True

    def _best_checking(self):
        save = False
        if dutil.is_main_process():
            entry = self.trainer.storage.latest().get(self._val_metric)
            if entry is None:
                logger.warning(
                    f"Given val metric {self._val_metric} does not seem to be computed/stored. "
                    "Will not be checkpointed based on that."
                )
            else:
                latest, it = entry
                if self.best_metric is None:
                    if self._update_best(latest, it):
                        save = True
                        logger.info(f"Saved first model at {self.best_metric:0.5f} @ {self.best_iter} steps")
                elif self._compare(latest, self.best_metric):
                    save = True
                    logger.info(
                        f"Saved best model as latest eval score for {self._val_metric} is {latest:0.5f}, "
                        f"better than last best score {self.best_metric:0.5f} @ iteration {self.best_iter}."
                    )
                    self._update_best(latest, it)
                else:
                    logger.info(
                        f"Not saving as latest eval score for {self._val_metric} is {latest:0.5f}, "
                        f"not better than best score {self.best_metric:0.5f} @ iteration {self.best_iter}."
                    )
        # the save is collective: every rank must take the same branch
        if dutil.broadcast_py_object(save, src=0):
            self._checkpointer.save(f"{self._file_prefix}")

    def after_step(self):
        nxt = self.trainer.iter + 1
        if self._period > 0 and nxt % self._period == 0 and nxt != self.trainer.max_iter:
            self._best_checking()

    def after_train(self):
        if self.trainer.iter + 1 >= self.trainer.max_iter:
            self._best_checking()


class EvalHook(HookBase):
    """Run ``eval_function`` every ``eval_period`` iterations and after the final one (must be
    enabled on all ranks or none)."""

    def __init__(self, eval_period, eval_function):
        self._period = eval_period
        self._func = eval_function

    def _do_eval(self):
        results = self._func()
        if results:
            assert isinstance(results, dict), "Eval function must return a dict. Got {} instead.".format(results)
            flat = flatten_results_dict(results)
            for k, v in flat.items():
                try:
                    float(v)
                except Exception:
                    raise ValueError(
                        "[EvalHook] eval_function should return a nested dict of float. "
                        "Got '{}: {}' instead.".format(k, v)
                    )
            self.trainer.storage.put_scalars(**flat, smoothing_hint=False)
        dutil.synchronize()

    def after_step(self):
        nxt = self.trainer.iter + 1
        if self._period > 0 and nxt % self._period == 0 and nxt != self.trainer.max_iter:
            self._do_eval()

    def after_train(self):
        # not after a crash: only when training actually reached the end
        if self.trainer.iter + 1 >= self.trainer.max_iter:
            self._do_eval()
        del self._func


class LRScheduler(HookBase):
    """Steps the LR scheduler after every iteration and logs the lr of the dominant param group."""

    def __init__(self, optimizer=None, scheduler=None):
        self._optimizer = optimizer
        self._scheduler = scheduler

    def before_train(self):
        self._optimizer = self._optimizer or self.trainer.optimizer
        self._best_param_group_id = LRScheduler.get_best_param_group_id(self._optimizer)

    @staticmethod
    def get_best_param_group_id(optimizer):
        """Index of the group whose lr is most representative: the biggest group, or – when every
        group holds one parameter – the first group with the most common lr."""
        groups = optimizer.param_groups
        sizes = [len(g["params"]) for g in groups]
        if max(sizes) == 1:
            common = Counter(g["lr"] for g in groups).most_common()[0][0]
            return next(i for i, g in enumerate(groups) if g["lr"] == common)
        return sizes.index(max(sizes))

    def after_step(self):
        lr = self.scheduler.get_last_lr()[self._best_param_group_id]
        self.trainer.storage.put_scalar("lr", lr, smoothing_hint=False)
        self.scheduler.step()

    @property
    def scheduler(self):
        return self._scheduler or self.trainer.lr_scheduler

    def state_dict(self):
        sd = getattr(self.scheduler, "state_dict", None)
        return sd() if sd else {}

    def load_state_dict(self, state_dict):
        if hasattr(self.scheduler, "load_state_dict"):
            logger.info("Loading scheduler from state_dict ...")
            self.scheduler.load_state_dict(state_dict)


# ---------------------------------------------------------------------------------------------------------------
# NEW (not in the reference): preemption-safe stop and a profiling window
# ---------------------------------------------------------------------------------------------------------------
class EmergencyCheckpointHook(HookBase):
    """SIGTERM (schedulers send it before killing a job) → write a resumable checkpoint at the next step boundary and
    stop.  The handler only sets a flag; at the end of a step the ranks agree on it (``all_reduce(MAX)`` — the signal may
    reach only some of them, but the save is collective), save ``model_{iter:07d}`` with the usual ``iteration`` entry so
    ``--resume`` continues from the following step, and leave the loop through :class:`TrainingInterrupted`."""

    def __init__(self, checkpointer, signals=None, check_period: int = 1):
        import signal

        self.checkpointer = checkpointer
        self.signals = tuple(signals) if signals is not None else (signal.SIGTERM,)
        self.check_period = max(1, int(check_period))
        self._flag = False
        self._previous = {}

    def _handler(self, signum, frame):
        self._flag = True
        logger.warning("signal %s received: checkpoint + stop at the next step boundary", signum)

    def before_train(self):
        import signal
        import threading

        if threading.current_thread() is threading.main_thread():      # signal.signal only works there
            for sig in self.signals:
                self._previous[sig] = signal.signal(sig, self._handler)

    def after_train(self):
        import signal

        for sig, old in self._previous.items():
            signal.signal(sig, old)
        self._previous = {}

    def _agreed(self) -> bool:
        import torch
        import torch.distributed as dist

        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
            return self._flag
        dev = dutil.get_device() if dist.get_backend() == "nccl" else "cpu"
        t = torch.tensor([1 if self._flag else 0], dtype=torch.int32, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return bool(t.item())

    def after_step(self):
        if (self.trainer.iter + 1) % self.check_period != 0:
            return
        if self._agreed():
            it = int(self.trainer.iter)
            self.checkpointer.save(f"model_{it:07d}", iteration=it)
            raise TrainingInterrupted(f"stopped by signal after iteration {it}; checkpoint model_{it:07d} written")


class ProfilerHook(HookBase):
    """Profile a window of iterations: every step inside ``[start_iter, start_iter + num_iters)`` is wrapped in a
    process-wide NVTX range ``train_step`` (select it with ``ncu/nsys --nvtx --nvtx-include train_step``; start/end
    ranges because the backward kernels are launched from the autograd thread) and, with ``torch_profiler=True``,
    recorded by ``torch.profiler`` into a Chrome trace ``{output_dir}/trace_rank{r}.json``."""

    def __init__(self, start_iter: int, num_iters: int = 3, output_dir: str = ".", torch_profiler: bool = True,
                 nvtx: bool = True):
        self.start_iter, self.num_iters = int(start_iter), max(1, int(num_iters))
        self.output_dir, self.use_torch_profiler, self.use_nvtx = output_dir, torch_profiler, nvtx
        self._prof, self._range = None, None

    def _inside(self) -> bool:
        return self.start_iter <= self.trainer.iter < self.start_iter + self.num_iters

    def before_step(self):
        import torch

        if not self._inside():
            return
        if self.use_torch_profiler and self._prof is None:
            acts = [torch.profiler.ProfilerActivity.CPU]
            if torch.cuda.is_available():
                acts.append(torch.profiler.ProfilerActivity.CUDA)
            self._prof = torch.profiler.profile(activities=acts, record_shapes=False)
            self._prof.__enter__()
        if self.use_nvtx and torch.cuda.is_available():
            self._range = torch.cuda.nvtx.range_start("train_step")

    def after_step(self):
        import os

        import torch

        if self._range is not None:
            torch.cuda.synchronize()
            torch.cuda.nvtx.range_end(self._range)
            self._range = None
        if self._prof is not None and self.trainer.iter + 1 >= self.start_iter + self.num_iters:
            self._prof.__exit__(None, None, None)
            os.makedirs(self.output_dir, exist_ok=True)
            path = os.path.join(self.output_dir, f"trace_rank{dutil.get_rank()}.json")
            self._prof.export_chrome_trace(path)
            logger.info("profiler: wrote %s", path)
            self._prof = None

    def after_train(self):
        if self._prof is not None:       # training ended inside the window
            self._prof.__exit__(None, None, None)
            self._prof = None


class FaultInjectionHook(HookBase):
    """Test facility for the failure-recovery path: ``LIBAI_B200_FAULT_INJECT="<rank>:<iteration>"`` makes
    that rank die abruptly (``os._exit``, no cleanup, no checkpoint) right after the given iteration — the launcher
    (``torchrun``) then tears the job down and a relaunch with ``--resume`` must continue from the last periodic
    checkpoint (``tests/test_fault_recovery_cpu.py``)."""

    def __init__(self, spec: str):
        rank, it = spec.split(":")
        self.rank, self.iteration = int(rank), int(it)

    def after_step(self):
        from libai_b200.utils import distributed as dutil

        if self.trainer.iter == self.iteration and dutil.get_rank() == self.rank:
            import os
            import sys

            sys.stderr.write(f"[fault injection] rank {self.rank} dies after iteration {self.iteration}\n")
            sys.stderr.flush()
            os._exit(17)
