"""Dynamic loss scaling for fp16 training (bf16 – the H100 default – needs none).

Spec: reference libai/models/utils/graph_base.py:53-61 – ``GradScaler(init_scale=65536·D,
growth_factor=2, backoff_factor=0.5, growth_interval=2000)``.
"""
import torch
import torch.distributed as dist

from libai_b200.utils import distributed as dutil


class DynamicLossScaler:
    def __init__(self, init_scale=2.0 ** 16, growth_factor=2.0, backoff_factor=0.5, growth_interval=2000):
        self.scale = float(init_scale)
        self.growth_factor, self.backoff_factor = growth_factor, backoff_factor
        self.growth_interval = int(growth_interval)
        self._good_steps = 0

    def scale_loss(self, loss):
        return loss * self.scale

    def check_and_update(self, optimizer) -> bool:
        """Inspect the (synced) gradients; returns True when the step must be skipped."""
        optimizer.sync_gradients()
        bad = torch.zeros((), dtype=torch.float32, device=dutil.get_device())
        for fg in optimizer._groups:
            if fg is not None:
                bad = bad + (~torch.isfinite(fg.grad_shard())).any().float()
        if dist.is_initialized() and dutil.get_world_size() > 1:
            dist.all_reduce(bad, op=dist.ReduceOp.MAX)
        overflow = bool(bad.item() > 0)
        optimizer.grad_scale = 1.0 / self.scale
        optimizer.found_inf = overflow
        if overflow:
            self.scale = max(self.scale * self.backoff_factor, 1.0)
            self._good_steps = 0
        else:
            self._good_steps += 1
            if self._good_steps >= self.growth_interval:
                self.scale *= self.growth_factor
                self._good_steps = 0
        return overflow

    def state_dict(self):
        return {"scale": self.scale, "good_steps": self._good_steps}

    def load_state_dict(self, sd):
        self.scale, self._good_steps = float(sd["scale"]), int(sd["good_steps"])
