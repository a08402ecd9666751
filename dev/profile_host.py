"""Host-side profile (cProfile) of a few training steps of a bench layout: where does the enqueue time go?

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 dev/profile_host.py --layout tp2
writes output/host_profile_<layout>_rank<r>.txt

With ``--device 1`` the timed steps are traced with torch.profiler (CUDA activity) instead, e.g. the headline:

    python dev/profile_host.py --layout dp --device 1 --steps 5
writes output/device_profile_<layout>_rank<r>.txt (kernel table) and .json: device time per step of each kernel class
(GEMM by operand layout, attention forward / backward, norm, elementwise, optimizer, PyTorch's own kernels)."""
import argparse
import cProfile
import io
import json
import os
import pstats
import re
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import bench  # noqa: E402


_GEMM_LAYOUT = {("false", "false"): "NT (forward)", ("false", "true"): "NN (dgrad)", ("true", "true"): "TN (wgrad)"}


def kernel_class(name: str) -> str:
    m = re.search(r"gemm_kernel<\d+, (true|false), (true|false), \d+, (true|false)>", name)
    if m:
        return ("fp8 " if m.group(3) == "true" else "") + "gemm " + _GEMM_LAYOUT[(m.group(1), m.group(2))]
    m = re.search(r"gemm_pingpong_kernel<(true|false)>", name)
    if m:
        return "gemm " + _GEMM_LAYOUT[("false", m.group(1))]
    if "attn_fwd" in name:
        return "attention fwd"
    if "attn_" in name:          # attn_bwd_kernel and its delta / dQ-convert kernels
        return "attention bwd"
    if "norm_fwd" in name or "norm_bwd" in name:
        return "norm"
    if any(k in name for k in ("adamw", "sqnorm", "zero_")):
        return "optimizer"
    if "lb::" in name:
        return "elementwise (native)"
    if "memcpy" in name.lower() or "memset" in name.lower():
        return "memcpy / memset"
    return "pytorch"


def device_summary(tprof, steps: int, res) -> dict:
    per_class, per_kernel = {}, {}
    for e in tprof.key_averages():
        us = getattr(e, "self_device_time_total", None)
        if us is None:
            us = e.self_cuda_time_total
        if us <= 0:
            continue
        per_kernel[e.key] = per_kernel.get(e.key, 0.0) + us / 1e3 / steps
        c = kernel_class(e.key)
        per_class[c] = per_class.get(c, 0.0) + us / 1e3 / steps
    top = sorted(per_kernel.items(), key=lambda kv: -kv[1])[:25]
    return {
        "ms_per_step_profiled": round(res["ms_per_step"], 2) if isinstance(res, dict) else None,
        "kernel_ms_per_step": round(sum(per_class.values()), 2),
        "classes_ms_per_step": {k: round(v, 2) for k, v in sorted(per_class.items(), key=lambda kv: -kv[1])},
        "top_kernels_ms_per_step": [[k[:140], round(v, 3)] for k, v in top],
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layout", default="tp2")
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--device", type=int, default=0, help="1: torch.profiler (CUPTI) kernel table of the timed steps instead of cProfile")
    a, rest = ap.parse_known_args()      # everything else goes to bench.py (e.g. --model llama7b --layers 8 --zero 2)
    sys.argv = [sys.argv[0], "--gpus", os.environ.get("WORLD_SIZE", "1"), "--layout", a.layout] + rest
    args = bench.parse_args()
    import torch

    from libai_b200.utils import distributed as dutil

    world, rank, local_rank = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local_rank)
    dutil.init_process_group("cuda")
    lay = bench.layout_of(args, world)
    prof = cProfile.Profile()
    import time as _time
    import types

    orig = _time.perf_counter
    state = {"on": False}
    tprof = None
    if a.device:
        from torch.profiler import ProfilerActivity, profile

        tprof = profile(activities=[ProfilerActivity.CUDA])

    # profile exactly the timed loop: measure_native reads perf_counter right before and right after it
    def hooked():
        if not state["on"]:
            state["on"] = True
            tprof.__enter__() if tprof is not None else prof.enable()
        else:
            if tprof is not None:
                torch.cuda.synchronize()
                tprof.__exit__(None, None, None)
            else:
                prof.disable()
        return orig()

    # only bench.py's own `time.perf_counter()` calls (the two around the timed loop) must trigger: rebind the name
    # `time` inside the bench module to a shim instead of patching the global module
    bench.time = types.SimpleNamespace(perf_counter=hooked, sleep=_time.sleep, time=_time.time)
    res = bench.measure_native(args, lay, world, rank, local_rank, a.steps, 4, False)
    bench.time = _time
    os.makedirs(os.path.join(REPO, "output"), exist_ok=True)
    if tprof is not None:
        table = tprof.key_averages().table(sort_by="cuda_time_total", row_limit=45, max_name_column_width=90)
        with open(os.path.join(REPO, "output", f"device_profile_{a.layout}_rank{rank}.txt"), "w") as f:
            f.write(f"{res}\nsteps profiled: {a.steps}\n\n{table}")
        summary = device_summary(tprof, a.steps, res)
        with open(os.path.join(REPO, "output", f"device_profile_{a.layout}_rank{rank}.json"), "w") as f:
            json.dump(summary, f, indent=1)
        if rank == 0:
            print(json.dumps(summary))
    else:
        buf = io.StringIO()
        pstats.Stats(prof, stream=buf).sort_stats("cumulative").print_stats(70)
        with open(os.path.join(REPO, "output", f"host_profile_{a.layout}_rank{rank}.txt"), "w") as f:
            f.write(f"{res}\n\n{buf.getvalue()}")
    if rank == 0:
        print(res)
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
