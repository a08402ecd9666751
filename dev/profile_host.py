"""Host-side profile (cProfile) of a few training steps of a bench layout: where does the enqueue time go?

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 dev/profile_host.py --layout tp2
writes output/host_profile_<layout>_rank<r>.txt"""
import argparse
import cProfile
import io
import os
import pstats
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import bench  # noqa: E402


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
