"""Where does the HOST time of a training step go?  Runs the benchmark model for a few steps under cProfile (1 GPU)
and prints the functions with the largest own time.  (Python / dispatcher overhead per kernel
matters when the step comes close to being launch-bound: `bench.py` reports `host_enqueue_ms_per_step`.)

    python tools/host_profile.py [--steps 6]
"""
import argparse
import cProfile
import io
import os
import pstats
import sys
import time

REPO = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, REPO)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=6)
    a = ap.parse_args()
    import torch

    import bench
    from libai_b200.engine import DefaultTrainer, default_setup

    sys.argv = [sys.argv[0]]          # bench's own defaults (the headline configuration)
    args = bench.parse_args()
    cfg = bench.build_cfg(args, 1)
    default_setup(cfg, argparse.Namespace(resume=False, config_file=""))
    trainer = DefaultTrainer(cfg)
    model, opt = trainer.model, trainer.optimizer
    it = iter(trainer.train_loader)
    batches = [DefaultTrainer.get_batch(next(it), "cuda") for _ in range(4)]

    def one(i):
        opt.zero_grad()
        out = model(**batches[i % 4])
        sum(v for k, v in out.items() if "loss" in k).backward()
        opt.step()

    for i in range(3):
        one(i)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pr = cProfile.Profile()
    pr.enable()
    for i in range(a.steps):
        one(i)
    pr.disable()
    enq = (time.perf_counter() - t0) / a.steps * 1e3
    torch.cuda.synchronize()
    total = (time.perf_counter() - t0) / a.steps * 1e3
    s = io.StringIO()
    st = pstats.Stats(pr, stream=s)
    st.sort_stats("tottime").print_stats(45)
    print(f"host enqueue (profiled, inflated by cProfile) {enq:.1f} ms/step, wall incl. device {total:.1f} ms/step")
    print(s.getvalue()[:9000])


if __name__ == "__main__":
    main()
