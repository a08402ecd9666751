"""Kill a rank mid-run → the launcher tears the job down → relaunch with ``--resume`` continues from the last periodic
checkpoint and ends with exactly the weights of an uninterrupted run.
Two data-parallel CPU ranks under ``torchrun`` (gloo)."""
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TINY = [
    "model.cfg.hidden_layers=2", "model.cfg.hidden_size=32", "model.cfg.ffn_hidden_size=64",
    "model.cfg.num_attention_heads=2", "model.cfg.vocab_size=64", "model.cfg.max_seq_length=16",
    "dataloader.train.dataset.0.vocab_size=64", "dataloader.train.dataset.0.seq_length=16",
    "dataloader.train.dataset.0.num_samples=256", "dataloader.train.num_workers=0",
    "train.train_micro_batch_size=4", "train.log_period=1", "train.amp.enabled=false", "train.warmup_ratio=0.0",
    "train.dist.pipeline_num_layers=2", "train.dist.data_parallel_size=2", "train.evaluation.enabled=false",
    "optim.lr=1e-2", "train.train_iter=10", "train.checkpointer.period=3",
]


def _launch(out_dir, port, resume=False, fault=None):
    env = dict(os.environ)
    env["PYTHONPATH"] = REPO + os.pathsep + env.get("PYTHONPATH", "")
    env["OMP_NUM_THREADS"] = "1"
    env["CUDA_VISIBLE_DEVICES"] = ""
    if fault:
        env["LIBAI_B200_FAULT_INJECT"] = fault
    else:
        env.pop("LIBAI_B200_FAULT_INJECT", None)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(REPO, "tools", "train_net.py"), "--config-file",
           os.path.join(REPO, "configs", "gpt2_synthetic.py")] + (["--resume"] if resume else []) + TINY + [
               f"train.output_dir={out_dir}"]
    return subprocess.run(cmd, cwd=REPO, env=env, capture_output=True, text=True, timeout=600)


def test_killed_rank_then_resume_matches_uninterrupted_run(tmp_path):
    full, cut = str(tmp_path / "full"), str(tmp_path / "cut")
    r = _launch(full, 29631)
    assert r.returncode == 0, r.stderr[-2000:]
    # rank 1 dies right after iteration 4: checkpoints of iterations 2 exists (period 3 → model_0000002), not 5
    r = _launch(cut, 29632, fault="1:4")
    assert r.returncode != 0, "the job must fail when a rank dies"
    assert "fault injection" in r.stderr
    saved = sorted(d for d in os.listdir(cut) if d.startswith("model_"))
    assert saved == ["model_0000002"], saved
    assert open(os.path.join(cut, "last_checkpoint")).read().strip() == "model_0000002"
    r = _launch(cut, 29633, resume=True)
    assert r.returncode == 0, r.stderr[-2000:]
    a = torch.load(os.path.join(full, "model_final", "model"), weights_only=False)
    b = torch.load(os.path.join(cut, "model_final", "model"), weights_only=False)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
