"""End-to-end: `tools/train_net.py` flow on CPU — training, periodic checkpoints, exact resume, evaluation, and
2-rank data-parallel training over gloo (the reference's model tests train real configs on 4 GPUs)."""
import json
import os
import sys

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "tools"))

TINY = [
    "model.cfg.hidden_layers=2", "model.cfg.hidden_size=32", "model.cfg.ffn_hidden_size=64",
    "model.cfg.num_attention_heads=2", "model.cfg.vocab_size=64", "model.cfg.max_seq_length=16",
    "dataloader.train.dataset.0.vocab_size=64", "dataloader.train.dataset.0.seq_length=16",
    "dataloader.train.dataset.0.num_samples=256", "dataloader.train.num_workers=0",
    "dataloader.test.0.dataset.vocab_size=64", "dataloader.test.0.dataset.seq_length=16",
    "dataloader.test.0.dataset.num_samples=8", "train.train_micro_batch_size=4", "train.test_micro_batch_size=4",
    "train.log_period=1", "train.amp.enabled=false", "train.warmup_ratio=0.0", "train.dist.pipeline_num_layers=2",
    "optim.lr=1e-2",
]


def _run(out_dir, extra, resume=False):
    import train_net
    from libai_b200.config import default_argument_parser

    argv = ["--config-file", os.path.join(REPO, "configs/gpt2_synthetic.py")] + (["--resume"] if resume else [])
    args = default_argument_parser().parse_args(argv + TINY + [f"train.output_dir={out_dir}"] + extra)
    train_net.main(args)
    metrics = [json.loads(ln) for ln in open(os.path.join(out_dir, "metrics.json"))]
    return [m for m in metrics if "total_loss" in m or "lm_loss" in m]


def _loss(m):
    return m.get("total_loss", m.get("lm_loss"))


def test_train_checkpoint_resume(tmp_path):
    full_dir, part_dir = str(tmp_path / "full"), str(tmp_path / "part")
    full = _run(full_dir, ["train.train_iter=12", "train.checkpointer.period=6"])
    assert len(full) >= 12 and all(3.0 < _loss(m) < 6.0 for m in full)     # uniform random tokens: loss ≈ ln(64)
    assert sorted(d for d in os.listdir(full_dir) if d.startswith("model_")) == ["model_0000005", "model_0000011", "model_final"]
    assert open(os.path.join(full_dir, "last_checkpoint")).read().strip() == "model_final"
    assert sorted(os.listdir(os.path.join(full_dir, "model_0000005"))) == ["lr_scheduler", "model", "optimizer"]

    # simulate a job killed after iteration 5: only the periodic checkpoint exists; resuming must continue the loss
    # curve of the uninterrupted run exactly (same data order via consumed_samples, same optimizer / LR state)
    import shutil

    os.makedirs(part_dir)
    shutil.copytree(os.path.join(full_dir, "model_0000005"), os.path.join(part_dir, "model_0000005"))
    with open(os.path.join(part_dir, "last_checkpoint"), "w") as f:
        f.write("model_0000005")
    resumed = _run(part_dir, ["train.train_iter=12", "train.checkpointer.period=6"], resume=True)
    assert sorted(m["iteration"] for m in resumed if m["iteration"] >= 6) == list(range(6, 12))
    # (logged losses are window-median smoothed, so exactness is checked on the final weights and optimizer state)
    a = torch.load(os.path.join(full_dir, "model_final", "model"), weights_only=False)
    b = torch.load(os.path.join(part_dir, "model_final", "model"), weights_only=False)
    assert a.keys() == b.keys()
    assert max((a[k].float() - b[k].float()).abs().max().item() for k in a) < 1e-6
    oa = torch.load(os.path.join(full_dir, "model_final", "optimizer"), weights_only=False)
    ob = torch.load(os.path.join(part_dir, "model_final", "optimizer"), weights_only=False)
    assert oa["step"] == ob["step"] == 12
    k0 = next(iter(oa["state"]))
    assert (oa["state"][k0]["exp_avg_sq"] - ob["state"][k0]["exp_avg_sq"]).abs().max() < 1e-9


def test_eval_only(tmp_path):
    out = str(tmp_path / "run")
    _run(out, ["train.train_iter=4", "train.checkpointer.period=100", "train.evaluation.enabled=true",
               "train.evaluation.eval_period=2", "train.evaluation.eval_iter=2"])
    assert os.path.isdir(os.path.join(out, "model_final"))


def _dp_worker(rank, world, out_dir):
    sys.path.insert(0, os.path.join(REPO, "tools"))
    metrics = _run(out_dir, ["train.train_iter=6", "train.checkpointer.period=100", "train.dist.data_parallel_size=2"])
    return [_loss(m) for m in metrics]


def test_two_rank_data_parallel(tmp_path):
    from tests.dist_utils import run_distributed

    res = run_distributed(_dp_worker, 2, str(tmp_path / "dp2"))
    losses = res[0]
    assert len(losses) >= 6 and all(3.0 < v < 6.0 for v in losses)


def test_sigterm_writes_checkpoint_and_resume_matches(tmp_path):
    """SIGTERM mid-run → emergency checkpoint at the step boundary + clean stop; ``--resume`` then
    finishes with exactly the weights of an uninterrupted run.  Also exercises the profiling window hook."""
    import signal

    from libai_b200.engine import DefaultTrainer, hooks

    full_dir, cut_dir = str(tmp_path / "full"), str(tmp_path / "cut")
    _run(full_dir, ["train.train_iter=10", "train.checkpointer.period=100"])

    orig = DefaultTrainer.build_hooks

    def with_kill(self):
        hs = orig(self)
        hs.insert(0, hooks.CallbackHook(after_step=lambda tr: os.kill(os.getpid(), signal.SIGTERM) if tr.iter == 3 else None))
        return hs

    DefaultTrainer.build_hooks = with_kill
    try:
        _run(cut_dir, ["train.train_iter=10", "train.checkpointer.period=100", "train.emergency_checkpoint.enabled=true",
                       "train.profiler.enabled=true", "train.profiler.start_iter=1", "train.profiler.num_iters=2"])
    finally:
        DefaultTrainer.build_hooks = orig
    saved = sorted(d for d in os.listdir(cut_dir) if d.startswith("model_"))
    assert "model_0000003" in saved and "model_0000009" not in saved, saved          # stopped right after iteration 3
    assert open(os.path.join(cut_dir, "last_checkpoint")).read().strip() in ("model_0000003", "model_final")
    assert os.path.exists(os.path.join(cut_dir, "profiler", "trace_rank0.json"))
    if os.path.isdir(os.path.join(cut_dir, "model_final")):                           # written by after_train at the stop
        import shutil

        shutil.rmtree(os.path.join(cut_dir, "model_final"))
    with open(os.path.join(cut_dir, "last_checkpoint"), "w") as f:
        f.write("model_0000003")
    _run(cut_dir, ["train.train_iter=10", "train.checkpointer.period=100"], resume=True)
    a = torch.load(os.path.join(full_dir, "model_final", "model"), weights_only=False)
    b = torch.load(os.path.join(cut_dir, "model_final", "model"), weights_only=False)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


def test_load_weight_refreshes_master_under_amp(tmp_path):
    """ADVICE r1 (high): ``train.load_weight`` into a bf16 (AMP) run must survive the first optimizer step — the fp32
    master copy is re-derived from the loaded parameters instead of keeping the random-init snapshot."""
    src = str(tmp_path / "src")
    _run(src, ["train.train_iter=2", "train.checkpointer.period=100"])
    ckpt = os.path.join(src, "model_final")
    saved = torch.load(os.path.join(ckpt, "model"), weights_only=False)
    dst = str(tmp_path / "dst")
    # lr = 0 → after one step the weights must still equal the loaded ones (bf16-rounded), not a random init
    _run(dst, ["train.train_iter=1", "train.checkpointer.period=100", "train.amp.enabled=true", f"train.load_weight={ckpt}",
               "optim.lr=0.0", "optim.weight_decay=0.0", "train.scheduler.warmup_iter=0"])
    out = torch.load(os.path.join(dst, "model_final", "model"), weights_only=False)
    k = "GPT_model.transformer.layers.0.mlp.dense_h_to_4h.weight"
    # (equal up to the bf16 rounding of the parameters; a stale random-init master would be off by ~1e-2)
    assert (out[k].float() - saved[k].float()).abs().max() < 5e-4, (out[k].float() - saved[k].float()).abs().max()


def _pp_eval_worker(rank, world, out_dir):
    sys.path.insert(0, os.path.join(REPO, "tools"))
    metrics = _run(out_dir, ["train.train_iter=4", "train.checkpointer.period=100", "train.dist.pipeline_parallel_size=2",
                             "train.num_accumulation_steps=2", "train.evaluation.enabled=true",
                             "train.evaluation.eval_period=2", "train.evaluation.eval_iter=2"])
    return [_loss(m) for m in metrics]


def test_two_stage_pipeline_train_and_eval(tmp_path):
    """ADVICE r1 (medium): evaluation under pp > 1 goes through the pipelined forward (stage hop + broadcast of the
    last stage's outputs) instead of calling ``forward_stage`` with no input on the later stages."""
    from tests.dist_utils import run_distributed

    out = str(tmp_path / "pp2")
    run_distributed(_pp_eval_worker, 2, out)
    assert os.path.isdir(os.path.join(out, "model_final"))


def _pp_load_pp1_worker(rank, world, ckpt, out_dir):
    sys.path.insert(0, os.path.join(REPO, "tools"))
    _run(out_dir, ["train.train_iter=1", "train.checkpointer.period=100", "train.dist.pipeline_parallel_size=2",
                   "train.num_accumulation_steps=2", f"train.load_weight={ckpt}", "optim.lr=0.0", "optim.weight_decay=0.0"])
    return 0


def test_pp1_checkpoint_into_pp2_fills_tied_copy(tmp_path):
    """ADVICE r1 (medium): a pp=1 checkpoint has no ``tied_weight_copy``; the last stage's LM-head copy must be filled
    from the embedding so both stay identical."""
    from tests.dist_utils import run_distributed

    src = str(tmp_path / "src")
    _run(src, ["train.train_iter=2", "train.checkpointer.period=100"])
    ckpt = os.path.join(src, "model_final")
    out = str(tmp_path / "pp2")
    run_distributed(_pp_load_pp1_worker, 2, ckpt, out)
    sd = torch.load(os.path.join(out, "model_final", "model"), weights_only=False)
    emb = sd["GPT_model.embeddings.token_embeddings.weight"]
    tied = sd["GPT_model.tied_weight_copy"]
    ref = torch.load(os.path.join(ckpt, "model"), weights_only=False)["GPT_model.embeddings.token_embeddings.weight"]
    assert torch.equal(emb, ref) and torch.equal(tied, ref)
