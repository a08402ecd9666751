"""The ``train`` namespace shared by every recipe (keys: reference configs/common/train.py:8-150;
additions are marked NEW)."""
from libai_b200.config import DictConfig, LazyCall
from libai_b200.evaluation import ClsEvaluator
from libai_b200.scheduler import WarmupCosineLR

train = dict(
    # Directory where output files are written
    output_dir="./output",
    # `train_micro_batch_size` is the number of samples per batch on each GPU;
    # train_mini_batch_size = train_micro_batch_size * num_accumulation_steps and
    # global_batch_size = micro * num_accumulation_steps * data_parallel_size.
    # Any one of the three can be left None and is derived.
    train_micro_batch_size=32,
    global_batch_size=None,
    num_accumulation_steps=None,
    # total training iterations (optimizer steps) / epochs; the larger one wins
    train_iter=10000,
    train_epoch=0,
    consumed_train_samples=0,
    consumed_valid_samples=0,
    train_samples=None,
    # fraction of warm-up iterations
    warmup_ratio=0,
    start_iter=0,
    # mixed precision: bf16 parameters + fp32 master weights (NEW: dtype "bf16" | "fp16";
    # fp16 enables the dynamic loss scaler)
    amp=dict(enabled=False, dtype="bf16"),
    # recompute each transformer layer in backward
    activation_checkpoint=dict(enabled=False),
    # NEW: capture forward+backward of every transformer block into CUDA graphs at the first step and replay them
    # (≈800 kernel launches per step become 48 graph launches; data-parallel and fused tensor-parallel layouts, static
    # shapes; anything else silently keeps eager launches)
    cuda_graphs=dict(enabled=True),
    # NEW: forward GEMMs of the linear layers with E4M3 operands (per-tensor dynamic scaling, wgmma e4m3,
    # fp32 accumulation, bf16 outputs); backward GEMMs stay bf16.  Opt-in: see docs/source/tutorials/basics/Kernels.md
    fp8=dict(enabled=False),
    # NEW: SIGTERM → write a resumable checkpoint at the next step boundary and stop (all ranks agree via all-reduce)
    emergency_checkpoint=dict(enabled=False, check_period=1),
    # NEW: profile iterations [start_iter, start_iter + num_iters): NVTX range "train_step" per step (for ncu / nsys
    # --nvtx-include) and a torch.profiler Chrome trace under {output_dir}/profiler/
    profiler=dict(enabled=False, start_iter=10, num_iters=3, torch_profiler=True, nvtx=True),
    # gradient bucket size for data-parallel reduction (names kept from the reference)
    nccl_fusion_threshold_mb=16,
    nccl_fusion_max_ops=24,
    # ZeRO: fp32 master weights + Adam moments partitioned over DP (fused NVLink reduce-scatter/Adam/all-gather);
    # stage 2 additionally partitions the gradients, stage 3 the parameters too (per-block buckets, optim/zero_buckets.py)
    zero_optimization=dict(enabled=False, stage=1),
    checkpointer=dict(period=5000, max_to_keep=100, save_model_after_n_epoch=None),
    test_micro_batch_size=32,
    evaluation=dict(
        enabled=True,
        evaluator=LazyCall(ClsEvaluator)(topk=(1, 5)),
        eval_period=5000,
        eval_after_n_epoch=None,
        eval_iter=1e5,  # running steps for validation/test
        eval_metric="Acc@1",
        eval_mode="max",
    ),
    # path of a checkpoint directory to load weights from (not a resume)
    load_weight="",
    log_period=20,
    # lr scheduler; `max_iter` and `warmup_iter` are injected by the trainer
    scheduler=LazyCall(WarmupCosineLR)(warmup_factor=0.001, alpha=0.01, warmup_method="linear"),
    dist=dict(
        data_parallel_size=1,
        tensor_parallel_size=1,
        pipeline_parallel_size=1,
        # must be set for pipeline parallelism: number of layer indices to spread over stages
        pipeline_num_layers=None,
        # e.g. [0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 3, 3]
        custom_pipeline_stage_id=None,
        # NEW: Megatron-style sequence parallelism inside the TP region with the collectives fused into the GEMM kernels
        # (AG→GEMM / GEMM→RS over NVLink peer memory).  "auto" = on for the models that support token-sharded
        # activations (GPT-2, BERT, Llama family: `supports_sequence_parallel`), off otherwise; True / False force it.
        sequence_parallel="auto",
        fused_tp_comm="auto",
    ),
    # "cuda" | "cpu": where batches are placed by get_batch
    input_placement_device="cuda",
    rdma_enabled=True,
    seed=1234,
)
train = DictConfig(train)
