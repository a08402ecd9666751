"""libai_b200 — a Hopper (sm_90a) native large-model training toolbox.

Same user-facing surface as LiBai (LazyConfig configs, DefaultTrainer, parallel layers, model
zoo) on PyTorch + hand-written CUDA kernels + NCCL/NVLink.
"""
__version__ = "0.1.0"
