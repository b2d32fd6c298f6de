"""distributed_training_guide_b200 — a H100-native (sm_90a) distributed causal-LM training
runtime with the capabilities of LambdaLabsML/distributed-training-guide.

Layout:  ``models/`` (Llama / GPT-2), ``ops/`` (autograd wrappers over the hand-written
kernels in ``csrc/``), ``parallel/`` (bootstrap, mesh, NVLink symmetric memory, DDP,
ZeRO-1, FSDP, TP/SP, 2-D, activation checkpointing, offload), ``utils/`` (CLI, logging,
timers, data, checkpointing), ``trainer.py`` (the loop every chapter script shares).
"""
__version__ = "0.1.0"

import os as _os


def _world_size_from_env() -> int:
    for k in ("WORLD_SIZE", "OMPI_COMM_WORLD_SIZE", "SLURM_NTASKS"):
        v = _os.environ.get(k)
        if v and v.isdigit():
            return int(v)
    return 1


# Multi-GPU jobs load every CUDA module at context creation.  The fused collective kernels SPIN on peers' flags;
# with the default lazy loading, the first launch of any kernel (ours or ATen's) may need a context-wide
# synchronisation to load its module — which waits for the spinning kernel, which waits for a peer whose own
# first launch is stuck the same way (the documented lazy-loading hazard for kernels that depend on each other's
# progress).  Round 1's 8-GPU stall in the first backward pass disappeared with eager loading.  Must be set before
# the CUDA context exists, hence at package import; an explicit user setting wins.
if _world_size_from_env() > 1:
    _os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")
