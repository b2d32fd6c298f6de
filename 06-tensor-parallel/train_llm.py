"""Chapter 06 — tensor parallel + sequence parallel across the GPUs of a node.

    torchrun --standalone --nproc-per-node gpu train_llm.py -d synthetic -m meta-llama/Llama-3.1-8B -b 16 -s 1024

Column-parallel q/k/v/gate/up and row-parallel o/down projections run as single wgmma kernels that
fetch / scatter their sequence-sharded operand over NVLink (all-gather->GEMM, GEMM->reduce-scatter);
the loss is vocab-parallel (parallel/tp.py).  Flags follow the reference chapter."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from distributed_training_guide_b200.parallel import strategies  # noqa: E402
from distributed_training_guide_b200.trainer import run_chapter  # noqa: E402

if __name__ == "__main__":
    run_chapter("06-tensor-parallel", lambda args: strategies.TensorParallel(args))
