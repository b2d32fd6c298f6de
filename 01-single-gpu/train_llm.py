"""Chapter 01 — train a causal LM on ONE device.

    python train_llm.py -d synthetic -m openai-community/gpt2            # CPU or GPU plumbing run
    python train_llm.py -d synthetic -m meta-llama/Llama-2-7b-hf -s 4096 -e llama-7b

Same flags, log records and checkpoint files as the reference chapter
(LambdaLabsML/distributed-training-guide ``01-single-gpu/train_llm.py``); the step itself
runs on this repository's sm_90a kernels (see README.md in this directory).
"""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from distributed_training_guide_b200.parallel.strategies import SingleDevice  # noqa: E402
from distributed_training_guide_b200.trainer import run_chapter  # noqa: E402

if __name__ == "__main__":
    run_chapter("01-single-gpu", SingleDevice)
