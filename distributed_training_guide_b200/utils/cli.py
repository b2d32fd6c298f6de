"""Command-line surface of the chapter scripts.

One builder covers the whole flag matrix of the reference (SURVEY.md §2.6; reference
parsers at ``01-single-gpu/train_llm.py:289-303``, ``04-...:370-385``, ``05-...:455-472``,
``07-2d-parallel/train_llm.py:388-403``, deepspeed ``train_llm.py:309-322``): every chapter
gets the common flags and opts into its extras by name.
"""
from __future__ import annotations

import argparse

COMMON = ("experiment-name", "dataset-name", "dataset-subset", "model-name", "save-dir", "seed",
          "num-epochs", "lr", "batch-size", "log-freq", "ckpt-freq", "seq-length")

CHAPTER_EXTRAS = {
    "01-single-gpu": ("fp8", "document-masking", "max-grad-norm"),
    "02-distributed-data-parallel": ("fp8", "document-masking", "max-grad-norm"),
    "04-fully-sharded-data-parallel": ("cpu-offload", "document-masking"),
    "05-training-llama-405b": ("cpu-offload", "checkpoint-activations", "prefetch-layers", "document-masking"),
    "06-tensor-parallel": (),
    "07-2d-parallel": ("tensor-parallel",),
    "deepspeed": ("local_rank", "zero_config"),
}


def positive_float(text: str) -> float:
    v = float(text)
    if not v > 0:
        raise argparse.ArgumentTypeError(f"must be > 0, got {text}")
    return v


def get_parser(chapter: str = "01-single-gpu", require_experiment: bool = False) -> argparse.ArgumentParser:
    extras = CHAPTER_EXTRAS[chapter]
    p = argparse.ArgumentParser(description=f"{chapter}: causal-LM training on H100")
    p.add_argument("-e", "--experiment-name", default=None, required=require_experiment,
                   help="enables checkpointing/resume under <save-dir>/<experiment-name>")
    p.add_argument("-d", "--dataset-name", default=None, required=True,
                   help="'synthetic', a local .bin/.txt/.jsonl path, or a Hugging Face dataset id")
    p.add_argument("--dataset-subset", default=None)
    p.add_argument("-m", "--model-name", default=None, required=True,
                   help="embedded config id (e.g. meta-llama/Llama-2-7b-hf) or a directory with config.json")
    p.add_argument("--save-dir", default="../outputs")
    p.add_argument("--seed", default=0, type=int)
    p.add_argument("--num-epochs", default=100, type=int)
    p.add_argument("--lr", default=3e-5, type=float)
    p.add_argument("-b", "--batch-size", default=1, type=int)
    p.add_argument("--log-freq", default=10, type=int)
    p.add_argument("--ckpt-freq", default=500, type=int)
    p.add_argument("-s", "--seq-length", default=1024, type=int)
    # additions of this framework (absent from the reference; all default to its behaviour)
    p.add_argument("--max-steps", default=None, type=int, help="stop after this many optimizer steps")
    p.add_argument("--num-samples", default=None, type=int, help="size of the synthetic dataset")
    p.add_argument("--grad-accum-steps", default=1, type=int,
                   help="micro-batches per optimizer step (reference: related-topics/gradient-accumulation)")
    p.add_argument("--deterministic", action="store_true",
                   help="seeded loaders + rng.pt in checkpoints (reference: related-topics/determinism)")
    p.add_argument("--lr-scaling", choices=("none", "linear", "sqrt"), default="none",
                   help="scale --lr by the data-parallel size (reference: related-topics/effective-batch-size-and-lr)")
    p.add_argument("--wandb", choices=("off", "rank0", "local-rank0", "all"), default="off",
                   help="reference: related-topics/wandb-configurations")
    p.add_argument("--device", default=None, help="cuda (default when available) or cpu")
    p.add_argument("--num-workers", default=1, type=int, help="DataLoader worker processes (reference: 1)")
    p.add_argument("--pretrained", choices=("auto", "require", "never"), default=None,
                   help="load local Hugging Face safetensors for --model-name (chapter 05 defaults to auto: load "
                        "them when they exist on disk; other chapters default to never = random init)")
    p.add_argument("--router-aux-loss-coef", default=0.0, type=float,
                   help="mixture-of-experts models (OLMoE, Qwen3-MoE): add this times the Switch load-balancing loss of every "
                        "layer's router to the loss (transformers' load_balancing_loss_func); the log record then "
                        "carries aux_loss (default: 0, off)")
    if "fp8" in extras:
        p.add_argument("--fp8", default=False, action="store_true",
                       help="run the decoder-layer projections (q|k|v, o, gate|up, down) as fp8 GEMMs with per-tensor "
                            "current scaling: x and W in e4m3, output gradients in e5m2")
    if "document-masking" in extras:
        p.add_argument("--document-masking", default=False, action="store_true",
                       help="packed documents: every sample carries position_ids that restart at 0 at each document, "
                            "attention stays inside each document and no token is trained to predict the next "
                            "document's first token (Llama models)")
        p.add_argument("--eos-token-id", default=None, type=int,
                       help="with --document-masking and a .bin dataset: a document starts after each occurrence of "
                            "this token id")
    if "max-grad-norm" in extras:
        p.add_argument("--max-grad-norm", default=None, type=positive_float,
                       help="clip the gradients by their global L2 norm before AdamW, as "
                            "torch.nn.utils.clip_grad_norm_(params, max_norm) does; the log record then carries the "
                            "pre-clip grad_norm (default: off)")
    if "cpu-offload" in extras:
        p.add_argument("--cpu-offload", default=False, action="store_true")
    if "checkpoint-activations" in extras:
        p.add_argument("--checkpoint-activations", default=False, action="store_true")
    if "prefetch-layers" in extras:
        p.add_argument("--prefetch-layers", default=False, action="store_true")
    if "tensor-parallel" in extras:
        p.add_argument("-tp", "--tensor-parallel", default=8, type=int)
    if "local_rank" in extras:
        p.add_argument("--local_rank", type=int, default=None)
    if "zero_config" in extras:
        p.add_argument("--deepspeed_config", default=None, help="DeepSpeed-style JSON (ds_config.json)")
        p.add_argument("--deepspeed", action="store_true", help="accepted for launcher compatibility")
    return p
