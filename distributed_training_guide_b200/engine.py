"""Public programmatic API: build a parallel training engine and step it.

    from distributed_training_guide_b200.engine import TrainEngine
    eng = TrainEngine.create("meta-llama/Llama-2-7b-hf", parallelism="ddp", batch_size=1, seq_length=4096)
    loss = eng.step(batch)        # batch: dict(input_ids, labels[, attention_mask]) on CPU (pinned) or GPU

The chapter scripts use the same strategies through ``trainer.train``; ``bench.py`` and the
tests drive them through this class.  One process per GPU; launch with ``torchrun`` for N > 1.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Optional

import torch

from .models import get_config
from .utils.lr import scale_lr

PARALLELISMS = ("single", "ddp", "ddp_allreduce", "fsdp", "tp", "2d")


def make_strategy(parallelism: str, args):
    from .parallel import strategies as S

    if parallelism == "single":
        return S.SingleDevice(args)
    if parallelism == "ddp":
        return S.DataParallelZero1(args)
    if parallelism == "ddp_allreduce":  # plain DDP: fused scale + all-reduce buckets, unsharded optimizer
        return S.DataParallelZero1(args, zero1=False)
    if parallelism == "fsdp":
        return S.FullyShardedDataParallel(args)
    if parallelism == "tp":
        return S.TensorParallel(args)
    if parallelism == "2d":
        return S.TwoDParallel(args)
    raise ValueError(f"unknown parallelism {parallelism!r}; expected one of {PARALLELISMS}")


class TrainEngine:
    def __init__(self, strategy, model, optimizer, lr_scheduler, config, args):
        self.strategy, self.model, self.optimizer, self.lr_scheduler = strategy, model, optimizer, lr_scheduler
        self.config, self.args = config, args
        self.env = strategy.env
        self.device = strategy.env.device
        self.steps_done = 0

    @classmethod
    def create(cls, model_name: str, parallelism: str = "auto", batch_size: int = 1, seq_length: int = 1024,
               lr: float = 3e-5, seed: int = 0, device: Optional[str] = None, tensor_parallel: Optional[int] = None,
               cpu_offload: bool = False, checkpoint_activations: bool = False, prefetch_layers: bool = False,
               num_layers: Optional[int] = None, lr_scaling: str = "none", fp8: bool = False,
               document_masking: bool = False, max_grad_norm: Optional[float] = None, **extra):
        """``fp8=True`` runs the decoder-layer projections in fp8 (``ops.linear(..., fp8=True)``); single and ddp
        engines only.
        ``document_masking=True``: batches that carry ``position_ids`` are packed documents, each starting where its
        position id is 0; attention and targets stay inside each document (single, ddp and fsdp engines, Llama).
        ``max_grad_norm``: clip the gradients by their global L2 norm before AdamW
        (``torch.nn.utils.clip_grad_norm_`` semantics; single and ddp engines); see ``grad_norm()``."""
        import os

        world = int(os.environ.get("WORLD_SIZE", "1"))
        if parallelism == "auto":
            parallelism = "ddp" if world > 1 else "single"
        if fp8:
            from .parallel.strategies import check_fp8_supported

            check_fp8_supported(parallelism)
        if document_masking:
            from .parallel.strategies import check_document_masking_supported

            check_document_masking_supported(parallelism)
        if max_grad_norm is not None:
            from .parallel.strategies import check_max_grad_norm_supported

            check_max_grad_norm_supported(parallelism)
            if not max_grad_norm > 0:
                raise ValueError(f"max_grad_norm must be > 0, got {max_grad_norm}")
        args = SimpleNamespace(
            model_name=model_name, batch_size=batch_size, seq_length=seq_length, lr=lr, seed=seed, device=device,
            tensor_parallel=tensor_parallel or world, cpu_offload=cpu_offload,
            checkpoint_activations=checkpoint_activations, prefetch_layers=prefetch_layers, lr_scaling=lr_scaling,
            fp8=fp8, document_masking=document_masking, max_grad_norm=max_grad_norm,
            experiment_name=None, save_dir="../outputs", deterministic=False, local_rank=None, **extra,
        )
        strategy = make_strategy(parallelism, args)
        strategy.setup(args)
        torch.manual_seed(seed)
        config = get_config(model_name, **({"num_hidden_layers": num_layers} if num_layers else {}))
        model = strategy.build_model(args, config)
        lr_eff = scale_lr(lr, strategy.dp_size, lr_scaling)
        optimizer = strategy.build_optimizer(args, model, lr_eff)
        lr_scheduler = strategy.build_lr_scheduler(args, optimizer, lr_eff)
        eng = cls(strategy, model, optimizer, lr_scheduler, config, args)
        eng.parallelism = parallelism
        return eng

    def grad_norm(self) -> Optional[torch.Tensor]:
        """The last step's global gradient L2 norm before clipping, as a device tensor (reading it synchronises);
        None while clipping is off."""
        return getattr(self.optimizer, "last_grad_norm", None)

    @property
    def tokens_per_step(self) -> int:
        return self.strategy.dp_size * self.args.batch_size * self.args.seq_length

    def step(self, batch) -> torch.Tensor:
        """One optimizer step: H2D (non-blocking, if the batch is on the host) -> forward ->
        backward (+ overlapped gradient collectives) -> AdamW -> LR schedule.  Returns the loss
        as a device tensor (reading it is the caller's choice, so the host can run ahead)."""
        s = self.strategy
        dev = self.device
        ev = self._phase_events() if self.phase_timing else None
        src = batch
        batch = {k: (v.to(dev, non_blocking=True) if v.device != dev else v) for k, v in batch.items()}
        if hasattr(src, "copied") and dev.type == "cuda":
            src.copied()  # native loader ring slot: guard it until these async copies have executed
        s.pre_step(self.model)
        batch = s.prepare_batch(batch)
        if ev:
            ev[0].record()
        out = self.model(**batch)
        if ev:
            ev[1].record()
        with s.grad_sync(self.model, enabled=True):
            s.backward(self.model, out.loss)
        if ev:
            ev[2].record()
        self.optimizer.step()
        self.lr_scheduler.step()
        self.optimizer.zero_grad(set_to_none=not self.args.cpu_offload)
        if ev:
            ev[3].record()
            self._phase_log.append(ev)
        self.steps_done += 1
        return out.loss.detach()

    # optional per-phase device timing (CUDA events; resolved lazily by phase_times_ms)
    phase_timing = False

    def _phase_events(self):
        if not hasattr(self, "_phase_log"):
            self._phase_log = []
        return [torch.cuda.Event(enable_timing=True) for _ in range(4)]

    def phase_times_ms(self, last_n=None):
        """Mean forward / backward / update device time of the last ``last_n`` timed steps."""
        log = getattr(self, "_phase_log", [])
        log = log[-last_n:] if last_n else log
        if not log:
            return {}
        torch.cuda.synchronize(self.device)
        f = sum(e[0].elapsed_time(e[1]) for e in log) / len(log)
        b = sum(e[1].elapsed_time(e[2]) for e in log) / len(log)
        u = sum(e[2].elapsed_time(e[3]) for e in log) / len(log)
        return {"forward": f, "backward": b, "update": u}

    def synthetic_batch(self, seed: int = 0, pinned: bool = True):
        """A host batch of random tokens of this engine's (batch_size, seq_length); tensor-parallel
        peers of one data-parallel replica get identical tokens."""
        g = torch.Generator().manual_seed(1000 * seed + self.strategy.dp_rank)
        ids = torch.randint(0, self.config.vocab_size, (self.args.batch_size, self.args.seq_length), generator=g)
        b = {"input_ids": ids, "attention_mask": torch.ones_like(ids), "labels": ids.clone()}
        if pinned and torch.cuda.is_available():
            b = {k: v.pin_memory() for k, v in b.items()}
        return b

    def close(self):
        self.strategy.teardown()
