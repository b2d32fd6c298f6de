"""The training loop every chapter script shares.

The reference copy-pastes ~250 lines of identical skeleton into seven scripts (SURVEY.md
§2.1); here each chapter's ``train_llm.py`` picks a *strategy* (``parallel/strategies.py``)
and calls :func:`train`.  Behaviour kept from the reference loop (``01-single-gpu/
train_llm.py:115-189``): epochs x steps, explicit ``next(batches)`` so data time is measured,
replay-and-discard resume, the ``data / forward / backward / update`` timers, the log record
schema (§5.5), checkpoint cadence and layout (§5.4).

Deliberate differences: phases are timed with CUDA events and the running loss is
accumulated on the device, so the host never blocks inside a step (the reference does 8
device syncs + ``loss.item()`` per step); the host only synchronises when a record is
logged.
"""
from __future__ import annotations

import logging

import torch
import torch.distributed as dist

from .models import get_config
from .utils import ckpt as ckpt_utils
from .utils import data as data_utils
from .utils.logging import setup_logging
from .utils.lr import scale_lr
from .utils.mem import get_mem_stats, reset_peak
from .utils.timers import LocalTimer

LOGGER = logging.getLogger("dtg_b200")


def _record(fn):
    """``torch.distributed.elastic``'s @record (exception -> $TORCHELASTIC_ERROR_FILE), the
    reference decorates every distributed ``main()`` with it (``02-...:31``)."""
    try:
        from torch.distributed.elastic.multiprocessing.errors import record

        return record(fn)
    except Exception:  # pragma: no cover
        return fn


def train(args, strategy):
    """Run the chapter.  Returns the final ``state`` dict plus the last log record."""
    data_utils.check_document_masking_args(args)
    env = strategy.setup(args)
    setup_logging(env.rank if strategy.log_rank_prefix else None)
    LOGGER.debug(args)
    LOGGER.debug(f"local_rank={env.local_rank} rank={env.rank} world_size={env.world_size}")
    device = env.device
    torch.manual_seed(args.seed)
    if getattr(args, "deterministic", False):
        torch.use_deterministic_algorithms(True, warn_only=True)

    config = get_config(args.model_name)
    model = strategy.build_model(args, config)
    LOGGER.info(f"Training {strategy.num_parameters(model)} model parameters")
    LOGGER.info(f"Initialized model uses {get_mem_stats(device)['curr_alloc_gb']}gb")

    with strategy.data_guard():
        train_data = data_utils.load_and_preprocess_data(args, config, dp_size=strategy.dp_size)
    LOGGER.debug(f"{len(train_data)} training samples")
    dataloader = data_utils.build_dataloader(
        train_data, args.batch_size, dp_size=strategy.dp_size, dp_rank=strategy.dp_rank, seed=args.seed,
        distributed=env.distributed, deterministic=getattr(args, "deterministic", False),
        num_workers=getattr(args, "num_workers", 1),
    )
    LOGGER.debug(f"{len(dataloader)} batches per epoch")

    lr = scale_lr(args.lr, strategy.dp_size, getattr(args, "lr_scaling", "none"))
    optimizer = strategy.build_optimizer(args, model, lr)
    lr_scheduler = strategy.build_lr_scheduler(args, optimizer, lr)

    is_experiment, exp_dir = ckpt_utils.experiment_dir(args)
    state = ckpt_utils.new_state()
    resumed = False
    if is_experiment and ckpt_utils.can_resume(exp_dir):
        state = strategy.load_checkpoint(exp_dir, model, optimizer, lr_scheduler)
        resumed = True
    if is_experiment:
        LOGGER.info(f"Resumed={resumed} | {state}")
    strategy.barrier()
    if is_experiment:
        strategy.make_experiment_dir(exp_dir)
    strategy.barrier()

    tracker = strategy.build_tracker(args, exp_dir if is_experiment else None, resumed, config)

    timers = {k: LocalTimer(device, name=k) for k in ["data", "forward", "backward", "update"]}
    accum = max(1, getattr(args, "grad_accum_steps", 1))
    running_loss = torch.zeros((), dtype=torch.float32, device=device)
    running_aux = torch.zeros((), dtype=torch.float32, device=device)   # MoE router aux loss (--router-aux-loss-coef)
    if resumed:
        running_loss += float(state["running_loss"])
    max_steps = getattr(args, "max_steps", None)
    last_info = None
    done = False
    seq_length = data_utils.clamp_seq_length(args.seq_length, config)

    for state["epoch"] in range(state["epoch"], args.num_epochs):
        LOGGER.info(f"Begin epoch {state['epoch']} at step {state['epoch_step']}")
        progress = _progress(len(dataloader), disable=env.rank > 0 or not strategy.show_progress)
        if state["epoch_step"] > 0:
            progress.update(state["epoch_step"])
        if hasattr(dataloader.sampler, "set_epoch"):
            dataloader.sampler.set_epoch(state["epoch"])
        batches = iter(dataloader)

        for i_step in range(len(dataloader)):
            with timers["data"], torch.no_grad():
                batch = next(batches)
                if i_step >= state["epoch_step"]:
                    batch = data_utils.to_device(batch, device)
            if i_step < state["epoch_step"]:
                continue  # resume: replay the sampler order, discard the batch (no H2D, no unshard)

            micro = (i_step % accum) + 1
            is_boundary = micro == accum or i_step == len(dataloader) - 1
            strategy.pre_step(model)
            with timers["forward"]:
                batch = strategy.prepare_batch(batch)
                outputs = model(**batch)
                loss = outputs.loss
                if accum > 1:
                    loss = loss / accum
                del batch

            with timers["backward"]:
                with strategy.grad_sync(model, enabled=is_boundary):
                    strategy.backward(model, loss)

            with timers["update"]:
                if is_boundary:
                    optimizer.step()
                    lr_scheduler.step()
                    optimizer.zero_grad(set_to_none=not getattr(args, "cpu_offload", False))

            state["epoch_step"] += 1
            running_loss += outputs.loss.detach().float()
            if getattr(outputs, "aux_loss", None) is not None:
                running_aux += outputs.aux_loss.detach().float()
            progress.update(1)
            if not is_boundary:
                continue
            state["global_step"] += 1

            if state["global_step"] % args.log_freq == 0:
                tok_per_step = strategy.dp_size * args.batch_size * seq_length * accum
                ms_per_step = sum(t.avg_elapsed_ms() for t in timers.values()) * accum
                state["running_loss"] = float(running_loss.item())
                info = {
                    "global_step": state["global_step"],
                    "lr": lr_scheduler.get_last_lr()[0],
                    "running_loss": state["running_loss"] / (args.log_freq * accum),
                    "epoch": state["epoch"],
                    "epoch_progress": state["epoch_step"] / len(dataloader),
                    "num_batches_remaining": len(dataloader) - i_step,
                    **get_mem_stats(device),
                    "tokens_per_s": 1000 * tok_per_step / max(ms_per_step, 1e-9),
                    "time/total": ms_per_step,
                    **{f"time/{k}": t.avg_elapsed_ms() for k, t in timers.items()},
                }
                if getattr(args, "max_grad_norm", None) is not None:
                    info["grad_norm"] = float(optimizer.last_grad_norm)  # pre-clip norm of this step
                if getattr(args, "router_aux_loss_coef", 0.0):
                    info["aux_loss"] = float(running_aux.item()) / (args.log_freq * accum)
                LOGGER.info(info)
                strategy.check_health()
                if tracker is not None:
                    tracker.log(info, step=state["global_step"])
                last_info = info
                reset_peak(device)
                running_loss.zero_()
                running_aux.zero_()
                state["running_loss"] = 0
                for t in timers.values():
                    t.reset()

            if is_experiment and state["global_step"] % args.ckpt_freq == 0:
                state["running_loss"] = float(running_loss.item())
                LOGGER.info("Saving checkpoint.")
                strategy.check_health()
                strategy.save_checkpoint(exp_dir, model, optimizer, lr_scheduler, state)

            if max_steps is not None and state["global_step"] >= max_steps:
                done = True
                break
        if done:
            break
        state["epoch_step"] = 0

    if tracker is not None:
        tracker.finish()
    strategy.teardown()
    if dist.is_available() and dist.is_initialized() and not getattr(args, "keep_process_group", False):
        dist.barrier()
        dist.destroy_process_group()
    return state, last_info


def _progress(n, disable):
    try:
        import tqdm

        return tqdm.tqdm(range(n), disable=disable)
    except Exception:  # pragma: no cover
        class _P:
            def update(self, k):
                pass

        return _P()


def run_chapter(chapter: str, strategy_factory, argv=None, require_experiment=False):
    """Entry point used by the chapter scripts: parse the chapter's flags, train."""
    from .utils.cli import get_parser

    args = get_parser(chapter, require_experiment).parse_args(argv)
    args.chapter = chapter

    @_record
    def main():
        return train(args, strategy_factory(args))

    return main()
