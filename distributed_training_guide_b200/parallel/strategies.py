"""Per-chapter strategies: how the model is placed, parallelised, stepped and checkpointed.

=====================================  =========================================================
chapter                                strategy
=====================================  =========================================================
01-single-gpu                          :class:`SingleDevice`
02-distributed-data-parallel           :class:`DataParallelZero1`   (DDP + ZeRO-1)
04-fully-sharded-data-parallel         :class:`FullyShardedDataParallel`
05-training-llama-405b                 :class:`FullyShardedDataParallel` (+offload, act-ckpt, prefetch)
06-tensor-parallel                     :class:`TensorParallel` (tp = world, dp = 1 per node)
07-2d-parallel                         :class:`TwoDParallel`   (FSDP x TP)
alternative-frameworks/deepspeed       :class:`ZeroConfigured` (ZeRO stage from a ds_config.json)
=====================================  =========================================================
"""
from __future__ import annotations

import contextlib
import logging
import os
from pathlib import Path

import torch
import torch.distributed as dist

from ..models import build_model
from ..utils import ckpt as ckpt_utils
from ..utils.lr import cosine_schedule
from . import bootstrap
from .flat import build_groups
from .optim import FlatAdamW

LOGGER = logging.getLogger("dtg_b200")


class Strategy:
    chapter = "base"
    log_rank_prefix = True
    show_progress = True

    def __init__(self, args=None):
        self.args = args
        self.env = None
        self.dp_size = 1
        self.dp_rank = 0
        self.groups = None

    # -- process / device -----------------------------------------------------------------
    def setup(self, args):
        dev = getattr(args, "device", None)
        self.env = bootstrap.init_distributed(device_type=dev, local_rank=getattr(args, "local_rank", None))
        self.dp_size, self.dp_rank = self.env.world_size, self.env.rank
        return self.env

    def barrier(self):
        if self.env.distributed:
            dist.barrier()

    def data_guard(self):
        if self.env.distributed:
            return bootstrap.rank0_first()
        return contextlib.nullcontext()

    def teardown(self):
        pass

    def check_health(self):
        """Raise if a device-side NVLink barrier timed out since the last check (called whenever the loop
        synchronises anyway: at every log record and checkpoint)."""
        for name in ("symm", "tp_symm", "dp_symm"):
            sg = getattr(self, name, None)
            if sg is not None:
                sg.check()

    # -- model / optimizer -----------------------------------------------------------------
    def dtype(self):
        return torch.bfloat16

    def build_model(self, args, config):
        raise NotImplementedError

    def num_parameters(self, model):
        return sum(p.numel() for p in model.parameters())

    def build_optimizer(self, args, model, lr):
        return FlatAdamW(self.groups, lr=lr)

    def build_lr_scheduler(self, args, optimizer, lr):
        return cosine_schedule(optimizer, lr)

    def build_tracker(self, args, exp_dir, resumed, config):
        from ..utils.tracking import build_tracker

        return build_tracker(args, self.env, exp_dir, resumed, config)

    # -- step hooks ---------------------------------------------------------------------------
    def pre_step(self, model):
        pass

    def prepare_batch(self, batch):
        return batch

    def grad_sync(self, model, enabled=True):
        return contextlib.nullcontext()

    def backward(self, model, loss):
        loss.backward()

    # -- checkpoints ----------------------------------------------------------------------------
    def make_experiment_dir(self, exp_dir: Path):
        if self.env.rank == 0:
            LOGGER.info("Creating experiment root directory")
            exp_dir.mkdir(parents=True, exist_ok=True)

    def save_checkpoint(self, exp_dir, model, optimizer, lr_scheduler, state):
        ckpt_utils.save_full(exp_dir, model, optimizer, lr_scheduler, state, rank=self.env.rank,
                             world_size=self.env.world_size if self.env.distributed else 1,
                             deterministic=getattr(self.args, "deterministic", False))

    def load_checkpoint(self, exp_dir, model, optimizer, lr_scheduler):
        return ckpt_utils.load_full(exp_dir, model, optimizer, lr_scheduler, self.env.device, rank=self.env.rank,
                                    world_size=self.env.world_size if self.env.distributed else 1,
                                    deterministic=getattr(self.args, "deterministic", False))


class SingleDevice(Strategy):
    """Chapter 01: one device, bf16, flat AdamW (reference ``01-single-gpu/train_llm.py``).
    Runs on CPU too (BASELINE.json config 01: GPT-2 124M plumbing)."""

    chapter = "01-single-gpu"
    log_rank_prefix = False

    def setup(self, args):
        dev = getattr(args, "device", None) or ("cuda" if torch.cuda.is_available() else "cpu")
        device = torch.device("cuda:0" if dev == "cuda" else dev)
        if device.type == "cuda":
            torch.cuda.set_device(device)
        self.env = bootstrap.DistEnv(rank=0, local_rank=0, world_size=1, device=device, distributed=False)
        return self.env

    def build_model(self, args, config):
        model = build_model(config, dtype=self.dtype(), device=self.env.device)
        self.groups, self.symm, self.registry = _flat_groups_on(self, model, 1)
        _load_pretrained(args, model=model)
        _apply_fp8(args, model)
        _apply_document_masking(args, model)
        _apply_router_aux_loss(args, model)
        return model

    def build_optimizer(self, args, model, lr):
        opt = FlatAdamW(self.groups, lr=lr, max_grad_norm=getattr(args, "max_grad_norm", None))
        if self.symm is not None and hasattr(model, "engine"):
            # one rank, same engine: AdamW of each bucket runs inside backward on a side stream as soon
            # as that bucket's gradients are final (the N=1 case of the fused reduce-scatter+AdamW kernel)
            from .ddp import DataParallelEngine

            self.engine = DataParallelEngine(model, self.groups, opt, symm=self.symm, registry=self.registry,
                                             zero1=True, world_size=1, rank=0)
        return opt

    def grad_sync(self, model, enabled=True):
        eng = getattr(self, "engine", None)
        if enabled or eng is None:
            return contextlib.nullcontext()
        return eng.no_sync()


#: engines whose decoder-layer projections can run in fp8 (``--fp8``); the FSDP / TP engines gather their operands
#: inside bf16 GEMM kernels that have no fp8 form
FP8_PARALLELISMS = ("single", "ddp", "ddp_allreduce")


def _apply_fp8(args, model):
    """``model.fp8 = args.fp8`` for the engines that support it (Llama models only)."""
    if not getattr(args, "fp8", False):
        return
    from ..models.llama import LlamaForCausalLM

    if not isinstance(model, LlamaForCausalLM):
        raise ValueError(f"fp8 applies to the Llama models' decoder layers, not {type(model).__name__}")
    if model.config.moe:
        raise ValueError(f"{model.config.name or model.config.arch}: fp8 does not cover the mixture-of-experts "
                         "layers (the grouped expert GEMMs are bf16); train it without --fp8")
    model.fp8 = True


def check_fp8_supported(parallelism: str):
    if parallelism not in FP8_PARALLELISMS:
        raise ValueError(f"fp8 is supported by the {', '.join(FP8_PARALLELISMS)} engines, not {parallelism!r}")


#: engines that run ``LlamaForCausalLM.forward`` and so support ``--document-masking``; the tensor-parallel and 2-D
#: engines run their own layer loop (``tp.model_forward``)
DOCUMENT_MASKING_PARALLELISMS = ("single", "ddp", "ddp_allreduce", "fsdp")


def _apply_document_masking(args, model):
    """``model.document_masking = args.document_masking`` (Llama models only)."""
    if not getattr(args, "document_masking", False):
        return
    from ..models.llama import LlamaForCausalLM

    if not isinstance(model, LlamaForCausalLM):
        raise ValueError(f"document masking applies to the Llama models, not {type(model).__name__}")
    model.document_masking = True


def _apply_router_aux_loss(args, model):
    """``model.router_aux_loss_coef = args.router_aux_loss_coef`` (mixture-of-experts models only)."""
    coef = float(getattr(args, "router_aux_loss_coef", 0.0) or 0.0)
    if coef == 0.0:
        return
    if coef < 0:
        raise ValueError(f"router_aux_loss_coef must be >= 0, got {coef}")
    if not getattr(getattr(model, "config", None), "moe", False):
        raise ValueError("router_aux_loss_coef applies to mixture-of-experts models (OLMoE, Qwen3-MoE)")
    model.router_aux_loss_coef = coef


def check_document_masking_supported(parallelism: str):
    if parallelism not in DOCUMENT_MASKING_PARALLELISMS:
        raise ValueError(f"document masking is supported by the {', '.join(DOCUMENT_MASKING_PARALLELISMS)} engines, "
                         f"not {parallelism!r}")


#: engines that can clip gradients by their global norm (``--max-grad-norm``): the data-parallel bucket engine keeps
#: every reduced gradient until ``optimizer.step()``; FSDP fuses its reduce-scatter with AdamW per layer and keeps no
#: reduced gradient shard, and tensor parallelism would need its replicated norm gains counted once
MAX_GRAD_NORM_PARALLELISMS = ("single", "ddp", "ddp_allreduce")


def check_max_grad_norm_supported(parallelism: str):
    if parallelism not in MAX_GRAD_NORM_PARALLELISMS:
        raise ValueError(f"gradient clipping (max_grad_norm) is supported by the "
                         f"{', '.join(MAX_GRAD_NORM_PARALLELISMS)} engines, not {parallelism!r}")


def _load_pretrained(args, model=None, engine=None, default="never"):
    from ..tools.load_hf import maybe_load_pretrained

    return maybe_load_pretrained(args, model=model, engine=engine, default=default)


def _flat_groups_on(strategy, model, world_size=1, pg=None):
    """Flat param/grad buffers for ``model``: NVLink-symmetric on CUDA, plain tensors on CPU.
    Returns (groups, symm_group_or_None, registry)."""
    from . import symm as symm_mod

    device = strategy.env.device
    if device.type == "cuda":
        sg = symm_mod.SymmGroup(device, pg=pg) if (world_size > 1 or pg is not None) else symm_mod.SymmGroup(device, ranks=[0])
        registry = {}
        # parameters + gradients of every group come out of ONE symmetric chunk (one handle exchange)
        esize = torch.empty((), dtype=strategy.dtype()).element_size()
        n_groups = len(list(model.model.layers)) + 2 if hasattr(model, "model") else 64
        sg.reserve(2 * esize * sum(p.numel() for p in model.parameters())
                   + 2 * n_groups * (8 * world_size * 16 * esize + 2 * sg.ALIGN))
        groups = build_groups(model, device, strategy.dtype(), world_size=world_size, alloc=sg.allocator(registry))
        return groups, sg, registry
    return build_groups(model, device, strategy.dtype(), world_size=world_size), None, {}


class DataParallelZero1(Strategy):
    """Chapter 02: DDP + ZeRO-1 with the bucket collective fused into one NVLink kernel
    (``parallel/ddp.py``).  ``zero1=False`` gives plain DDP (fused scale + all-reduce)."""

    chapter = "02-distributed-data-parallel"

    def __init__(self, args=None, zero1: bool = True):
        super().__init__(args)
        self.zero1 = zero1
        self.engine = None
        self.symm = None

    def build_model(self, args, config):
        env = self.env
        with self.data_guard():
            model = build_model(config, dtype=self.dtype(), device=env.device)
        self.groups, self.symm, self.registry = _flat_groups_on(self, model, env.world_size)
        with self.data_guard():
            _load_pretrained(args, model=model)
        if env.distributed and env.world_size > 1:
            # Replicas must start identical.  torch DDP broadcasts rank 0's parameters in its constructor (13.5 GB for
            # a 7B model, SURVEY.md N1); here the weights are a pure function of (seed, parameter name), so the
            # replicas already agree and a checksum per group is enough — the broadcast is kept as the repair path.
            sums = torch.stack([g.param.float().sum() for g in self.groups])
            ref = sums.clone()
            dist.broadcast(ref, src=0)
            if not torch.equal(sums, ref):
                LOGGER.warning("replica differs from rank 0 after initialisation; broadcasting rank 0's parameters")
            flag = torch.tensor([0.0 if torch.equal(sums, ref) else 1.0], device=sums.device)
            dist.all_reduce(flag)
            if float(flag.item()) > 0:
                for g in self.groups:
                    dist.broadcast(g.param, src=0)
        _apply_fp8(args, model)
        _apply_document_masking(args, model)
        _apply_router_aux_loss(args, model)
        self.model = model
        return model

    def build_optimizer(self, args, model, lr):
        from .ddp import DataParallelEngine

        env = self.env
        shard = (env.rank, env.world_size) if (self.zero1 and env.world_size > 1) else None
        opt = FlatAdamW(self.groups, lr=lr, shard=shard, max_grad_norm=getattr(args, "max_grad_norm", None))
        self.engine = DataParallelEngine(model, self.groups, opt, symm=self.symm, registry=self.registry,
                                         zero1=self.zero1, world_size=env.world_size, rank=env.rank)
        return opt

    def grad_sync(self, model, enabled=True):
        if enabled or self.engine is None:
            return contextlib.nullcontext()
        return self.engine.no_sync()

    def teardown(self):
        if self.symm is not None:
            torch.cuda.synchronize()
            self.symm.check()


class FullyShardedDataParallel(Strategy):
    """Chapters 04 / 05: ZeRO-3 over the data-parallel group with the NVLink copy-engine unshard and the fused
    reduce-scatter + AdamW kernel (``parallel/fsdp.py``); meta-device construction, optional CPU
    offload of the optimizer, activation checkpointing and explicit prefetch flags."""

    chapter = "04-fully-sharded-data-parallel"

    def __init__(self, args=None):
        super().__init__(args)
        self.engine = None
        self.symm = None

    def build_model(self, args, config):
        from . import symm as symm_mod
        from .fsdp import FSDPEngine

        env = self.env
        if getattr(args, "cpu_offload", False):
            # the CPU optimizer is the critical path with offload: give every rank its share of the cores
            # (reference 05-training-llama-405b/train_llm.py:69-72; torchrun defaults OMP_NUM_THREADS to 1)
            ngpu = max(1, torch.cuda.device_count() if torch.cuda.is_available() else 1)
            torch.set_num_threads(max(torch.get_num_threads(), (os.cpu_count() or 1) // ngpu))
        with self.data_guard():
            model = build_model(config, dtype=self.dtype(), device="meta", init=False)
        if env.device.type == "cuda":
            self.symm = symm_mod.SymmGroup(env.device) if env.world_size > 1 else symm_mod.SymmGroup(env.device, ranks=[0])
        self.engine = FSDPEngine(model, env, self.dtype(), symm=self.symm, world_size=env.world_size, rank=env.rank,
                                 seed=getattr(args, "seed", 0), cpu_offload=getattr(args, "cpu_offload", False),
                                 prefetch=True, prefetch_depth=2 if getattr(args, "prefetch_layers", False) else 1)
        model.activation_checkpointing = bool(getattr(args, "checkpoint_activations", False))
        _apply_document_masking(args, model)
        _apply_router_aux_loss(args, model)
        self.groups = self.engine.groups
        self.model = model
        # chapter 05 (reference 05:76-145): rank 0 reads the checkpoint, every rank keeps its slice of each group
        _load_pretrained(args, engine=self.engine,
                         default="auto" if str(getattr(args, "chapter", "")).startswith("05") else "never")
        return model

    def num_parameters(self, model):
        return model.config.num_parameters()

    def grad_sync(self, model, enabled=True):
        if enabled or self.engine is None:
            return contextlib.nullcontext()
        return self.engine.no_sync()

    def build_optimizer(self, args, model, lr):
        return self.engine.build_optimizer(lr)

    def pre_step(self, model):
        self.engine.pre_step()

    def save_checkpoint(self, exp_dir, model, optimizer, lr_scheduler, state):
        env = self.env
        ws = env.world_size if env.distributed else 1
        if env.device.type == "cuda":
            torch.cuda.synchronize()
        ckpt_utils.save_sharded(exp_dir, self.engine.sharded_state(), lr_scheduler, state, env.rank, ws,
                                extra_rank0={"optimizer_steps.json": self.engine.optimizer_steps(),
                                             "layout.json": self.engine.layout_description()})
        self.barrier()

    def load_checkpoint(self, exp_dir, model, optimizer, lr_scheduler):
        env = self.env
        ws = env.world_size if env.distributed else 1
        st = ckpt_utils.load_sharded(exp_dir, self.engine.sharded_state(), lr_scheduler, env.device, env.rank, ws)
        steps = ckpt_utils.load_json_side_file(exp_dir, "optimizer_steps.json")
        if steps is not None:
            self.engine.set_optimizer_steps(steps)
        self.engine.after_load()
        return st

    def make_experiment_dir(self, exp_dir: Path):
        # shared mount: global rank 0 creates it; node-local disk: each node's local rank 0 (reference 04:162-168)
        creator = self.env.rank == 0 if exp_dir.parent.is_mount() or self.env.world_size == 1 else self.env.local_rank == 0
        if creator:
            LOGGER.info("Creating experiment root directory")
            exp_dir.mkdir(parents=True, exist_ok=True)
        self.barrier()
        (exp_dir / f"rank-{self.env.rank}").mkdir(parents=True, exist_ok=True)  # per-rank dir (reference 04:170-172)

    def teardown(self):
        if self.symm is not None:
            torch.cuda.synchronize()
            self.symm.check()


class TwoDParallel(Strategy):
    """Chapters 06 / 07: tensor parallel + sequence parallel inside a contiguous ``tp`` group
    (``parallel/tp.py``: collectives fused into the wgmma GEMMs), and — when the data-parallel
    size is > 1 — FSDP of the TP-local shards over the strided ``dp`` group (``parallel/fsdp.py``),
    i.e. the 2-D mesh of ``07-2d-parallel/train_llm.py:47-53,121-123``.  The sampler is keyed on
    the dp coordinate so TP peers read identical batches (``06-tensor-parallel/train_llm.py:141-147``)."""

    chapter = "07-2d-parallel"

    def __init__(self, args=None, tp_size=None):
        super().__init__(args)
        self.tp_size_arg = tp_size
        self.engine = None
        self.mesh = None
        self.tp_symm = None
        self.dp_symm = None

    def _tp_size(self, args, world):
        t = self.tp_size_arg or getattr(args, "tensor_parallel", None) or world
        return min(int(t), world)

    def setup(self, args):
        from .mesh import build_mesh

        env = super().setup(args)
        self.tp_size = self._tp_size(args, env.world_size)
        self.mesh = build_mesh(env.world_size, env.rank, self.tp_size, create_groups=env.distributed)
        self.dp_size, self.dp_rank = self.mesh.dp_size, self.mesh.dp_rank
        return env

    def build_model(self, args, config):
        from . import symm as symm_mod
        from .fsdp import FSDPEngine
        from .tp import TensorParallelRuntime, TPContext

        env, mesh = self.env, self.mesh
        if getattr(config, "moe", False):
            raise ValueError(
                f"{config.name or config.arch}: tensor parallelism does not support mixture-of-experts layers; train "
                "it with the single-GPU, DDP or FSDP engines (chapters 01, 02, 04, 05)")
        if getattr(config, "full_qk_norm", False):
            # the layer path below is the tensor-parallel one at every tp size, and it has no full-width norm
            raise ValueError(
                f"{config.name or config.arch}: tensor parallelism does not support the full-width q/k norm (OLMo 2): "
                "its statistic spans the q (k) heads that tensor parallelism splits across ranks; train it with the "
                "single-GPU, DDP or FSDP engines (chapters 01, 02, 04, 05)")
        if getattr(config, "parallel_residual", False):
            raise ValueError(
                f"{config.name or config.arch}: tensor parallelism does not support GPT-NeoX's parallel residual: the "
                "tensor-parallel layer path runs attention and MLP one after the other on separate norms of the "
                "updated stream; train it with the single-GPU, DDP or FSDP engines (chapters 01, 02, 04, 05)")
        if getattr(config, "all_bias", False):
            raise ValueError(
                f"{config.name or config.arch}: tensor parallelism does not support biases on the row-parallel "
                "o_proj / c_proj (StarCoder2): they must be added once after the reduction, which the tensor-parallel "
                "layer path does not do; train it with the single-GPU, DDP or FSDP engines (chapters 01, 02, 04, 05)")
        cuda = env.device.type == "cuda"
        seed = getattr(args, "seed", 0)
        use_fsdp = mesh.dp_size > 1
        with self.data_guard():
            model = build_model(config, dtype=self.dtype(), device="meta" if use_fsdp else env.device,
                                tp_size=mesh.tp_size, init=False)
        model.tp_rank = mesh.tp_rank
        if cuda:
            if mesh.tp_size > 1:
                self.tp_symm = symm_mod.SymmGroup(env.device, pg=mesh.tp_group)
            else:
                self.tp_symm = symm_mod.SymmGroup(env.device, ranks=[0])
        max_tokens = args.batch_size * args.seq_length
        ctx = TPContext(mesh.tp_size, mesh.tp_rank, mesh.tp_group, self.tp_symm, env.device, config.hidden_size,
                        max_tokens, config.num_hidden_layers, self.dtype())
        self.tp_ctx = ctx
        if use_fsdp:
            if cuda:
                self.dp_symm = symm_mod.SymmGroup(env.device, pg=mesh.dp_group)
            self.engine = FSDPEngine(model, env, self.dtype(), symm=self.dp_symm, pg=mesh.dp_group,
                                     world_size=mesh.dp_size, rank=mesh.dp_rank, seed=seed,
                                     cpu_offload=getattr(args, "cpu_offload", False),
                                     init_fn=lambda p, n: _tp_init(model, p, n, seed), pre_reduce=self._sync_replicated)
            self.groups = self.engine.groups
        else:
            model.init_weights(seed=seed)
            self.registry = {}
            alloc = self.tp_symm.allocator(self.registry) if cuda else None
            self.groups = build_groups(model, env.device, self.dtype(), world_size=mesh.tp_size, alloc=alloc)
        model.tp = TensorParallelRuntime(ctx)
        model.activation_checkpointing = bool(getattr(args, "checkpoint_activations", False))
        self.model = model
        return model

    def num_parameters(self, model):
        return model.config.num_parameters()

    # replicated parameters (norm gains) see only this rank's sequence shard: sum their grads over tp
    def _norm_regions(self, g):
        out = []
        for n, p, o in zip(g.names, g.params, g.offsets):
            if n.endswith("norm.weight") or n.endswith("layernorm.weight"):
                out.append((o, p.numel()))
        return out

    def _sync_replicated(self, g):
        ctx = self.tp_ctx
        if ctx.t == 1:
            return
        regions = self._norm_regions(g)
        if not regions:
            return
        # adjacent norm gains (input / post-attention layernorm) are reduced with one launch
        merged = [list(regions[0])]
        for off, n in regions[1:]:
            if off == merged[-1][0] + merged[-1][1]:
                merged[-1][1] += n
            else:
                merged.append([off, n])
        for off, n in merged:
            view = g.grad[off:off + n]
            if not ctx.use_kernels:
                ctx.all_reduce_(view)
                continue
            buf = getattr(self, "registry", {}).get(g.grad.data_ptr()) if self.engine is None else None
            if buf is not None and n % (8 * ctx.t) == 0:
                # pure TP: the flat gradient buffer is itself tp-symmetric -> all-reduce (sum) in place
                self.tp_symm.allreduce_scale_(buf, off, n, 1.0, blocks=4)
                continue
            # 2-D: gradient slots are symmetric over the dp group; bounce through a tp-symmetric scratch
            if not hasattr(self, "_norm_scratch"):
                # sized once (the allocation is collective) for the largest run of adjacent norm gains of any group
                biggest = max(sum(m for _, m in self._norm_regions(gg)) for gg in self.groups)
                self._norm_scratch = self.tp_symm.alloc(max(_round_up_to(biggest, 8 * ctx.t), 8 * ctx.t * 16),
                                                        self.dtype())
            sc = self._norm_scratch
            sc.local[:n].copy_(view)
            self.tp_symm.allreduce_scale_(sc, 0, _round_up_to(n, 8 * ctx.t), 1.0, blocks=4)
            view.copy_(sc.local[:n])

    def build_optimizer(self, args, model, lr):
        if self.engine is not None:
            return self.engine.build_optimizer(lr)
        opt = FlatAdamW(self.groups, lr=lr)
        if os.environ.get("DTG_TP_OVERLAP_OPT", "1") != "0":
            from .ddp import LocalOverlapEngine

            # pure TP: per-bucket norm-gradient sync + AdamW inside backward (optimizer.step() just joins)
            self.local_engine = LocalOverlapEngine(model, self.groups, opt, self.env.device,
                                                   pre_update=self._sync_replicated)
        return opt

    local_engine = None

    def grad_sync(self, model, enabled=True):
        self._boundary = enabled  # read by backward() on the engine-less path (DTG_TP_OVERLAP_OPT=0)
        eng = self.engine if self.engine is not None else self.local_engine
        if enabled or eng is None or not hasattr(eng, "no_sync"):
            return contextlib.nullcontext()
        return eng.no_sync()

    _boundary = True

    def pre_step(self, model):
        if self.engine is not None:
            self.engine.pre_step()

    def backward(self, model, loss):
        loss.backward()
        if self.engine is None and self.local_engine is None and self._boundary:
            # pure TP without the in-backward optimizer: sum the replicated (norm-gain) gradients over the tp group
            # once per optimizer step — on the boundary micro-batch, after local accumulation
            for g in self.groups:
                self._sync_replicated(g)

    def save_checkpoint(self, exp_dir, model, optimizer, lr_scheduler, state):
        env = self.env
        ws = env.world_size if env.distributed else 1
        if env.device.type == "cuda":
            torch.cuda.synchronize()
        ckpt_utils.save_sharded(exp_dir, self._sharded_state(optimizer), lr_scheduler, state, env.rank, ws,
                                extra_rank0={"optimizer_steps.json": self._optimizer_steps(optimizer)})
        self.barrier()

    def load_checkpoint(self, exp_dir, model, optimizer, lr_scheduler):
        env = self.env
        ws = env.world_size if env.distributed else 1
        st = ckpt_utils.load_sharded(exp_dir, self._sharded_state(optimizer), lr_scheduler, env.device, env.rank, ws)
        steps = ckpt_utils.load_json_side_file(exp_dir, "optimizer_steps.json")
        if steps is not None:  # AdamW bias correction continues where it stopped (moments alone are not enough)
            if self.engine is not None:
                self.engine.set_optimizer_steps(steps)
            else:
                for g in self.groups:
                    optimizer.state[g.param]["step"] = int(steps.get(g.name, 0))
        if self.engine is not None:
            self.engine.after_load()
        return st

    def _optimizer_steps(self, optimizer):
        if self.engine is not None:
            return self.engine.optimizer_steps()
        return {g.name: int(optimizer.state[g.param]["step"]) for g in self.groups}

    def _sharded_state(self, optimizer):
        if self.engine is not None:
            return self.engine.sharded_state()
        model_sd = {g.name: g.param for g in self.groups}
        opt_sd = {}
        for g in self.groups:
            st = optimizer.state[g.param]
            opt_sd[f"{g.name}.exp_avg"], opt_sd[f"{g.name}.exp_avg_sq"] = st["exp_avg"], st["exp_avg_sq"]
        return {"model": model_sd, "optimizer": opt_sd}

    def teardown(self):
        for sg in (self.tp_symm, self.dp_symm):
            if sg is not None:
                torch.cuda.synchronize()
                sg.check()


def _round_up_to(x, m):
    return (x + m - 1) // m * m


def _tp_init(model, p, name, seed):
    from ..models.llama import init_parameter_, tp_shard_spec

    init_parameter_(p, name, seed, **tp_shard_spec(name, p, model.tp_size, model.tp_rank))


class TensorParallel(TwoDParallel):
    """Chapter 06: tensor parallel over all GPUs of the node (``tp = gpus on node``), data parallel
    across nodes — the mesh of ``06-tensor-parallel/train_llm.py:37-55``.  (Unlike the reference, the
    data-parallel replicas ARE kept in sync: with dp > 1 this is the 2-D engine, SURVEY.md §8 #7.)"""

    chapter = "06-tensor-parallel"

    def _tp_size(self, args, world):
        if self.tp_size_arg:
            return min(self.tp_size_arg, world)
        import os

        local = int(os.environ.get("LOCAL_WORLD_SIZE", "0")) or (torch.cuda.device_count() if torch.cuda.is_available() else world)
        return max(1, min(local, world))
