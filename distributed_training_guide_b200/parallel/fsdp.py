"""Fully-sharded data parallelism (ZeRO-3) on NVLink symmetric memory (chapters 04 / 05).

Reference: ``fully_shard(layer, reshard_after_forward=True, mp_policy=MixedPrecisionPolicy(bf16,
reduce fp32), offload_policy=CPUOffloadPolicy())`` per decoder layer + root group
(``04-fully-sharded-data-parallel/train_llm.py:83-90``, ``05-training-llama-405b/train_llm.py:100-106``),
meta-device construction (``04:76-95``), ``model.unshard()`` prefetch of the root group (``04:187-188``),
explicit forward/backward prefetch (``05:148-161``).  torch FSDP2 runs, per group, copy-in ->
``all_gather_into_tensor`` -> copy-out in forward and again in backward, then chunk_cat(+fp32 cast) ->
``reduce_scatter_tensor`` -> cast, then a separate fused AdamW over DTensor shards (SURVEY.md N4/N5/K12).

Here each group (embedding, every decoder layer, head) is one flat parameter:
  * the 1/N shard of every rank lives in a symmetric buffer; UNSHARD = a one-warp device barrier plus N
    peer-to-peer copies on the copy engines (``comm.cu: comm_allgather_ce``; the SM pull kernel
    ``allgather_kernel`` is kept behind ``DTG_FSDP_AG=sm``) straight into a rotating "full" slot the layer's
    parameter views point at — no copy-in/copy-out and no SM time — prefetched one or two layers ahead on a
    side stream;
  * gradients are written by the wgrad GEMMs into a rotating symmetric "grad" slot; when the
    layer's backward boundary fires, ONE kernel reduce-scatters the slot (pull + fp32 sum),
    applies AdamW to this rank's shard of parameters and optimizer state, and leaves the updated
    shard in place for the next unshard (``rs_adamw_kernel<PUSH_PARAMS=false>``) — the optimizer step
    is hidden inside backward and there is no separate reduce_scatter / cast / step;
  * reshard-after-forward is implicit: 3 full slots rotate across layers (2 for gradients).

``--cpu-offload`` keeps optimizer state (+ an fp32-free master shard) in pinned host memory: the
kernel is then a plain reduce-scatter, the shard gradient goes D2H, AdamW runs on the CPU and the
updated shard returns H2D before the next unshard (plumbing flag, like the reference's).
On CPU (gloo tests) the same schedule runs with ``torch.distributed`` collectives.
"""
from __future__ import annotations

import contextlib
import os
from typing import Dict, List, Optional

import torch
import torch.distributed as dist
from torch.autograd import Variable

from ..models.llama import LlamaDecoderLayer, LlamaForCausalLM, init_parameter_
from ..ops import reference as ref
from ..ops import join_wgrad_stream
from ..utils.timers import nvtx_range
from .ddp import boundary
from .flat import ALIGN, FlatGroup, _round_up, install_fused_views
from .optim import FlatAdamW


class ShardGroup:
    """What the optimizer sees of a group: this rank's parameter shard."""

    def __init__(self, name, shard_param, per, flat: FlatGroup):
        self.name, self.param, self.padded_numel, self.flat = name, shard_param, per, flat
        self.grad = None

    def zero_grad(self):
        self.flat.zero_grad_counters()

    def shard_range(self, rank, world):
        return 0, self.padded_numel


def _zero_counters(self):
    for p in self.params:
        p._dtg_writes = 0
    for f in self.fused.values():
        f._dtg_writes = 0


FlatGroup.zero_grad_counters = _zero_counters


class _GatherSpec:
    """Handle on a weight matrix of an FSDP group for ``ops._Linear``: where it sits in the group's flat buffer."""

    def __init__(self, eng, g, off, numel, rows, cols):
        self.eng, self.g, self.off, self.numel, self.rows, self.cols = eng, g, off, numel, rows, cols

    def pending(self) -> bool:
        return self.eng.gather_pending(self)

    def gemm(self, a, b_kmajor: bool, bias=None):
        """a @ W^T (+ bias) (``b_kmajor``: forward) or a @ W (dgrad) with W gathered from the ranks' shards by the GEMM
        itself.  The bias is a 1-D parameter of the group's prefetched tail, already local."""
        return self.eng._gather_gemm(self, a, b_kmajor, bias)


class FSDPEngine:
    N_FULL_SLOTS = 3
    N_GRAD_SLOTS = 2

    def __init__(self, model, env, dtype, symm=None, pg=None, world_size=1, rank=0, seed=0, cpu_offload=False,
                 prefetch=True, lr=3e-5, init_fn=None, pre_reduce=None, prefetch_depth=None):
        self.model, self.env, self.dtype = model, env, dtype
        self.symm, self.pg, self.world, self.rank = symm, pg, world_size, rank
        self.device = env.device
        self.use_kernels = symm is not None
        self.cpu_offload = cpu_offload
        self.prefetch = prefetch
        self._prefetch_depth_req = int(os.environ.get("DTG_FSDP_PREFETCH", prefetch_depth or 1))
        self.sync_enabled = True
        self.pre_reduce = pre_reduce  # 2-D: sum the replicated (norm) gradients over the tp group first
        core = model.model
        self.layers = list(core.layers)
        L = len(self.layers)
        # Llama: gradients are written by the wgrad kernels (direct write, fused q|k|v / gate|up views).  Anything else
        # (GPT-2: the reference's smoke model) gets its gradients from autograd, which ACCUMULATES into p.grad — those
        # buffers are cleared before use — and may tie lm_head to the embedding, which then stays gathered all step.
        self.is_llama = isinstance(model, LlamaForCausalLM)
        self.direct_write = self.use_kernels and self.is_llama
        self.tied = bool(getattr(model.config, "tie_word_embeddings", False))
        assert self.is_llama or init_fn is None, "tensor-parallel slices are implemented for the Llama family"
        esize = torch.empty((), dtype=dtype).element_size()
        # Unshard fused into the consuming GEMMs (csrc/gemm_wgmma.cu, B_MODE 3): the big matrices of a group are
        # gathered by the GEMM kernel that reads them; only the small tail (norm gains) keeps a prefetched copy.
        # Needs every matrix to start and end on a chunk boundary of the flat layout and every shard to be a whole
        # number of chunks.  Selected with DTG_FSDP_GATHER=gemm; the DEFAULT is the copy-engine unshard of whole groups
        # ("ce"): one 16 KB x 2 bounce ring per CTA does not keep enough NVLink bytes in flight to feed a GEMM that consumes
        # 7/8 remote weights, while the copy engines prefetch a whole layer ahead for free.
        self.fused_gather = (self.use_kernels and self.is_llama and world_size > 1 and esize == 2 and init_fn is None
                             and os.environ.get("DTG_FSDP_GATHER", "ce") == "gemm")

        def pick_chunk(named):
            """largest power-of-two chunk (16 KB .. 512 KB) that tiles every matrix of the group; 0 = not eligible"""
            mats = [p.numel() * esize for _, p in named if p.dim() == 2]
            seen_small = False
            for _, p in named:              # matrices first, small tensors last (so matrix offsets stay aligned)
                if p.dim() == 2 and seen_small:
                    return 0
                seen_small = seen_small or p.dim() != 2
            c = 512 << 10
            while mats and c >= (16 << 10):
                if all(m % c == 0 for m in mats):
                    return c
                c >>= 1
            return 0

        def pad_of(named):
            c = pick_chunk(named) if self.fused_gather else 0
            base = ALIGN * world_size * 16
            return max(base, world_size * c // esize) if c else base

        def layout(named):
            off = 0
            for _, p in named:
                off = _round_up(off + p.numel(), ALIGN)
            pad = pad_of(named)
            return _round_up(max(off, pad), pad)

        layer_named = []
        if self.is_llama:
            for i, layer in enumerate(self.layers):
                named = dict(layer.named_parameters())
                assert set(named) == set(layer.flat_order), f"layer {i}: parameters outside flat_order"
                layer_named.append([(f"model.layers.{i}.{n}", named[n]) for n in layer.flat_order])
            embed_named = [("model.embed_tokens.weight", core.embed_tokens.weight)]
            head_named = [("model.norm.weight", core.norm.weight)]
            if not self.tied:  # a tied lm_head IS the embedding parameter (it lives in the embed group)
                head_named.insert(0, ("lm_head.weight", model.lm_head.weight))  # matrix first: chunk-aligned
            default_init = lambda p, n: init_parameter_(p, n, seed)  # noqa: E731
        else:
            from ..models.gpt2 import init_parameter_ as gpt2_init

            for i, layer in enumerate(self.layers):
                layer_named.append([(f"transformer.h.{i}.{n}", p) for n, p in layer.named_parameters()])
            embed_named = [("transformer.wte.weight", core.wte.weight), ("transformer.wpe.weight", core.wpe.weight)]
            head_named = [(f"transformer.ln_f.{n}", p) for n, p in core.ln_f.named_parameters()]
            assert self.tied and model.lm_head.weight is core.wte.weight, "GPT-2 layout expects a tied lm_head"
            default_init = lambda p, n: gpt2_init(p, n, seed, L)  # noqa: E731
        max_layer = max(layout(n) for n in layer_named) if layer_named else ALIGN * world_size * 16

        def local(n):
            return torch.zeros(n, dtype=dtype, device=self.device)

        def symmetric(n):
            if self.use_kernels:
                b = symm.alloc(n, dtype)
                self._symm_of[b.local.data_ptr()] = b
                return b.local
            return local(n)

        self._symm_of: Dict[int, object] = {}
        self.full_slots = [local(max_layer) for _ in range(min(self.N_FULL_SLOTS, max(L, 1)))]
        self.grad_slots = [symmetric(max_layer) for _ in range(min(self.N_GRAD_SLOTS, max(L, 1)))]
        self.prefetch_depth = max(1, min(self._prefetch_depth_req, len(self.full_slots) - 1))
        self.groups: List[FlatGroup] = []
        self.shards: List[ShardGroup] = []
        self.slot_of: Dict[str, int] = {}
        self.gslot_of: Dict[str, int] = {}

        def make_group(name, named, full_buf, grad_buf):
            bufs = [full_buf, grad_buf]
            n_pad = layout(named)

            def alloc(n, dt):
                return bufs.pop(0)[:n]

            g = FlatGroup(name, named, self.device, dtype, pad_multiple=pad_of(named), alloc=alloc, with_grad=True,
                          direct_write=self.direct_write)
            assert g.padded_numel == n_pad
            g.chunk_bytes = pick_chunk(named) if (self.fused_gather and name != "embed") else 0
            # deterministic init of the whole group inside the slot, then keep only my shard
            for n, p in named:
                if init_fn is not None:
                    init_fn(p, n)  # tensor-parallel slices
                else:
                    default_init(p, n)
            per = g.padded_numel // world_size
            sh = symmetric(per)
            sh.copy_(g.param[rank * per:(rank + 1) * per])
            self.groups.append(g)
            self.shards.append(ShardGroup(name, sh, per, g))
            return g

        self.embed = make_group("embed", embed_named, local(layout(embed_named)), symmetric(layout(embed_named)))
        for i, named in enumerate(layer_named):
            fs, gs = i % len(self.full_slots), i % len(self.grad_slots)
            g = make_group(f"layer{i}", named, self.full_slots[fs], self.grad_slots[gs])
            self.slot_of[g.name], self.gslot_of[g.name] = fs, gs
            layer = self.layers[i]
            layer._flat_group = g
            if not self.is_llama:
                continue
            install_fused_views(layer, g, i)
        self.head = make_group("head", head_named, local(layout(head_named)), symmetric(layout(head_named)))
        self.layer_groups = self.groups[1:1 + L]
        self.shard_of = {s.name: s for s in self.shards}
        if self.fused_gather:
            self._install_gather_specs(model)
        model._flat_groups = self.groups
        model.engine = self

        # bookkeeping for the schedule
        self.slot_owner = [None] * len(self.full_slots)   # which group's parameters a full slot holds
        self._unsharded = set()
        if self.use_kernels:
            self.comm_stream = torch.cuda.Stream(device=self.device)
            # unshard on the copy engines (DTG_FSDP_AG=sm selects the SM pull kernel instead)
            self.ag_copy_engine = os.environ.get("DTG_FSDP_AG", "ce") != "sm"
            self.ag_done: Dict[str, torch.cuda.Event] = {}
            self.slot_free = [None] * len(self.full_slots)
            self.rs_done: Dict[str, torch.cuda.Event] = {}
            self._done = torch.cuda.Event()
        self._in_backward = False
        self._tails = []
        self.optimizer: Optional[FlatAdamW] = None
        # DTG_COMM_TRACE=1: CUDA events around every gather / reduce kernel and around every point where the
        # compute stream waits for the communication stream (see comm_trace_summary)
        self.trace = [] if (self.use_kernels and os.environ.get("DTG_COMM_TRACE")) else None
        # after the constructor every slot holds the LAST group that was initialised in it
        for i, g in enumerate(self.layer_groups):
            self.slot_owner[self.slot_of[g.name]] = None
        if self.use_kernels:
            torch.cuda.synchronize(self.device)
        if world_size > 1 and dist.is_initialized():
            dist.barrier(group=pg)

    # -- unshard fused into the consuming GEMMs ------------------------------------------------------------
    def _install_gather_specs(self, model):
        """Give every matrix that a linear op reads (fused q|k|v and gate|up, o_proj, down_proj, lm_head) a
        ``_dtg_gather`` handle: ``ops._Linear`` then runs the GEMM that also gathers the weight from the ranks'
        shards (first use after the group became live) or the plain GEMM (already gathered).

        Reference: FSDP2's per-layer all-gather in front of the layer's first matmul and again in backward
        (``fully_shard(layer, reshard_after_forward=True)``, ``04-fully-sharded-data-parallel/train_llm.py:83-90``) and
        the root ``model.unshard()`` prefetch (``04:187-188``): there three NCCL-side kernels per gather (copy-in,
        all_gather_into_tensor, copy-out), here none — the bytes move inside the consuming wgmma GEMM."""
        self.gather_pads = self.symm.new_pad_set()   # these kernels run on the compute stream: own pad + epochs
        self._counters, self._ngather = {}, {}
        esize = 2

        def counters_for(full):
            key = full.data_ptr()
            if key not in self._counters:
                self._counters[key] = torch.zeros(max(64, full.numel() * esize // (16 << 10) + 1), dtype=torch.int32,
                                                  device=self.device)
            return self._counters[key]

        def spec(g, holder, off, numel, rows, cols):
            holder._dtg_gather = _GatherSpec(self, g, off, numel, rows, cols)

        for g in self.groups:
            g._gathered, g._full_now = set(), False
            if not g.chunk_bytes:
                g.tail = None
                continue
            counters_for(g.param)
            by_name = dict(zip(g.names, zip(g.params, g.offsets, g.shapes)))
            covered = set()
            for fname, fw in g.fused.items():
                if fw.data.dim() != 2:   # the fused q|k|v bias (Qwen2): 1-D, it lives in the prefetched tail
                    continue
                members = [n for n in g.names if any(n.endswith(m) for m in LlamaDecoderLayer.FUSED[fname])]
                off = by_name[members[0]][1]
                rows = sum(by_name[n][2][0] for n in members)
                cols = by_name[members[0]][2][1]
                spec(g, fw, off, rows * cols, rows, cols)
                covered.update(members)
            end_of_matrices = 0
            for n, (p, off, shape) in by_name.items():
                if len(shape) != 2:
                    continue
                end_of_matrices = max(end_of_matrices, off + shape[0] * shape[1])
                if n not in covered:
                    spec(g, p, off, shape[0] * shape[1], shape[0], shape[1])
            # what is left after the matrices (norm gains): a prefetched copy-engine gather of that flat range
            g.tail = (end_of_matrices, g.numel) if g.numel > end_of_matrices else None

    def _gather_gemm(self, sp, a, b_kmajor, bias=None):
        g = sp.g
        C = self.symm.C
        full = g.param
        sh = self.shard_of[g.name]
        M = a.shape[0]
        out = torch.empty(M, sp.rows if b_kmajor else sp.cols, dtype=a.dtype, device=a.device)
        key = (full.data_ptr(), sp.off)
        n = self._ngather.get(key, 0) + 1
        self._ngather[key] = n
        shift = g.chunk_bytes.bit_length() - 1
        ppc = g.chunk_bytes // (16 << 10)
        with nvtx_range(f"gather_gemm:{g.name}"):
            C.gemm_bgather(a, full, out, b_kmajor, sp.rows, sp.cols, self._symm_of[sh.param.data_ptr()].ptrs,
                           sh.padded_numel, sp.off, sp.numel, self._counters[full.data_ptr()], n * ppc, shift,
                           self.gather_pads.ptrs, self.rank, 0, bias)   # epoch 0: no entry barrier (see the kernel)
        g._gathered.add(sp.off)
        return out

    # -- optimizer ---------------------------------------------------------------------------------
    def build_optimizer(self, lr):
        state_device = torch.device("cpu") if self.cpu_offload else None
        opt = FlatAdamW(self.shards, lr=lr, state_device=state_device)
        if self.cpu_offload:
            for s in self.shards:
                st = opt.state[s.param]
                st["exp_avg"] = st["exp_avg"].pin_memory() if torch.cuda.is_available() else st["exp_avg"]
                st["exp_avg_sq"] = st["exp_avg_sq"].pin_memory() if torch.cuda.is_available() else st["exp_avg_sq"]
                st["cpu_param"] = s.param.detach().to("cpu").clone()
                st["cpu_grad"] = torch.zeros_like(st["cpu_param"])
                if torch.cuda.is_available():
                    st["cpu_param"], st["cpu_grad"] = st["cpu_param"].pin_memory(), st["cpu_grad"].pin_memory()
                st["gpu_grad"] = torch.zeros_like(s.param)
        opt.external_step = self._optimizer_step
        self.optimizer = opt
        return opt

    # -- unshard / reshard ---------------------------------------------------------------------------
    def _is_live(self, g: FlatGroup) -> bool:
        if g.name in ("embed", "head"):
            return g.name in self._unsharded
        return self.slot_owner[self.slot_of[g.name]] == g.name

    def unshard(self, g: FlatGroup, force_full: bool = False):
        """Make ``g``'s parameters available in its full buffer.  Copy-engine path: the whole group is gathered now
        (asynchronously on the comm stream).  Fused path (``g.chunk_bytes``): only the small tail is copied now; every
        matrix is gathered by the first GEMM that reads it (``_gather_gemm``)."""
        if self._is_live(g):
            if force_full and self.use_kernels and getattr(g, "chunk_bytes", 0) and not g._full_now:
                self._set_dead(g)
            else:
                return
        sh = self.shard_of[g.name]
        if g.name in ("embed", "head"):
            self._unsharded.add(g.name)
        else:
            self.slot_owner[self.slot_of[g.name]] = g.name
        if not self.use_kernels:
            if self.world > 1:
                parts = [torch.empty_like(sh.param) for _ in range(self.world)]
                dist.all_gather(parts, sh.param, group=self.pg)
                g.param.copy_(torch.cat(parts))
            else:
                g.param.copy_(sh.param)
            return
        lazy = bool(getattr(g, "chunk_bytes", 0)) and not force_full
        g._gathered = set()
        g._full_now = not lazy
        with torch.cuda.stream(self.comm_stream):
            if g.name not in ("embed", "head"):
                ev = self.slot_free[self.slot_of[g.name]]
                if ev is not None:
                    self.comm_stream.wait_event(ev)  # the slot's previous layer has finished computing
            t0 = self._trace_begin()
            with nvtx_range(f"unshard:{g.name}"):
                if lazy:
                    # what the GEMMs do not fetch themselves: my own slice (a local copy) and the small tail
                    per = sh.padded_numel
                    # (raw copies, not tensor ops: an in-place torch op on the slot would bump the autograd version
                    # of every weight view another layer saved for its backward)
                    self.symm.gather_range_(self._symm_of[sh.param.data_ptr()], g.param, self.rank * per,
                                            (self.rank + 1) * per, per, barrier=False)
                    # the device barrier in front of the tail copies is also what orders every later read of the
                    # peers' shards (by the gather warps of this group's GEMMs, which wait for `ag_done`) behind
                    # the peers' previous optimizer work on their communication streams
                    if g.tail is not None:
                        self.symm.gather_range_(self._symm_of[sh.param.data_ptr()], g.param, g.tail[0], g.tail[1],
                                                sh.padded_numel)
                    else:
                        self.symm.barrier_()
                else:
                    if getattr(g, "chunk_bytes", 0):
                        g._gathered = {"all"}
                    self.symm.allgather_(self._symm_of[sh.param.data_ptr()], g.param, 0, sh.padded_numel,
                                         copy_engine=self.ag_copy_engine)
            self._trace_end("unshard", t0)
            ev = torch.cuda.Event()
            ev.record(self.comm_stream)
            self.ag_done[g.name] = ev

    def _set_dead(self, g):
        if g.name in ("embed", "head"):
            self._unsharded.discard(g.name)
        else:
            self.slot_owner[self.slot_of[g.name]] = None

    def gather_pending(self, sp) -> bool:
        g = sp.g
        return bool(g.chunk_bytes) and self._is_live(g) and "all" not in g._gathered and sp.off not in g._gathered

    def wait_unsharded(self, g: FlatGroup, force_full: bool = False):
        self.unshard(g, force_full)
        if self.use_kernels:
            t0 = self._trace_begin()
            torch.cuda.current_stream().wait_event(self.ag_done[g.name])
            self._trace_end("stall_unshard_bwd" if self._in_backward else "stall_unshard_fwd", t0)

    def release(self, g: FlatGroup):
        """The compute stream is done with ``g``'s full parameters (its slot may be overwritten)."""
        if g.name in ("embed", "head"):
            self._unsharded.discard(g.name)
            return
        if self.use_kernels:
            ev = torch.cuda.Event()
            ev.record()
            self.slot_free[self.slot_of[g.name]] = ev

    # -- model hooks ------------------------------------------------------------------------------------
    def pre_step(self):
        """``model.unshard()`` of the reference: start gathering the first groups while data loads."""
        self.unshard(self.embed)
        if self.layer_groups:
            self.unshard(self.layer_groups[0])

    def pre_forward(self, model):
        if not self.direct_write:  # autograd accumulates into these (torch.distributed path, non-Llama models)
            self.embed.grad.zero_()
            self.head.grad.zero_()
        self.wait_unsharded(self.embed)

    def pre_layer(self, i, layer, x, residual):
        g = self.layer_groups[i]
        self.wait_unsharded(g)
        if i == 0 and not self.tied:  # a tied lm_head needs the embedding again at the end of forward
            self.release(self.embed)
        # forward prefetch: depth 1 is FSDP2's implicit prefetch; --prefetch-layers (ch05) uses every
        # rotating slot (the slot of layer i+2 is the one layer i-1 just released)
        L = len(self.layer_groups)
        for d in range(1, self.prefetch_depth + 1):
            if i + d < L:
                self.unshard(self.layer_groups[i + d])
            elif i + d == L:
                self.unshard(self.head)
        return boundary(lambda i=i: self._post_backward_layer(i), x, residual)

    def post_layer(self, i, layer, x, residual):
        self.release(self.layer_groups[i])
        return boundary(lambda i=i: self._pre_backward_layer(i), x, residual)

    def pre_head(self, x, residual):
        self.wait_unsharded(self.head)
        if self.tied:
            self.wait_unsharded(self.embed)
        return boundary(self._post_backward_head, x, residual)

    # -- backward schedule ---------------------------------------------------------------------------------
    def _enter_backward(self):
        if not self._in_backward:
            self._in_backward = True
            Variable._execution_engine.queue_callback(self._finalize_backward)

    def _post_backward_head(self):
        self._enter_backward()
        self._reduce(self.head)
        self.release(self.head)

    def _pre_backward_layer(self, i):
        self._enter_backward()
        g = self.layer_groups[i]
        self.wait_unsharded(g)
        for d in range(1, self.prefetch_depth + 1):  # backward prefetch of the previous layer(s)
            if i - d >= 0:
                self.unshard(self.layer_groups[i - d])
        if self.use_kernels:
            # the gradient slot was last used by layer i + N_GRAD_SLOTS: its reduce-scatter must be done
            j = i + len(self.grad_slots)
            if j < len(self.layer_groups):
                ev = self.rs_done.get(self.layer_groups[j].name)
                if ev is not None:
                    t0 = self._trace_begin()
                    torch.cuda.current_stream().wait_event(ev)
                    self._trace_end("stall_grad_slot", t0)
        if not self.direct_write:
            g.grad.zero_()

    def _post_backward_layer(self, i):
        g = self.layer_groups[i]
        self._reduce(g)
        self.release(g)
        # keep the slot bookkeeping honest: the parameters in this slot are stale after the update
        self.slot_owner[self.slot_of[g.name]] = None

    def _finalize_backward(self):
        self._in_backward = False
        self._reduce(self.embed)
        self._unsharded.discard("embed")
        if self.use_kernels:
            self._done.record(self.comm_stream)
            if self.measure_tail:
                # exposed communication: how long the communication stream runs past the end of backward
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                d = torch.cuda.Event(enable_timing=True)
                d.record(self.comm_stream)
                self._tails.append((e, d))

    measure_tail = False

    def exposed_comm_ms(self, last_steps=None):
        """Mean time per step the communication stream (reduce-scatter + AdamW of the last groups) kept running after
        backward had finished on the compute stream; None if not measured (bench.py sets ``measure_tail``)."""
        tails = self._tails[-last_steps:] if last_steps else self._tails
        if not tails:
            return None
        torch.cuda.synchronize()
        return sum(max(0.0, a.elapsed_time(b)) for a, b in tails) / len(tails)

    @contextlib.contextmanager
    def no_sync(self):
        """Gradient accumulation (``--grad-accum-steps``): inside this context a micro-batch's gradients are still
        reduce-scattered (the gradient slots rotate between layers, nothing full-size survives a micro-batch) but
        only ACCUMULATED into an fp32 shard-sized buffer; the optimizer runs on the boundary micro-batch."""
        old, self.sync_enabled = self.sync_enabled, False
        try:
            yield
        finally:
            self.sync_enabled = old

    def _reduce(self, g: FlatGroup):
        """reduce-scatter(mean) of ``g``'s gradient slot fused with AdamW on this rank's shard.  While gradients are
        being accumulated over micro-batches the reduce-scatter lands in an fp32 shard accumulator instead and AdamW
        runs once, on the boundary."""
        sh = self.shard_of[g.name]
        opt = self.optimizer
        st = opt.state[sh.param]
        if self.pre_reduce is not None:
            self.pre_reduce(g)
        boundary = self.sync_enabled
        accumulating = (not boundary) or st.get("acc_pending", False)
        if not self.use_kernels:
            if self.world > 1:
                buf = g.grad.float()
                dist.all_reduce(buf, group=self.pg)
                gshard = (buf / self.world)[self.rank * sh.padded_numel:(self.rank + 1) * sh.padded_numel]
            else:
                gshard = g.grad.float()
            g.zero_grad_counters()  # the next write into this gradient buffer opens a new window
            if accumulating:
                if "acc" not in st:
                    st["acc"] = torch.zeros(sh.padded_numel, dtype=torch.float32, device=gshard.device)
                st["acc"].add_(gshard)
                st["acc_pending"] = True
                if not boundary:
                    return
                gshard = st["acc"].clone()
                st["acc"].zero_()
                st["acc_pending"] = False
            st["step"] += 1
            if self.cpu_offload:  # the update itself happens in optimizer.step() on the host copies
                st["cpu_grad"].copy_((gshard * opt.grad_scale).to(st["cpu_grad"].dtype))
                return
            lr, b1, b2, eps, wd = opt.hyper()
            ref.adamw_step(sh.param, gshard.to(sh.param.dtype), st["exp_avg"], st["exp_avg_sq"], lr, b1, b2, eps, wd,
                           st["step"], opt.grad_scale)
            return
        join_wgrad_stream()
        ev = torch.cuda.Event()
        ev.record()
        gbuf = self._symm_of[g.grad.data_ptr() if g.name in ("embed", "head") else
                             self.grad_slots[self.gslot_of[g.name]].data_ptr()]
        g.zero_grad_counters()
        with torch.cuda.stream(self.comm_stream):
            self.comm_stream.wait_event(ev)
            scale = opt.grad_scale / self.world
            if accumulating:
                if "gpu_grad" not in st:
                    st["gpu_grad"] = torch.zeros_like(sh.param)
                if "acc" not in st:
                    st["acc"] = torch.zeros(sh.padded_numel, dtype=torch.float32, device=sh.param.device)
                self.symm.reduce_scatter_(gbuf, st["gpu_grad"], 0, g.padded_numel, scale)
                st["acc"].add_(st["gpu_grad"])
                st["acc_pending"] = True
                if boundary:
                    st["step"] += 1
                    st["gpu_grad"].copy_(st["acc"])
                    st["acc"].zero_()
                    st["acc_pending"] = False
                    if self.cpu_offload:
                        st["cpu_grad"].copy_(st["gpu_grad"], non_blocking=True)
                    else:
                        lr, b1, b2, eps, wd = opt.hyper()
                        self.symm.C.adamw_flat(sh.param, st["gpu_grad"], st["exp_avg"], st["exp_avg_sq"], lr, b1, b2,
                                               eps, wd, st["step"], 1.0)
            elif self.cpu_offload:
                st["step"] += 1
                self.symm.reduce_scatter_(gbuf, st["gpu_grad"], 0, g.padded_numel, scale)
                st["cpu_grad"].copy_(st["gpu_grad"], non_blocking=True)
            else:
                st["step"] += 1
                t0 = self._trace_begin()
                with nvtx_range(f"reduce_adamw:{g.name}"):
                    self.symm.rs_adamw_(gbuf, None, sh.param, st["exp_avg"], st["exp_avg_sq"], False, 0,
                                        g.padded_numel, opt.hyper(), st["step"], scale)
                self._trace_end("reduce_adamw", t0)
            done = torch.cuda.Event()
            done.record(self.comm_stream)
            self.rs_done[g.name] = done

    # -- optional device-side trace ---------------------------------------------------------------------------------
    def _trace_begin(self):
        if self.trace is None:
            return None
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e

    def _trace_end(self, kind, t0):
        if t0 is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.trace.append((kind, t0, e))

    def comm_trace_summary(self, last_steps=None):
        """Per step: device time of the unshard / reduce kernels (communication stream) and how long the compute
        stream sat in each kind of wait."""
        if not self.trace:
            return {}
        torch.cuda.synchronize()
        steps = max(1, self._trace_steps)
        per = {}
        for kind, a, b in self.trace:
            per.setdefault(kind, []).append(a.elapsed_time(b))
        return {k: {"per_step_ms": round(sum(v) / steps, 2), "mean_ms": round(sum(v) / len(v), 3), "n": len(v) // steps}
                for k, v in per.items()}

    _trace_steps = 0

    # -- optimizer step: everything already happened inside backward ------------------------------------------
    def _optimizer_step(self):
        opt = self.optimizer
        if self.use_kernels:
            t0 = self._trace_begin()
            torch.cuda.current_stream().wait_event(self._done)
            self._trace_end("stall_tail", t0)
            self._trace_steps += 1
        if self.cpu_offload:
            if self.use_kernels:
                self.comm_stream.synchronize()
            lr, b1, b2, eps, wd = opt.hyper()
            for sh in self.shards:
                st = opt.state[sh.param]
                ref.adamw_step(st["cpu_param"], st["cpu_grad"], st["exp_avg"], st["exp_avg_sq"], lr, b1, b2, eps, wd,
                               st["step"], 1.0)
                if self.use_kernels:
                    with torch.cuda.stream(self.comm_stream):  # ordered before the next unshard
                        sh.param.copy_(st["cpu_param"], non_blocking=True)
                else:
                    sh.param.copy_(st["cpu_param"])

    # -- checkpoint payload --------------------------------------------------------------------------------------
    def sharded_state(self):
        opt = self.optimizer
        model_sd = {s.name: s.param for s in self.shards}
        opt_sd = {}
        for s in self.shards:
            st = opt.state[s.param]
            opt_sd[f"{s.name}.exp_avg"] = st["exp_avg"]
            opt_sd[f"{s.name}.exp_avg_sq"] = st["exp_avg_sq"]
        return {"model": model_sd, "optimizer": opt_sd}

    def layout_description(self):
        """Where every named parameter sits inside its group's flat buffer (saved next to sharded checkpoints so
        tools can cut the groups back into tensors without re-deriving padding / ordering rules)."""
        return {g.name: {"padded_numel": g.padded_numel, "names": list(g.names), "offsets": list(g.offsets),
                         "shapes": [list(s) for s in g.shapes]} for g in self.groups}

    def optimizer_steps(self):
        return {s.name: self.optimizer.state[s.param]["step"] for s in self.shards}

    def set_optimizer_steps(self, steps):
        for s in self.shards:
            self.optimizer.state[s.param]["step"] = int(steps.get(s.name, 0))

    def after_load(self):
        """A checkpoint was loaded into the GPU shards: refresh what was derived from them at construction — with
        ``--cpu-offload`` the host master copy AdamW updates (it was snapshotted from the freshly initialised
        weights in ``build_optimizer`` and would otherwise overwrite the loaded ones at the first step)."""
        if self.optimizer is None:
            return
        for s in self.shards:
            st = self.optimizer.state[s.param]
            if "cpu_param" in st:
                st["cpu_param"].copy_(s.param)
        # every full slot is stale now
        for i in range(len(self.slot_owner)):
            self.slot_owner[i] = None
        self._unsharded.clear()

    def full_state_dict(self):
        """Gather every group and return an HF-named full state dict (for export / tests)."""
        out = {}
        for g in self.groups:
            if g.name not in ("embed", "head"):
                self.slot_owner[self.slot_of[g.name]] = None
            else:
                self._unsharded.discard(g.name)
            self.wait_unsharded(g, force_full=True)
            if self.use_kernels:
                torch.cuda.synchronize(self.device)
            for n, p in zip(g.names, g.params):
                out[n] = p.detach().clone()
            if g.name in ("embed", "head"):
                self._unsharded.discard(g.name)
            else:
                self.slot_owner[self.slot_of[g.name]] = None
        return out
