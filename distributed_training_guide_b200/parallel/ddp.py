"""Data parallelism with the gradient collective fused into the bucket kernel (chapter 02).

Reference: ``DistributedDataParallel(model, bucket_cap_mb=500, gradient_as_bucket_view=True)`` plus
``ZeroRedundancyOptimizer(AdamW, fused=True)`` (``02-distributed-data-parallel/train_llm.py:66-68,
87-89``).  There, torch's C++ Reducer copies/pre-divides gradients into ≤500 MiB buckets and launches
one NCCL all-reduce per bucket on a side stream; ZeRO-1 then updates 1/N of the tensors per rank and
issues ~291 per-tensor NCCL broadcasts that are fully exposed in ``optimizer.step()`` (SURVEY.md N2/N3).

Here a *bucket* is a flat group (embedding, each decoder layer, head) whose gradients the wgrad
GEMMs already wrote into one symmetric buffer.  When the autograd boundary in front of a layer
fires (all of that layer's gradients are final) the engine launches, on a communication stream and
overlapped with the rest of backward, ONE kernel per bucket:

  * ``zero1=True``  reduce-scatter (pull my 1/N slice from all peers over NVLink) -> 1/N scale ->
                    AdamW on my optimizer-state shard -> push the updated bf16 parameters into every
                    replica (``comm.cu: rs_adamw_kernel<PUSH_PARAMS=true>``).  ``optimizer.step()`` then
                    only joins the communication stream: no all-reduce, no broadcasts.
  * ``zero1=False`` two-shot all-reduce with the 1/N scale fused (``allreduce_scale_kernel``); the
                    optimizer then updates the full replica locally (plain DDP).

``no_sync()`` (gradient accumulation, reference related-topics/gradient-accumulation) skips the
bucket kernels on non-boundary micro-batches; the wgrad GEMMs keep accumulating in place.
On CPU (gloo tests) the same engine falls back to ``torch.distributed`` collectives.

Gradient clipping (``optimizer.max_grad_norm``, ``csrc/grad_clip.cu``) needs the norm of every bucket before any
update, so the step is split: in backward each bucket kernel only reduces its slice, stores it (ZeRO-1: in this
rank's own slice of its gradient buffer; all-reduce: in every replica) and sums the squares of what it stored; in
``optimizer.step()`` one finalize kernel turns those partial sums into the global norm and the clip factor on the
device, and an AdamW kernel per bucket applies it (ZeRO-1: then pushes the new parameters to every replica).  With
clipping off nothing of this runs.
"""
from __future__ import annotations

import contextlib
import os
from typing import List

import torch
import torch.distributed as dist
from torch.autograd import Variable

from ..ops import join_wgrad_stream
from ..utils.timers import nvtx_range
from .flat import FlatGroup
from .optim import FlatAdamW


class _Boundary(torch.autograd.Function):
    """Identity in forward; in backward, runs ``callback()`` once the gradients of everything
    downstream of this point (i.e. the whole layer behind it) have been produced."""

    @staticmethod
    def forward(ctx, callback, x, residual):
        ctx.callback = callback
        ctx.has_res = residual is not None
        if residual is None:
            return x.view_as(x)
        return x.view_as(x), residual.view_as(residual)

    @staticmethod
    def backward(ctx, *grads):
        ctx.callback()
        if ctx.has_res:
            return None, grads[0], grads[1]
        return None, grads[0], None


def boundary(callback, x, residual):
    if not torch.is_grad_enabled():
        return x, residual
    out = _Boundary.apply(callback, x, residual)
    if residual is None:
        return out, None
    return out


class DataParallelEngine:
    def __init__(self, model, groups: List[FlatGroup], optimizer: FlatAdamW, symm=None, registry=None, pg=None,
                 zero1: bool = True, world_size: int = 1, rank: int = 0):
        self.model, self.groups, self.optimizer = model, groups, optimizer
        self.symm, self.registry, self.pg = symm, registry or {}, pg
        self.zero1, self.world, self.rank = zero1, world_size, rank
        self.sync_enabled = True
        self._in_backward = False
        self.by_name = {g.name: g for g in groups}
        self.use_kernels = symm is not None
        if self.use_kernels:
            self.comm_stream = torch.cuda.Stream(device=symm.device)
            self._done = torch.cuda.Event()
        model.engine = self
        optimizer.external_step = self._optimizer_step
        self._pending = []  # buckets reduced this step (for the CPU fallback's deferred update)
        self.measure_tail, self._tails = False, []  # bench.py: two events per step -> exposed_comm_ms()
        # DTG_COMM_TRACE=1: CUDA events around every bucket kernel (see comm_trace_summary)
        self.trace = [] if (self.use_kernels and os.environ.get("DTG_COMM_TRACE")) else None
        # DTG_DEBUG_MARKERS=1: keep, per bucket of the current step, the event recorded on the compute stream when
        # the bucket became ready and the one behind its kernel on the communication stream (stall post-mortems)
        self.markers = {} if (self.use_kernels and os.environ.get("DTG_DEBUG_MARKERS")) else None
        self.clip = getattr(optimizer, "max_grad_norm", None) is not None
        if self.clip and self.use_kernels:
            self._setup_clip()

    def _setup_clip(self):
        """Device buffers of the clipped step: per bucket, its parameter element ranges and one fp64 partial sum of
        squares per CTA; a symmetric slot per rank for the cross-rank sum; (norm, coef) in fp32."""
        dev, blocks = self.symm.device, self.symm.comm_blocks
        self._bucket_index = {g.name: i for i, g in enumerate(self.groups)}
        self._ranges = {}
        for g in self.groups:
            merged = []
            for o, shape in zip(g.offsets, g.shapes):
                n = 1
                for d in shape:
                    n *= d
                if merged and merged[-1][1] == o:
                    merged[-1][1] = o + n   # adjacent parameters: one range
                elif n:
                    merged.append([o, o + n])
            self._ranges[g.name] = torch.tensor(merged or [[0, 0]], dtype=torch.int64, device=dev)
        self._partials = torch.zeros(len(self.groups) * blocks, dtype=torch.float64, device=dev)
        self._slots = self.symm.alloc(2, torch.float64)   # one sum per step parity (collective allocation)
        self._clip_out = torch.zeros(2, dtype=torch.float32, device=dev)
        self._clip_steps = 0

    # -- hooks called by the model ---------------------------------------------------------------
    def pre_forward(self, model):
        pass

    def pre_layer(self, i, layer, x, residual):
        g = getattr(layer, "_flat_group", None)
        if g is None:
            return x, residual
        return boundary(lambda g=g: self._bucket_ready(g), x, residual)

    def post_layer(self, i, layer, x, residual):
        return x, residual

    def pre_head(self, x, residual):
        g = self.by_name.get("head")
        if g is None:
            return x, residual
        return boundary(lambda g=g: self._bucket_ready(g), x, residual)

    # -- gradient synchronisation ---------------------------------------------------------------------
    @contextlib.contextmanager
    def no_sync(self):
        old, self.sync_enabled = self.sync_enabled, False
        try:
            yield
        finally:
            self.sync_enabled = old

    def _bucket_ready(self, g: FlatGroup):
        if not self._in_backward:
            self._in_backward = True
            Variable._execution_engine.queue_callback(self._finalize_backward)
        if self.sync_enabled:
            self._launch(g)

    def _finalize_backward(self):
        self._in_backward = False
        if not self.sync_enabled:
            return
        g = self.by_name.get("embed")
        if g is not None:
            self._launch(g)  # the embedding gradient is only complete at the very end of backward
        if self.use_kernels:
            self._done.record(self.comm_stream)
            if self.measure_tail:
                # exposed communication: how long the communication stream runs past the end of backward
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                d = torch.cuda.Event(enable_timing=True)
                d.record(self.comm_stream)
                self._tails.append((e, d))
            if self.trace is not None:
                e = torch.cuda.Event(enable_timing=True)
                e.record()  # end of backward on the compute stream
                d = torch.cuda.Event(enable_timing=True)
                d.record(self.comm_stream)
                self.trace.append(("end", e, d))

    def _launch(self, g: FlatGroup):
        if not self.use_kernels:
            self._launch_fallback(g)
            return
        join_wgrad_stream()
        ev = torch.cuda.Event()
        ev.record()  # on the compute stream: this bucket's wgrad kernels are all enqueued before it
        gbuf = self.registry[g.grad.data_ptr()]
        with torch.cuda.stream(self.comm_stream):
            self.comm_stream.wait_event(ev)
            if self.trace is not None:
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record()
                self._run_bucket(g, gbuf)
                t1.record()
                self.trace.append((g.name, t0, t1))
                return
            self._run_bucket(g, gbuf)
            if self.markers is not None:
                done = torch.cuda.Event()
                done.record(self.comm_stream)
                self.markers[g.name] = (ev, done)

    def describe_progress(self) -> str:
        """Which buckets of the step in flight have (a) become ready on the compute stream and (b) finished their
        fused kernel on the communication stream — event queries only, safe to call while the device is wedged."""
        if not self.markers:
            return "(no markers: set DTG_DEBUG_MARKERS=1)"
        ready = [n for n, (a, b) in self.markers.items() if a.query()]
        done = [n for n, (a, b) in self.markers.items() if b.query()]
        names = list(self.markers)
        return (f"buckets launched this step: {len(names)} (last {names[-1]}); compute stream reached: "
                f"{ready[-1] if ready else None} ({len(ready)}); comm stream finished: {done[-1] if done else None} "
                f"({len(done)}); comm stream idle: {self.comm_stream.query()}")

    def exposed_comm_ms(self, last_steps=None):
        """Mean time per step the communication stream kept running after backward had finished on the compute
        stream (the part of the bucket kernels that is NOT hidden under backward); None if not measured."""
        tails = self._tails[-last_steps:] if last_steps else self._tails
        if not tails:
            return None
        torch.cuda.synchronize()
        return sum(max(0.0, a.elapsed_time(b)) for a, b in tails) / len(tails)

    def comm_trace_summary(self, last_steps=None):
        """{"bucket_ms": mean device time per bucket kernel, "sum_ms": per step, "tail_ms": how long the
        communication stream runs past the end of backward} from the DTG_COMM_TRACE events."""
        if not self.trace:
            return {}
        torch.cuda.synchronize()
        ends = [i for i, t in enumerate(self.trace) if t[0] == "end"]
        if last_steps:
            start = ends[-last_steps - 1] + 1 if len(ends) > last_steps else 0
        else:
            start = 0
        rows = self.trace[start:]
        n_steps = max(1, sum(1 for t in rows if t[0] == "end"))
        per = {}
        for name, a, b in rows:
            if name != "end":
                key = "layer" if name.startswith("layer") else name
                per.setdefault(key, []).append(a.elapsed_time(b))
        tails = [a.elapsed_time(b) for name, a, b in rows if name == "end"]
        return {"bucket_ms": {k: round(sum(v) / len(v), 3) for k, v in per.items()},
                "sum_ms": round(sum(sum(v) for v in per.values()) / n_steps, 2),
                "tail_ms": round(sum(tails) / len(tails), 3) if tails else None}

    def _run_bucket(self, g, gbuf):
        with nvtx_range(f"bucket:{g.name}"):
            self._run_bucket_impl(g, gbuf)

    def _run_bucket_impl(self, g, gbuf):
        opt = self.optimizer
        if self.clip:
            # reduce + sum of squares only; the update waits for the global norm (_clipped_step)
            blocks = self.symm.comm_blocks
            i = self._bucket_index[g.name]
            scale = (opt.grad_scale if self.zero1 else 1.0) / self.world
            self.symm.reduce_sumsq_(gbuf, 0, g.padded_numel, scale, not self.zero1, self._ranges[g.name],
                                    self._partials[i * blocks:(i + 1) * blocks], blocks)
            return
        if self.zero1:
            st = opt.state[g.param]
            st["step"] += 1
            pbuf = self.registry[g.param.data_ptr()]
            self.symm.rs_adamw_(gbuf, pbuf, None, st["exp_avg"], st["exp_avg_sq"], True, 0, g.padded_numel,
                                opt.hyper(), st["step"], opt.grad_scale / self.world)
        else:
            self.symm.allreduce_scale_(gbuf, 0, g.padded_numel, 1.0 / self.world)

    def _launch_fallback(self, g: FlatGroup):
        """torch.distributed path (CPU / gloo): all-reduce now, sharded update in optimizer.step()."""
        if self.world > 1:
            buf = g.grad.float()
            dist.all_reduce(buf, group=self.pg)
            g.grad.copy_((buf / self.world).to(g.grad.dtype))
        self._pending.append(g)

    # -- optimizer step ---------------------------------------------------------------------------------
    def _clipped_step(self):
        """On the communication stream, behind the bucket kernels of backward: the global norm and clip factor
        (one finalize kernel), then AdamW with ``g *= coef`` per bucket; ZeRO-1 pushes the new parameters of its
        shard into every replica and ends with one device barrier, so no rank starts its next forward before every
        push has landed."""
        opt, sg, C = self.optimizer, self.symm, self.symm.C
        lr, b1, b2, eps, wd = opt.hyper()
        with torch.cuda.stream(self.comm_stream), nvtx_range("clip:step"):
            # ZeRO-1 folded grad_scale into the stored gradient; plain DDP stored g / N and AdamW applies grad_scale
            norm_scale = 1.0 if self.zero1 else opt.grad_scale
            sg.clip_finalize_(self._partials, self._slots, self._clip_steps & 1, norm_scale, opt.max_grad_norm,
                              self._clip_out)
            self._clip_steps += 1
            coef = self._clip_out[1:]
            for g in self.groups:
                st = opt.state[g.param]
                st["step"] += 1
                if self.zero1:
                    lo, hi = g.shard_range(self.rank, self.world)
                    pbuf = self.registry[g.param.data_ptr()]
                    mc = (pbuf.mc_ptr + 2 * lo) if (sg.nvls and pbuf.mc_ptr and self.world > 1) else 0
                    dst = [] if mc else [pbuf.ptrs[(self.rank + k) % self.world] + 2 * lo for k in range(self.world)]
                    C.comm_adamw_clip(dst, mc, g.param[lo:hi], g.grad[lo:hi], st["exp_avg"], st["exp_avg_sq"],
                                      lr, b1, b2, eps, wd, st["step"], 1.0, coef)
                else:
                    C.comm_adamw_clip([g.param.data_ptr()], 0, g.param, g.grad, st["exp_avg"], st["exp_avg_sq"],
                                      lr, b1, b2, eps, wd, st["step"], opt.grad_scale, coef)
            if self.zero1 and self.world > 1:
                sg.barrier_()
            self._done.record(self.comm_stream)
        torch.cuda.current_stream().wait_event(self._done)
        opt.last_grad_norm = self._clip_out[0].clone()

    def _optimizer_step(self):
        opt = self.optimizer
        if self.use_kernels:
            if self.clip:
                self._clipped_step()
                return
            torch.cuda.current_stream().wait_event(self._done)  # join the communication stream
            if not self.zero1:
                for g in self.groups:
                    opt.step_group(g)
            return
        coef = opt.clip_coefficient()  # over the all-reduced full gradients: the same on every rank
        for g in self.groups:
            opt.step_group(g, coef)  # on its shard when ZeRO-1 (optimizer built with shard=(rank, world))
            if self.zero1 and self.world > 1:
                lo, hi = g.shard_range(self.rank, self.world)
                shards = [torch.empty(hi - lo, dtype=torch.float32) for _ in range(self.world)]
                dist.all_gather(shards, g.param[lo:hi].float(), group=self.pg)
                g.param.copy_(torch.cat(shards).to(g.param.dtype))
        self._pending.clear()


class LocalOverlapEngine(DataParallelEngine):
    """Optimizer-in-backward without a data-parallel collective (pure tensor parallelism, dp = 1).

    When a bucket's gradients are final, ``pre_update(g)`` runs on the compute stream (tensor parallelism: sum
    the replicated norm-gain gradients over the tp group) and AdamW for that bucket runs on a side stream under
    the rest of backward, so ``optimizer.step()`` only joins that stream (the reference runs one fused AdamW
    over the whole model after backward, ``06-tensor-parallel/train_llm.py:151,236``)."""

    def __init__(self, model, groups, optimizer, device, pre_update=None):
        super().__init__(model, groups, optimizer, symm=None, world_size=1, rank=0)
        self.pre_update = pre_update
        self.device = torch.device(device)
        self.use_kernels = self.device.type == "cuda"
        if self.use_kernels:
            self.comm_stream = torch.cuda.Stream(device=self.device)
            self._done = torch.cuda.Event()

    def _launch(self, g: FlatGroup):
        if self.pre_update is not None:
            self.pre_update(g)
        if not self.use_kernels:
            self.optimizer.step_group(g)
            return
        join_wgrad_stream()
        ev = torch.cuda.Event()
        ev.record()
        with torch.cuda.stream(self.comm_stream):
            self.comm_stream.wait_event(ev)
            self.optimizer.step_group(g)

    def _optimizer_step(self):
        if self.use_kernels:
            torch.cuda.current_stream().wait_event(self._done)
