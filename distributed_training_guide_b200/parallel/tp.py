"""Tensor parallelism with Megatron-style sequence parallelism (chapters 06 / 07).

Reference plan (``06-tensor-parallel/train_llm.py:79-121``): embedding ColwiseParallel (hidden-sharded,
output redistributed to sequence shards), q/k/v/gate/up ColwiseParallel, o/down RowwiseParallel with
``output_layouts=Shard(1)``, norms SequenceParallel, ``PrepareModuleInput`` all-gathers before attention
and MLP, lm_head ColwiseParallel with replicated logits.  DTensor turns each of those into a standalone
NCCL all-gather / reduce-scatter / all-to-all sitting on the critical path of every block
(SURVEY.md N7-N10).

Here the activations between blocks are sequence shards ``[T/t, H]`` living in NVLink-symmetric
buffers, and the collectives disappear into the tensor-core kernels:

  * column-parallel linear = ONE wgmma GEMM kernel in which a few communication CTAs bulk-copy the
    peers' row tiles over NVLink into the local gathered buffer and publish per-tile flags, while the
    GEMM CTAs start on the local rows and acquire a tile's flag before their TMA reads it (all-gather ->
    GEMM, ``gemm_ag``; a variant that TMA-loads every tile from its owner, ``gemm_dist`` mode 1, re-fetches
    remote tiles once per N tile because peer memory bypasses the local L2);
  * row-parallel linear = ONE GEMM whose epilogue stores each row chunk straight into the owner's
    staging slot (GEMM -> reduce-scatter, mode 2); the owner sums the t partials (+ residual) in the
    kernel that feeds the next RMSNorm;
  * their weight gradients contract over the full sequence and read the copy the forward (resp. dgrad)
    kernel gathered, so backward needs no second all-gather (K-gathered GEMM modes 3 / 4 also exist);
  * lm_head logits stay vocabulary-sharded and the loss is a vocab-parallel cross entropy (the
    "loss parallel" the reference only documents, ``06-tensor-parallel/README.md:241-271``);
  * the embedding is hidden-sharded and its all-to-all is fused into the lookup kernel.

Cross-rank ordering uses the device-side barrier kernel of ``SymmGroup`` (one tiny launch before a
gather / after a push).  On CPU (gloo tests) every op falls back to ``torch.distributed``.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch
import torch.distributed as dist

from .. import _ext, ops
from ..ops import reference as ref


class TPContext:
    """Per-model tensor-parallel state: group, symmetric scratch buffers, geometry."""

    def __init__(self, tp_size, tp_rank, pg, symm, device, hidden, max_tokens, n_layers, dtype):
        self.t, self.rank, self.pg, self.symm, self.device = tp_size, tp_rank, pg, symm, device
        self.H, self.dtype = hidden, dtype
        self.use_kernels = symm is not None
        self.max_tokens = max_tokens
        assert max_tokens % tp_size == 0
        self.rpp = max_tokens // tp_size  # rows (tokens) per rank
        if self.use_kernels and tp_size > 1 and self.rpp % 256 != 0:
            raise ValueError(
                f"tensor parallelism: tokens per rank = batch x seq / tp = {max_tokens} / {tp_size} = {self.rpp} must be "
                "a multiple of 256 (one CTA-pair row tile of the fused all-gather -> GEMM kernel); raise -b or -s")
        self.n_layers = n_layers
        if self.use_kernels:
            import os

            Tl, H = self.rpp, hidden
            T = max_tokens
            # column-parallel inputs, one FULL [T, H] slot per use ([layer][attn-in | mlp-in] + lm_head input):
            # a rank writes its own rows, the all-gather->GEMM kernel fetches the others into the same slot and
            # the gathered copy is what the weight-gradient GEMM reads in backward (no second gather)
            self.act = symm.alloc((2 * n_layers + 1) * T * H, dtype)
            # GEMM -> reduce-scatter.  With an NVLS multicast binding: two [T, H] buffers the row-parallel GEMMs write
            # their full partial into (local stores), reduced in the switch by the consumer (`reduce_scatter_partial`).
            # Without: per-rank staging slots the GEMM epilogue pushes row chunks into.
            self.mc_rs = bool(getattr(symm, "multicast", False)) and tp_size > 1 \
                and os.environ.get("DTG_TP_RS", "mc") == "mc"
            if self.mc_rs:
                self.part = [symm.alloc(T * H, dtype) for _ in range(2)]
                self._part_i = 0
                self.stage = []
            else:
                self.stage = [symm.alloc(tp_size * Tl * H, dtype) for _ in range(2)]  # reduce-scatter landing zones
            self.gbuf = [symm.alloc(T * H, dtype) for _ in range(2)]             # gathered grads of row-parallel outputs
            self.flags = torch.zeros(max(1, T // 256), dtype=torch.int32, device=device)
            self.ag_epoch = 0
            self.n_comm = int(os.environ.get("DTG_TP_COMM_CLUSTERS", "4"))
            self.x0 = symm.alloc(Tl * H, dtype)    # embedding output (all-to-all target)
            self.dx0 = symm.alloc(Tl * H, dtype)   # its gradient
            self.stats = symm.alloc(max_tokens * 4, torch.float32)
            self._stage_i = 0
            self._gbuf_i = 0

    # symmetric slices ---------------------------------------------------------------------------
    def act_slot(self, idx):
        """(full [T, H] view of slot idx, view of my rows inside it, per-rank base pointers of the slot)."""
        n = self.max_tokens * self.H
        full = self.act.local[idx * n:(idx + 1) * n].view(self.max_tokens, self.H)
        mine = full[self.rank * self.rpp:(self.rank + 1) * self.rpp]
        return full, mine, [p + idx * n * 2 for p in self.act.ptrs]

    def gather_gemm(self, bufs, b, out, b_kmajor, bias=None):
        """out = all_gather_rows(symmetric buffer) @ op(b) (+ bias): ONE kernel, the gather runs on communication
        CTAs, the bias is added in the epilogue (forward form only)."""
        self.ag_epoch += 1
        self.symm.C.gemm_ag(bufs, b, out, b_kmajor, self.rank, self.rpp, self.flags, self.ag_epoch, self.symm.pad_ptrs,
                            self.symm._epochs(1), self.n_comm, bias)

    def row_parallel_gemm(self, a, w, trans_b, residual):
        """reduce_scatter_rows(a @ op(w)) (+ residual) -> [T/t, H] for this rank (GPU kernels).

        Reference: ``RowwiseParallel(output_layouts=Shard(1))`` on ``o_proj`` / ``down_proj``
        (``06-tensor-parallel/train_llm.py:99,108``): a cuBLAS GEMM followed by a standalone NCCL reduce-scatter."""
        C = self.symm.C
        T, Tl, H = a.shape[0], self.rpp, self.H
        y = torch.empty(Tl, H, dtype=a.dtype, device=a.device)
        if self.mc_rs:
            # ONE plain wgmma GEMM into my copy of the partial buffer + ONE kernel that barriers and reads my
            # rows through the multicast address (in-switch fp32 sum) fused with the residual add.  Two buffers
            # alternate: a buffer is rewritten two GEMMs later, after a barrier every rank passed in between.
            pb = self.part[self._part_i]
            self._part_i ^= 1
            ops.gemm(a, w, out=pb.local.view(T, H), trans_b=trans_b)
            C.tp_reduce_mc(pb.mc_ptr + self.rank * Tl * H * 2, residual, y, self.symm.pad_ptrs, self.rank,
                           self.symm._epochs(1), self.symm.err)
            return y
        st = self.next_stage()
        my_slot = self.rank * Tl * H * 2
        k = a.shape[1]
        C.gemm_dist(2, [a.data_ptr()], [w.data_ptr()], [p + my_slot for p in st.ptrs], T, H, k, a.stride(0), w.stride(0),
                    H, trans_b, False, self.t, self.rank, Tl)
        self.barrier()
        C.tp_reduce_parts(st.local.view(self.t, Tl, H), residual, y)
        return y

    def next_stage(self):
        b = self.stage[self._stage_i]
        self._stage_i ^= 1
        return b

    def next_gbuf(self):
        b = self.gbuf[self._gbuf_i]
        self._gbuf_i ^= 1
        return b

    def barrier(self):
        if self.use_kernels:
            self.symm.barrier_()
        elif self.t > 1:
            dist.barrier(group=self.pg)

    # torch.distributed fallbacks ----------------------------------------------------------------------
    def all_gather_rows(self, x_local):
        if self.t == 1:
            return x_local
        parts = [torch.empty_like(x_local) for _ in range(self.t)]
        dist.all_gather(parts, x_local.contiguous(), group=self.pg)
        return torch.cat(parts, dim=0)

    def reduce_scatter_rows(self, x_full):
        if self.t == 1:
            return x_full
        buf = x_full.float().contiguous()
        dist.all_reduce(buf, group=self.pg)
        return buf[self.rank * self.rpp:(self.rank + 1) * self.rpp].to(x_full.dtype)

    def all_reduce_(self, x):
        if self.t > 1:
            buf = x.float()
            dist.all_reduce(buf, group=self.pg)
            x.copy_(buf.to(x.dtype))
        return x


class _ColumnParallelLinear(torch.autograd.Function):
    """y_full[T, n_local] = all_gather_rows(x_local)[T, H] @ W_local[n_local, H]^T (+ b_local[n_local])

    A bias is split with the output features.  Every rank's output gradient covers all T tokens, so the gradient of
    its bias slice is complete without any reduction over the group."""

    @staticmethod
    def forward(ctx, x_local, w, owner, tp: TPContext, slot, bias=None, bias_owner=None):
        ctx.tp, ctx.owner, ctx.slot = tp, owner, slot
        ctx.bias, ctx.bias_owner = bias, bias_owner
        T, H, n = tp.rpp * tp.t, x_local.shape[1], w.shape[0]
        if not tp.use_kernels:
            xf = tp.all_gather_rows(x_local)
            ctx.save_for_backward(x_local, w)
            return xf @ w.t() if bias is None else xf @ w.t() + bias
        full, mine, ptrs = tp.act_slot(slot)
        mine.copy_(x_local)          # my sequence shard, where the peers' copy engines can reach it
        out = torch.empty(T, n, dtype=x_local.dtype, device=x_local.device)
        tp.gather_gemm(ptrs, w, out, True, bias)   # barrier + all-gather + GEMM in one kernel; `full` is now complete
        ctx.save_for_backward(w)
        return out

    @staticmethod
    def backward(ctx, dy):
        tp, owner = ctx.tp, ctx.owner
        dy = dy.contiguous()
        T, n = dy.shape
        db = None
        if ctx.bias is not None:
            bo = ctx.bias_owner if ctx.bias_owner is not None else ctx.bias
            if tp.use_kernels:
                db = ops._emit_bias_grad(bo, dy, ctx.bias)
            else:
                db = _route_dw(bo, dy.float().sum(0).to(ctx.bias.dtype))
        if not tp.use_kernels:
            x_local, w = ctx.saved_tensors
            xf = tp.all_gather_rows(x_local)
            dw = dy.t() @ xf
            dx = tp.reduce_scatter_rows(dy @ w)
            return dx, dw if owner is None else _route_dw(owner, dw), None, None, None, db, None
        C = _ext.load()
        (w,) = ctx.saved_tensors
        H = w.shape[1]
        full, _, _ = tp.act_slot(ctx.slot)
        # wgrad: dW[n, H] (+)= dy^T[n, T] @ x_full[T, H]   (the copy gathered by the forward kernel)
        gbuf = owner._dtg_grad
        acc = owner._dtg_writes > 0
        owner._dtg_writes += 1
        ops.gemm(dy, full, out=gbuf, trans_a=True, accumulate=acc)
        # dgrad: dx[T/t, H] = reduce_scatter_rows(dy[T, n] @ W[n, H])
        dx = tp.row_parallel_gemm(dy, w, False, None)
        return dx, None, None, None, None, db, None


def _route_dw(owner, dw):
    """CPU path: put a weight gradient where the flat-buffer protocol expects it."""
    g = getattr(owner, "_dtg_grad", None)
    if g is None:
        return dw
    if getattr(owner, "_dtg_writes", 0) > 0:
        g.add_(dw.to(g.dtype))
    else:
        g.copy_(dw.to(g.dtype))
    owner._dtg_writes = getattr(owner, "_dtg_writes", 0) + 1
    return None


class _RowParallelLinear(torch.autograd.Function):
    """y_local[T/t, H] = reduce_scatter_rows( x[T, k_local] @ W_local[H, k_local]^T ) (+ residual)"""

    @staticmethod
    def forward(ctx, x, w, owner, tp: TPContext, residual):
        ctx.tp, ctx.owner = tp, owner
        ctx.has_res = residual is not None
        T, k = x.shape
        H = w.shape[0]
        ctx.save_for_backward(x, w)
        if not tp.use_kernels:
            y = tp.reduce_scatter_rows(x @ w.t())
            return y + residual if residual is not None else y
        return tp.row_parallel_gemm(x, w, True, residual)

    @staticmethod
    def backward(ctx, dy_local):
        tp, owner = ctx.tp, ctx.owner
        x, w = ctx.saved_tensors
        dy_local = dy_local.contiguous()
        T, k = x.shape
        H = w.shape[0]
        dres = dy_local if ctx.has_res else None
        if not tp.use_kernels:
            dyf = tp.all_gather_rows(dy_local)
            dx = dyf @ w
            dw = dyf.t() @ x
            return dx, dw if owner is None else _route_dw(owner, dw), None, None, dres
        gb = tp.next_gbuf()
        gfull = gb.local.view(T, H)
        gfull[tp.rank * tp.rpp:(tp.rank + 1) * tp.rpp].copy_(dy_local)
        # dgrad: dx[T, k] = all_gather_rows(dy)[T, H] @ W[H, k]   (gather + GEMM in one kernel)
        dx = torch.empty(T, k, dtype=x.dtype, device=x.device)
        tp.gather_gemm(gb.ptrs, w, dx, False)
        # wgrad: dW[H, k] (+)= dy_full^T[H, T] @ x[T, k]   (reads the copy the dgrad kernel gathered)
        gbuf = owner._dtg_grad
        acc = owner._dtg_writes > 0
        owner._dtg_writes += 1
        ops.gemm(gfull, x, out=gbuf, trans_a=True, accumulate=acc)
        return dx, None, None, None, dres


class _HiddenParallelEmbedding(torch.autograd.Function):
    """x_local[T/t, H]: every rank looks up its H/t columns for all tokens and pushes them to the owner."""

    @staticmethod
    def forward(ctx, ids, w, tp: TPContext):
        ctx.tp, ctx.w = tp, w
        ids = ids.reshape(-1).contiguous()
        ctx.save_for_backward(ids)
        if not tp.use_kernels:
            part = w[ids]                                   # [T, H/t]
            if tp.t == 1:
                return part
            cols = [torch.empty_like(part) for _ in range(tp.t)]
            dist.all_gather(cols, part, group=tp.pg)
            full = torch.cat(cols, dim=1)                   # [T, H]
            return full[tp.rank * tp.rpp:(tp.rank + 1) * tp.rpp].contiguous()
        C = _ext.load()
        C.tp_embed_fwd(ids, w, tp.x0.ptrs, tp.rpp, tp.H, tp.rank)
        tp.barrier()
        return tp.x0.local.view(tp.rpp, tp.H).clone()

    @staticmethod
    def backward(ctx, dx_local):
        tp, w = ctx.tp, ctx.w
        (ids,) = ctx.saved_tensors
        Hl = w.shape[1]
        g = getattr(w, "_dtg_grad", None)
        if not tp.use_kernels:
            dxf = tp.all_gather_rows(dx_local.contiguous())           # [T, H]
            dcols = dxf[:, tp.rank * Hl:(tp.rank + 1) * Hl]
            dw = torch.zeros_like(w, dtype=torch.float32)
            dw.index_add_(0, ids, dcols.float())
            return None, _route_dw(w, dw.to(w.dtype)), None
        C = _ext.load()
        tp.dx0.local.view(tp.rpp, tp.H).copy_(dx_local)
        tp.barrier()
        # summed in fp32 and rounded once per row; overwrite mode (the first write this step) zeroes absent rows
        acc = getattr(w, "_dtg_writes", 0) > 0
        w._dtg_writes = getattr(w, "_dtg_writes", 0) + 1
        C.tp_embed_bwd(ids, tp.dx0.ptrs, g, tp.rpp, tp.H, tp.rank, acc)
        return None, None, None


class _VocabParallelCE(torch.autograd.Function):
    """mean CE over the full vocabulary from vocabulary-sharded logits [T, V/t]."""

    @staticmethod
    def forward(ctx, logits, targets, tp: TPContext, v0):
        targets = targets.contiguous()
        if not tp.use_kernels:
            lf = logits.float()
            m = lf.max(dim=-1).values
            gm = m.clone()
            if tp.t > 1:
                dist.all_reduce(gm, op=dist.ReduceOp.MAX, group=tp.pg)
            se = (lf - gm[:, None]).exp().sum(-1)
            tl = torch.zeros_like(se)
            loc = targets - v0
            mine = (targets >= 0) & (loc >= 0) & (loc < logits.shape[1])
            tl[mine] = lf[mine, loc[mine]]
            if tp.t > 1:
                dist.all_reduce(se, group=tp.pg)
                dist.all_reduce(tl, group=tp.pg)
            lse = gm + se.log()
            valid = targets >= 0
            nv = valid.sum().clamp(min=1)
            loss = ((lse - tl) * valid).sum() / nv
            p = (lf - lse[:, None]).exp()
            p[mine, loc[mine]] -= 1
            p = p * (valid[:, None] / nv)
            ctx.save_for_backward(p.to(logits.dtype))
            return loss
        C = _ext.load()
        T = logits.shape[0]
        stats = tp.stats.local[: T * 4]
        C.vp_ce_stats(logits, targets, stats, v0)
        tp.barrier()
        loss = C.vp_ce_grad(logits, targets, tp.stats.ptrs, v0)   # logits storage now holds dlogits
        ctx.save_for_backward(logits.detach())
        return loss

    @staticmethod
    def backward(ctx, dloss):
        (dlogits,) = ctx.saved_tensors
        if dlogits.is_cuda:
            _ext.load().scale_inplace(dlogits, dloss.reshape(1).float())
            return dlogits, None, None, None
        return dlogits * dloss, None, None, None


# ------------------------------------------------------------------------------------------------
# model / layer forward under tensor parallelism
# ------------------------------------------------------------------------------------------------
class TensorParallelRuntime:
    """Installed as ``model.tp`` (and so ``layer.tp``): owns the TP forward of the Llama model."""

    def __init__(self, ctx: TPContext):
        self.ctx = ctx

    def layer_forward(self, layer, x, residual, cos, sin):
        """x, residual: sequence shards [T/t, H]; returns (mlp_out_local, residual_local)."""
        tp = self.ctx
        att, mlp = layer.self_attn, layer.mlp
        y, h = layer.input_layernorm(x, residual)
        w, owner = layer.fused_weight("qkv")
        b, b_owner = layer.fused_weight("qkv_bias")
        qkv = _ColumnParallelLinear.apply(y, w, owner, tp, 2 * layer.layer_idx, b, b_owner)
        S = cos.shape[-2]   # the tables are [S, d/2], or [B, S, d/2] from position ids
        a = att.attend(qkv.view(-1, S, qkv.shape[-1]), cos, sin).flatten(0, 1)
        h2 = _RowParallelLinear.apply(a, att.o_proj.weight, att.o_proj.weight, tp, h)   # residual add fused
        y2, _ = layer.post_attention_layernorm(h2, None)
        w, owner = layer.fused_weight("gate_up")
        gu = _ColumnParallelLinear.apply(y2, w, owner, tp, 2 * layer.layer_idx + 1)
        act = ops.swiglu(gu)
        out = _RowParallelLinear.apply(act, mlp.down_proj.weight, mlp.down_proj.weight, tp, None)
        return out, h2

    def model_forward(self, model, input_ids, labels, cos, sin):
        tp = self.ctx
        T = input_ids.numel()
        assert T == tp.max_tokens, f"tensor-parallel buffers were sized for {tp.max_tokens} tokens, got {T}"
        y = model.decoder(input_ids, cos, sin,
                          embed=lambda ids: _HiddenParallelEmbedding.apply(ids, model.model.embed_tokens.weight, tp))
        logits = _ColumnParallelLinear.apply(y, model.lm_head.weight, model.lm_head.weight, tp, 2 * tp.n_layers)
        loss = None
        if labels is not None:
            tgt = ref.shift_labels(labels).reshape(-1)
            v0 = tp.rank * model.lm_head.weight.shape[0]
            loss = _VocabParallelCE.apply(logits, tgt, tp, v0)
            logits = None
        return SimpleNamespace(loss=loss, logits=logits)
