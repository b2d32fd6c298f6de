"""Flat parameter / gradient buffers.

Every engine in this package (single GPU, DDP, ZeRO-1, FSDP, TP, 2-D) keeps a *group* of
parameters (one decoder layer, the embedding, the head) in ONE contiguous buffer, with a
second contiguous buffer for its gradients:

  * the wgmma wgrad GEMM writes straight into the gradient view, so there is no autograd
    accumulation pass and no bucket copy (what torch DDP needs ``gradient_as_bucket_view``
    and a C++ Reducer for; reference ``02-distributed-data-parallel/train_llm.py:66-68``);
  * q|k|v and gate|up are adjacent in the buffer, so the fused projections cost nothing;
  * AdamW is one kernel launch per group over the flat range;
  * when the buffers come from the NVLink symmetric heap (``parallel/symm.py``) peers can
    read/write them directly, which is what the fused collective kernels use instead of
    FSDP's copy-in / copy-out (SURVEY.md K11/K12).
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch
from torch import nn

ALIGN = 8  # elements; 16 bytes for bf16 -> every view stays TMA/vector-load aligned


def _round_up(x, m):
    return (x + m - 1) // m * m


class FlatGroup:
    """A named list of parameters living in one flat tensor (+ one flat grad tensor)."""

    def __init__(self, name: str, named_params: Sequence[Tuple[str, nn.Parameter]], device, dtype,
                 pad_multiple: int = ALIGN, alloc: Optional[Callable[[int, torch.dtype], torch.Tensor]] = None,
                 with_grad: bool = True, direct_write: bool = False):
        self.name = name
        self.names = [n for n, _ in named_params]
        self.params = [p for _, p in named_params]
        self.shapes = [tuple(p.shape) for p in self.params]
        self.offsets = []
        off = 0
        for p in self.params:
            self.offsets.append(off)
            off = _round_up(off + p.numel(), ALIGN)
        self.numel = off
        self.padded_numel = _round_up(max(off, pad_multiple), pad_multiple)
        self.device, self.dtype = torch.device(device), dtype
        self.direct_write = direct_write
        alloc = alloc or (lambda n, dt: torch.zeros(n, dtype=dt, device=device))
        self.param = alloc(self.padded_numel, dtype)
        self.grad = alloc(self.padded_numel, dtype) if with_grad else None
        self.fused: Dict[str, object] = {}
        self.ready_callbacks: List[Callable] = []
        with torch.no_grad():
            for p, o in zip(self.params, self.offsets):
                view = self.param[o:o + p.numel()].view(p.shape)
                if not p.is_meta:
                    view.copy_(p.data)
                    p.data = view
                else:
                    # meta-device construction (FSDP): give the parameter object real storage in place
                    torch.utils.swap_tensors(p, nn.Parameter(view, requires_grad=p.requires_grad))
                if with_grad:
                    g = self.grad[o:o + p.numel()].view(p.shape)
                    p._dtg_grad = g
                    p._dtg_writes = 0
                    p.grad = g
                p._dtg_group = self

    # -- views ----------------------------------------------------------------------------
    def index_of(self, name):
        return self.names.index(name)

    def fused_view(self, names: Sequence[str]):
        """(data, grad) 2-D views spanning adjacent 2-D parameters that share their column count."""
        idx = [self.index_of(n) for n in names]
        assert idx == list(range(idx[0], idx[0] + len(idx))), "fused parameters must be adjacent"
        cols = self.shapes[idx[0]][1]
        rows = 0
        for i in idx:
            assert self.shapes[i][1] == cols
            assert self.offsets[i] == self.offsets[idx[0]] + rows * cols, "padding between fused parameters"
            rows += self.shapes[i][0]
        o = self.offsets[idx[0]]
        data = self.param[o:o + rows * cols].view(rows, cols)
        grad = self.grad[o:o + rows * cols].view(rows, cols) if self.grad is not None else None
        return data, grad

    def fused_view_1d(self, names: Sequence[str]):
        """(data, grad) 1-D views spanning adjacent 1-D parameters with no padding between them (the q|k|v bias)."""
        idx = [self.index_of(n) for n in names]
        assert idx == list(range(idx[0], idx[0] + len(idx))), "fused parameters must be adjacent"
        n = 0
        for i in idx:
            assert len(self.shapes[i]) == 1
            assert self.offsets[i] == self.offsets[idx[0]] + n, "padding between fused parameters"
            n += self.shapes[i][0]
        o = self.offsets[idx[0]]
        return self.param[o:o + n], (self.grad[o:o + n] if self.grad is not None else None)

    # -- gradient bookkeeping -----------------------------------------------------------------
    def zero_grad(self):
        """Start a new accumulation window.  With ``direct_write`` (every parameter's gradient
        is produced by a kernel that overwrites on first use) this only resets counters;
        otherwise the flat gradient is cleared for autograd's in-place accumulation."""
        for p in self.params:
            p._dtg_writes = 0
            if self.grad is not None and p.grad is None:
                p.grad = p._dtg_grad
        for f in self.fused.values():
            f._dtg_writes = 0
        if self.grad is not None and not self.direct_write:
            self.grad.zero_()

    def shard_range(self, rank: int, world: int) -> Tuple[int, int]:
        assert self.padded_numel % world == 0
        n = self.padded_numel // world
        return rank * n, (rank + 1) * n


def install_fused_views(layer, g: FlatGroup, i: int):
    """Give decoder layer ``i`` its fused weights (q|k|v, gate|up) and, with q/k/v biases, the fused q|k|v bias, as
    views of its flat group ``g``."""
    from ..models.llama import FusedWeight, LlamaDecoderLayer

    for fname, members in LlamaDecoderLayer.FUSED.items():
        data, grad = g.fused_view([f"model.layers.{i}.{m}" for m in members])
        layer._fused[fname] = g.fused[fname] = FusedWeight(data, grad)
    if layer.self_attn.q_proj.bias is not None:
        data, grad = g.fused_view_1d([f"model.layers.{i}.{m}" for m in LlamaDecoderLayer.QKV_BIAS_ORDER])
        layer._fused["qkv_bias"] = g.fused["qkv_bias"] = FusedWeight(data, grad)


def build_groups(model: nn.Module, device, dtype, world_size: int = 1, alloc=None, direct_write=None,
                 with_grad: bool = True) -> List[FlatGroup]:
    """Partition ``model`` into flat groups: ``embed``, one per decoder layer, ``head``.

    Order = order of first gradient *completion in reverse*: head is ready first in backward,
    the embedding last.  Tied embeddings collapse embed+head into the ``embed`` group.
    ``pad_multiple`` makes every group divisible into ``world_size`` 16-byte aligned shards.
    """
    from ..models.llama import LlamaDecoderLayer, LlamaForCausalLM

    pad = ALIGN * world_size * 16  # shards stay 256-byte aligned
    is_llama = isinstance(model, LlamaForCausalLM)
    if direct_write is None:
        direct_write = is_llama and torch.device(device).type == "cuda"
    groups: List[FlatGroup] = []
    seen = set()

    def mk(name, named):
        named = [(n, p) for n, p in named if id(p) not in seen]
        for _, p in named:
            seen.add(id(p))
        if not named:
            return None
        g = FlatGroup(name, named, device, dtype, pad_multiple=pad, alloc=alloc, with_grad=with_grad,
                      direct_write=direct_write)
        groups.append(g)
        return g

    core = model.model
    layers = list(core.layers)
    layer_param_ids = {id(p) for l in layers for p in l.parameters()}
    pre, post = [], []
    first_layer_seen = False
    for n, p in model.named_parameters():
        if id(p) in layer_param_ids:
            first_layer_seen = True
            continue
        (post if first_layer_seen else pre).append((n, p))
    mk("embed", pre)
    for i, layer in enumerate(layers):
        named = dict(layer.named_parameters())
        if isinstance(layer, LlamaDecoderLayer):
            assert set(named) == set(layer.flat_order), f"layer {i}: parameters outside flat_order"
            ordered = [(f"model.layers.{i}.{n}", named[n]) for n in layer.flat_order]
        else:
            prefix = "transformer.h" if hasattr(core, "h") else "model.layers"
            ordered = [(f"{prefix}.{i}.{n}", p) for n, p in named.items()]
        g = mk(f"layer{i}", ordered)
        layer._flat_group = g
        if isinstance(layer, LlamaDecoderLayer) and g is not None:
            install_fused_views(layer, g, i)
    mk("head", post)
    model._flat_groups = groups
    return groups
