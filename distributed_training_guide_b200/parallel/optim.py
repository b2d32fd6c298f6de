"""AdamW over flat buffers.

Reference: ``torch.optim.AdamW(model.parameters(), lr=args.lr, fused=True)``
(``01-single-gpu/train_llm.py:73``) — betas (0.9, 0.999), eps 1e-8, weight-decay 1e-2,
optimizer states in the parameter dtype (bf16, no fp32 master copy; SURVEY.md C15).  Here the
update is ONE hand-written kernel launch per flat group (``csrc/adamw.cu``) instead of ATen's
multi-tensor-apply, and the same kernel body is reused inside the fused
reduce-scatter+AdamW(+all-gather) NVLink kernels of the ZeRO-1 / FSDP engines.

``FlatAdamW`` subclasses ``torch.optim.Optimizer`` so LR schedulers, ``state_dict`` /
``load_state_dict`` and ``zero_grad`` behave as usual.  ``shard=(rank, world)`` restricts the
update (and the optimizer state) to this rank's 1/world slice of every group.

``max_grad_norm`` clips the gradients by their global L2 norm first (``torch.nn.utils.clip_grad_norm_``
semantics, ``ref.clip_coefficient``); ``last_grad_norm`` then holds the pre-clip norm of the last step.  On CUDA
the data-parallel engine computes both on the device (``csrc/grad_clip.cu``); here is the reference path.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch

from .. import _ext
from ..ops import reference as ref
from .flat import FlatGroup


class FlatAdamW(torch.optim.Optimizer):
    def __init__(self, groups: List[FlatGroup], lr=3e-5, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2,
                 shard: Optional[Tuple[int, int]] = None, state_dtype=None, grad_scale: float = 1.0,
                 state_device=None, max_grad_norm: Optional[float] = None):
        self.flat_groups = groups
        self.shard = shard
        self.grad_scale = grad_scale
        if max_grad_norm is not None and not max_grad_norm > 0:
            raise ValueError(f"max_grad_norm must be > 0, got {max_grad_norm}")
        self.max_grad_norm = max_grad_norm
        #: pre-clip global gradient norm of the last step (fp32 tensor; None while clipping is off)
        self.last_grad_norm = None
        #: set by engines that apply the update inside their fused collective kernels
        self.external_step = None
        params = [g.param for g in groups]
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        for g in groups:
            lo, hi = self.range_of(g)
            dt = state_dtype or g.param.dtype
            dev = state_device or g.param.device
            self.state[g.param] = {
                "step": 0,
                "exp_avg": torch.zeros(hi - lo, dtype=dt, device=dev),
                "exp_avg_sq": torch.zeros(hi - lo, dtype=dt, device=dev),
            }

    def range_of(self, g: FlatGroup):
        if self.shard is None:
            return 0, g.padded_numel
        return g.shard_range(*self.shard)

    @property
    def lr(self):
        return self.param_groups[0]["lr"]

    def hyper(self):
        pg = self.param_groups[0]
        return pg["lr"], pg["betas"][0], pg["betas"][1], pg["eps"], pg["weight_decay"]

    @torch.no_grad()
    def step_group(self, g: FlatGroup, coef=None):
        """AdamW on this rank's range of one group (kernel on CUDA, reference math on CPU).  ``coef``: gradient
        clipping factor (reference path only; on CUDA the clipped update runs in ``csrc/grad_clip.cu``)."""
        st = self.state[g.param]
        st["step"] += 1
        lr, b1, b2, eps, wd = self.hyper()
        lo, hi = self.range_of(g)
        p, gr = g.param[lo:hi], g.grad[lo:hi]
        if _ext.use_cuda_kernel("adamw", p, gr, st["exp_avg"]):
            if coef is not None:
                raise RuntimeError("the clipped AdamW update on CUDA runs in DataParallelEngine (csrc/grad_clip.cu)")
            _ext.load().adamw_flat(p, gr, st["exp_avg"], st["exp_avg_sq"], lr, b1, b2, eps, wd, st["step"],
                                   self.grad_scale)
        else:
            ref.adamw_step(p, gr, st["exp_avg"], st["exp_avg_sq"], lr, b1, b2, eps, wd, st["step"], self.grad_scale,
                           coef=coef)

    @torch.no_grad()
    def global_grad_norm(self):
        """Reference math: the L2 norm of the full gradients as AdamW consumes them (times ``grad_scale``), over each
        parameter element once (never the padding of a flat group), summed in fp64; an fp32 tensor."""
        total = torch.zeros((), dtype=torch.float64, device=self.flat_groups[0].grad.device)
        for g in self.flat_groups:
            for o, shape in zip(g.offsets, g.shapes):
                n = 1
                for d in shape:
                    n *= d
                total += (g.grad[o:o + n].double() * self.grad_scale).square().sum()
        return total.sqrt().float()

    @torch.no_grad()
    def clip_coefficient(self):
        """Compute ``last_grad_norm`` and return the clip factor of this step (None while clipping is off)."""
        if self.max_grad_norm is None:
            return None
        self.last_grad_norm = self.global_grad_norm()
        return ref.clip_coefficient(self.last_grad_norm, self.max_grad_norm)

    @torch.no_grad()
    def step(self, closure=None):
        if self.external_step is not None:
            return self.external_step()
        coef = self.clip_coefficient()
        for g in self.flat_groups:
            self.step_group(g, coef)

    def zero_grad(self, set_to_none: bool = True):
        # gradients live permanently in the flat buffers; "zeroing" = opening a new window
        for g in self.flat_groups:
            g.zero_grad()
