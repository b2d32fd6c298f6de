"""Activation (gradient) checkpointing of decoder layers.

Reference: ``--checkpoint-activations`` -> ``apply_activation_checkpointing(model, checkpoint_wrapper,
auto_wrap_policy={LlamaDecoderLayer, ...})`` applied after ``fully_shard``
(``05-training-llama-405b/train_llm.py:163-178``).  Here it is a thin autograd Function: the layer
runs without saving activations, and is re-run (same kernels, same parameters — FSDP keeps them
unsharded through the layer's backward) when its gradient is needed.  Parameter gradients produced by
the recomputed graph go straight into the flat gradient buffers as usual.
"""
from __future__ import annotations

import torch


class _CheckpointLayer(torch.autograd.Function):
    @staticmethod
    def forward(ctx, layer, cos, sin, doc_start, x, residual):
        ctx.layer, ctx.cos, ctx.sin, ctx.doc_start = layer, cos, sin, doc_start
        ctx.has_res = residual is not None
        ctx.save_for_backward(x, *([residual] if residual is not None else []))
        with torch.no_grad():
            out, res = layer(x, residual, cos, sin, doc_start)
        return out, res

    @staticmethod
    def backward(ctx, d_out, d_res):
        saved = ctx.saved_tensors
        x = saved[0].detach().requires_grad_(True)
        residual = saved[1].detach().requires_grad_(True) if ctx.has_res else None
        with torch.enable_grad():
            out, res = ctx.layer(x, residual, ctx.cos, ctx.sin, ctx.doc_start)
        outs, grads = [], []
        for o, g in ((out, d_out), (res, d_res)):
            if g is not None and o.requires_grad:
                outs.append(o)
                grads.append(g)
        torch.autograd.backward(outs, grads)
        return None, None, None, None, x.grad, (residual.grad if ctx.has_res else None)


def checkpoint_layer(layer, x, residual, cos, sin, doc_start=None):
    """``doc_start``: None or the int32 [B,S] document starts the layer's attention masks with."""
    return _CheckpointLayer.apply(layer, cos, sin, doc_start, x, residual)
