"""Op layer: every hot op of the Llama training step as an ``autograd.Function``.

On CUDA tensors each op calls a hand-written sm_90a kernel from the in-tree
extension (``csrc/``): wgmma/TMA GEMM (fwd / dgrad / wgrad) in bf16 and, for
``fp8_linear``, in fp8 with its amax and cast-transpose kernels, wgmma
flash-attention, fused residual-add+RMSNorm and norm-then-add (OLMo 2), in-place RoPE on the fused qkv buffer
(after Qwen3's per-head or OLMo 2's full-width QK-norm in the same kernel; partial rotary for GPT-NeoX), SwiGLU,
fused residual-add+LayerNorm and GELU-tanh (StarCoder2), GPT-NeoX's dual LayerNorm, exact GELU and parallel-residual
output GEMMs, in-place
softmax-cross-entropy, embedding gather / scatter-add and flat AdamW.  On CPU tensors the same Functions run the reference math in
``ops/reference.py`` (chapter 01's CPU config and the gloo tests).

Replaces what the reference obtains implicitly from cuBLAS / SDPA / flash-attn /
ATen / Inductor (SURVEY.md §2.4, K1-K10).

Weight-gradient protocol: a parameter may carry ``_dtg_grad`` (a view into a flat,
possibly NVLink-symmetric, gradient buffer).  wgrad kernels then write (first use
after ``zero_grad``) or accumulate (later uses / micro-batches) straight into that
view and the Function returns ``None`` for the weight, so autograd never allocates
or copies a gradient.  ``parallel/flat.py`` owns those buffers.
"""
from __future__ import annotations

import math

import torch

from .. import _ext
from . import reference as ref

__all__ = [
    "linear", "fused_linear", "rms_norm", "add_rms_norm", "rms_norm_add", "rope_qkv_", "qk_norm_rope_",
    "olmo_qk_norm_rope_", "attention_qkv", "document_starts", "swiglu", "cross_entropy", "layer_norm",
    "add_layer_norm", "gelu_tanh", "gelu", "layer_norm2", "parallel_out",
    "embedding", "gemm", "fp8_linear", "fp8_amax", "fp8_cast", "gemm_fp8", "bias_grad", "ref",
]


# --------------------------------------------------------------------------------------
# helpers
# --------------------------------------------------------------------------------------
# EXPERIMENTAL (DTG_WGRAD_STREAM=1, off by default): issue the weight-gradient GEMM of a linear layer on a side
# stream so that it runs next to the data-gradient GEMM of the same layer; both are persistent kernels, so the
# CTAs of one fill the SMs the other leaves idle in its last partial wave.  Engines call ``join_wgrad_stream()``
# before they publish a bucket's gradients.
_WGRAD_SIDE = {"enabled": bool(__import__("os").environ.get("DTG_WGRAD_STREAM")), "stream": None, "dirty": False}


def _wgrad_stream(device):
    st = _WGRAD_SIDE
    if st["stream"] is None:
        st["stream"] = torch.cuda.Stream(device=device)
    return st["stream"]


def join_wgrad_stream():
    """Make the current stream wait for weight gradients issued on the side stream (no-op when the feature is off)."""
    st = _WGRAD_SIDE
    if st["dirty"]:
        torch.cuda.current_stream().wait_stream(st["stream"])
        st["dirty"] = False


def _emit_weight_grad(param, compute_into, shape_like):
    """Route a weight gradient.

    ``compute_into(out, accumulate)`` must write the gradient into ``out`` (a tensor of
    the parameter's shape), adding to it when ``accumulate``.  Returns the tensor to hand
    back to autograd (``None`` when it went into the flat buffer).
    """
    buf = getattr(param, "_dtg_grad", None)
    if buf is not None:
        n = getattr(param, "_dtg_writes", 0)
        compute_into(buf, n > 0)
        param._dtg_writes = n + 1
        hook = getattr(param, "_dtg_ready_hook", None)
        if hook is not None:
            hook(param)
        return None
    out = torch.empty_like(shape_like)
    compute_into(out, False)
    return out


def gemm(a, b, out=None, trans_a=False, trans_b=False, accumulate=False, bias=None):
    """out[M,N] (+)= op(a) @ op(b) (+ bias) on the wgmma GEMM (bf16 in, fp32 accumulate in registers).

    ``op(a)`` is ``a`` ([M,K]) or ``a.T`` when ``trans_a`` (a given as [K,M]);
    ``op(b)`` is ``b`` ([K,N]) or ``b.T`` when ``trans_b`` (b given as [N,K]).
    ``bias`` ([N] bf16, forward layout and overwrite mode only) is added to the fp32 accumulators before the one
    rounding to bf16, in the kernel's epilogue.
    """
    M = a.shape[1] if trans_a else a.shape[0]
    N = b.shape[0] if trans_b else b.shape[1]
    if out is None:
        out = torch.empty(M, N, dtype=a.dtype, device=a.device)
        accumulate = False
    if _ext.use_cuda_kernel("gemm", a, b, out):
        if bias is None:
            _ext.load().gemm(a, b, out, trans_a, trans_b, accumulate)
        else:
            _ext.load().gemm(a, b, out, trans_a, trans_b, accumulate, bias=bias)
    else:
        A = a.t() if trans_a else a
        Bm = b.t() if trans_b else b
        r = (A.float() @ Bm.float())
        if bias is not None:
            r = r + bias.float()
        if accumulate:
            out.add_(r.to(out.dtype))
        else:
            out.copy_(r.to(out.dtype))
    return out


def bias_grad(dy):
    """fp32 [N] column sums of ``dy`` [T, N] (the gradient of a bias added to every row).  bf16 CUDA tensors run the
    sm_90a kernel: per-CTA fp32 partial rows summed in a fixed order, no atomics, so two runs are bit-identical."""
    if _ext.use_cuda_kernel("gemm", dy) and dy.dtype == torch.bfloat16:
        return _ext.load().bias_grad(dy)
    return dy.float().sum(0)


def _emit_bias_grad(bias_param, dy2, bias):
    """The bias gradient of a linear op from its 2-D output gradient, routed like a norm gain's (overwrite on the
    first write of a step, accumulate after it)."""
    if bias_param is None:
        return None
    return _emit_weight_grad(bias_param, _norm_dw_into(bias_grad(dy2)), bias)


# --------------------------------------------------------------------------------------
# linear
# --------------------------------------------------------------------------------------
class _Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, w_param, bias=None, bias_param=None):
        # x: [..., K], w: [N, K]; w_param is the nn.Parameter that owns the grad-buffer hooks; bias: None or [N],
        # added in the GEMM's epilogue, with bias_param (or the bias itself) owning its gradient routing
        x2 = x.reshape(-1, x.shape[-1])
        ctx.save_for_backward(x2, w)
        ctx.w_param = w_param if w_param is not None else w
        ctx.bias = bias
        ctx.bias_param = (bias_param if bias_param is not None else bias) if bias is not None else None
        ctx.x_shape = x.shape
        gs = getattr(ctx.w_param, "_dtg_gather", None)   # FSDP: the weight may still have to be gathered
        if gs is not None and x2.is_cuda and gs.pending():
            y = gs.gemm(x2 if x2.is_contiguous() else x2.contiguous(), True, bias)   # unshard fused into this GEMM
        else:
            y = gemm(x2, w, trans_b=True, bias=bias)
        return y.view(*x.shape[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x2, w = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        dx, dw = _linear_grads(dy2, x2, w, ctx.w_param, ctx.x_shape, ctx.needs_input_grad[0],
                               ctx.needs_input_grad[1])
        db = _emit_bias_grad(ctx.bias_param, dy2, ctx.bias)
        return dx, dw, None, db, None


def _linear_grads(dy2, x2, w, w_param, x_shape, need_dx, need_dw):
    """(dx, dw) of ``y = x @ w.T`` from the 2-D output gradient ``dy2``: the dgrad GEMM (re-gathering an FSDP weight
    inside it while its gather is pending) and the wgrad GEMM routed through ``_emit_weight_grad``."""
    dx = None
    if need_dx:
        gs = getattr(w_param, "_dtg_gather", None)
        if gs is not None and dy2.is_cuda and gs.pending():
            dx = gs.gemm(dy2, False).view(x_shape)   # FSDP: re-gather the weight inside the dgrad GEMM
        else:
            dx = gemm(dy2, w).view(x_shape)  # [T,N] @ [N,K]
    dw = None
    if need_dw or getattr(w_param, "_dtg_grad", None) is not None:
        side = _WGRAD_SIDE["enabled"] and dy2.is_cuda and getattr(w_param, "_dtg_grad", None) is not None
        if side:
            cur, ss = torch.cuda.current_stream(), _wgrad_stream(dy2.device)
            ss.wait_stream(cur)               # dy2 / x2 were produced on the compute stream
            dy2.record_stream(ss)             # keep the caching allocator from recycling them too early
            x2.record_stream(ss)
            with torch.cuda.stream(ss):
                dw = _emit_weight_grad(w_param,
                                       lambda out, acc: gemm(dy2, x2, out=out, trans_a=True, accumulate=acc), w)
            _WGRAD_SIDE["dirty"] = True
        else:
            dw = _emit_weight_grad(
                w_param,
                lambda out, acc: gemm(dy2, x2, out=out, trans_a=True, accumulate=acc),  # dy^T @ x
                w,
            )
    return dx, dw


def linear(x, w, bias=None):
    """y = x @ w.T (+ bias).  bf16 CUDA tensors run the wgmma GEMM, the bias in its epilogue."""
    if _ext.use_cuda_kernel("gemm", x, w) and x.dtype == torch.bfloat16:
        if bias is None:
            return _Linear.apply(x, w, w)
        return _Linear.apply(x, w, w, bias, bias)
    return ref.linear(x, w, bias)


def fused_linear(x, w, owner=None, bias=None, bias_owner=None):
    """``linear`` over a fused weight (q|k|v or gate|up).  ``owner`` is the
    ``models.llama.FusedWeight`` carrying the flat-gradient view, or None when ``w`` is an
    ordinary autograd tensor (e.g. a ``torch.cat`` of the individual parameters).  ``bias`` /
    ``bias_owner``: the fused bias (q|k|v, Qwen2) and what carries its flat-gradient view, likewise."""
    if _ext.use_cuda_kernel("gemm", x, w) and x.dtype == torch.bfloat16:
        if bias is None:
            return _Linear.apply(x, w, owner if owner is not None else w)
        return _Linear.apply(x, w, owner if owner is not None else w, bias, bias_owner)
    return ref.linear(x, w, bias)


# --------------------------------------------------------------------------------------
# fp8 linear (per-tensor current scaling; x and W in e4m3, dy in e5m2)
# --------------------------------------------------------------------------------------
def fp8_amax(t):
    """max |t| of a 2-D bf16 tensor as a one-element fp32 tensor on its device."""
    if _ext.use_cuda_kernel("fp8", t):
        return _ext.load().fp8_amax(t)
    return t.float().abs().max().reshape(1)


def fp8_cast(t, dtype, rowwise=True, transposed=True, amax=None):
    """``(t8, t8_T, scale_inv)`` of a 2-D bf16 tensor quantised to ``dtype`` (see ``ref.fp8_quantize``): the
    row-major copy and / or its transpose (None when not asked for) and the one-element fp32 dequantisation scale,
    which stays on the device.  ``amax`` (from ``fp8_amax``) is computed when not given.  CUDA: the amax and
    cast-transpose kernels."""
    if amax is None:
        amax = fp8_amax(t)
    if _ext.use_cuda_kernel("fp8", t):
        return _ext.load().fp8_cast_transpose(t, amax, dtype == torch.float8_e5m2, rowwise, transposed)
    t8, scale_inv = ref.fp8_quantize(t, dtype, amax)
    return (t8 if rowwise else None), (t8.t().contiguous() if transposed else None), scale_inv


def gemm_fp8(a8, scale_inv_a, b8, scale_inv_b, out=None, accumulate=False, out_dtype=torch.bfloat16, bias=None):
    """out[M,N] (+)= scale_inv_a * scale_inv_b * a8[M,K] @ b8[N,K].T (+ bias) with fp32 accumulation.  a8 is e4m3 or
    e5m2, b8 e4m3, both with K contiguous; ``out`` may be a strided view (of a flat gradient).  ``bias`` ([N] bf16,
    e4m3 a8, overwrite mode) is added in the epilogue: bf16(acc * scale + bias) with one rounding."""
    if out is None:
        out = torch.empty(a8.shape[0], b8.shape[0], dtype=out_dtype, device=a8.device)
        accumulate = False
    if _ext.use_cuda_kernel("fp8", a8, b8, out):
        if bias is None:
            _ext.load().gemm_fp8(a8, b8, out, scale_inv_a, scale_inv_b, accumulate)
        else:
            _ext.load().gemm_fp8(a8, b8, out, scale_inv_a, scale_inv_b, accumulate, bias=bias)
    else:
        r = ref.fp8_gemm(a8, scale_inv_a, b8, scale_inv_b)
        if bias is not None:
            r = r + bias.float()
        out.copy_((out.float() + r) if accumulate else r)
    return out


class _FP8Linear(torch.autograd.Function):
    """y = x @ W.T with every GEMM in fp8: forward X8 . W8^T, dgrad dY8 . (W8^T)^T, wgrad (dY8^T) . (X8^T)^T.  The
    fp8 GEMM takes K-major operands only, so forward casts x into both layouts and keeps the transposed copy (1 byte
    per element) for backward instead of the bf16 input; backward casts dy into both layouts.  W8^T is cast again in
    backward from the weight, which does not change before its gradient is computed, with the amax forward measured,
    so it is bit-identical to the forward's quantisation; keeping it from forward instead would hold 1 byte per
    parameter through the step (6.5 GB for Llama-2-7B, more than an 80 GB H100 has left at S 4096)."""

    @staticmethod
    def forward(ctx, x, w, w_param, bias=None, bias_param=None):
        x2 = x.reshape(-1, x.shape[-1])
        x8, x8t, sx = fp8_cast(x2, torch.float8_e4m3fn)
        amax_w = fp8_amax(w)
        w8, _, sw = fp8_cast(w, torch.float8_e4m3fn, transposed=False, amax=amax_w)
        if bias is None:
            y = gemm_fp8(x8, sx, w8, sw, out_dtype=x.dtype)
        else:
            y = gemm_fp8(x8, sx, w8, sw, out_dtype=x.dtype, bias=bias)
        ctx.save_for_backward(x8t, sx, w, amax_w)
        ctx.w_param = w_param
        ctx.bias = bias
        ctx.bias_param = (bias_param if bias_param is not None else bias) if bias is not None else None
        ctx.x_shape = x.shape
        return y.view(*x.shape[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, dy):
        x8t, sx, w, amax_w = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1])
        if not dy2.is_contiguous():
            dy2 = dy2.contiguous()
        dy8, dy8t, sdy = fp8_cast(dy2, torch.float8_e5m2, rowwise=ctx.needs_input_grad[0])
        dx, dw = _fp8_linear_grads(dy8, dy8t, sdy, x8t, sx, w, amax_w, ctx.w_param, ctx.x_shape, dy.dtype,
                                   ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        db = _emit_bias_grad(ctx.bias_param, dy2, ctx.bias)   # from the bf16 dy, not its fp8 copy
        return dx, dw, None, db, None


def _fp8_linear_grads(dy8, dy8t, sdy, x8t, sx, w, amax_w, w_param, x_shape, dtype, need_dx, need_dw):
    """(dx, dw) of an fp8 linear from the e5m2 output gradient (both layouts) and the forward's saved transposed
    e4m3 input: the dgrad GEMM against W8^T re-cast with the forward's amax, and the wgrad GEMM routed through
    ``_emit_weight_grad``."""
    dx = None
    if need_dx:
        _, w8t, sw = fp8_cast(w, torch.float8_e4m3fn, rowwise=False, amax=amax_w)
        dx = gemm_fp8(dy8, sdy, w8t, sw, out_dtype=dtype).view(x_shape)  # [T,N] . [K,N]^T
    dw = None
    if need_dw or getattr(w_param, "_dtg_grad", None) is not None:
        dw = _emit_weight_grad(
            w_param,
            lambda out, acc: gemm_fp8(dy8t, sdy, x8t, sx, out=out, accumulate=acc),  # [N,T] . [K,T]^T
            w_param,
        )
    return dx, dw


def fp8_linear(x, w, owner=None, bias=None, bias_owner=None):
    """``linear`` with fp8 GEMMs (forward, dgrad and wgrad).  ``owner`` is what carries the flat-gradient view: the
    ``models.llama.FusedWeight`` of a fused weight, or the parameter itself; None when ``w`` is an ordinary autograd
    tensor.  ``bias`` / ``bias_owner`` likewise for a bias added in the forward GEMM's epilogue; its gradient is
    summed from the bf16 output gradient.  CPU tensors run the same quantisation through ``ops/reference.py``."""
    if bias is None:
        return _FP8Linear.apply(x, w, owner if owner is not None else w)
    return _FP8Linear.apply(x, w, owner if owner is not None else w, bias, bias_owner)


# --------------------------------------------------------------------------------------
# parallel-residual branch (GPT-NeoX): x = attn @ Wd^T + act @ W4^T + bd + b4 in one [T, H] buffer
# --------------------------------------------------------------------------------------
def _bias_sum(bd, b4):
    return (bd.float() + b4.float()).to(bd.dtype)


def _emit_shared_bias_grad(dy2, bd, b4):
    """One column sum of ``dy2`` is the gradient of both biases; each is routed like a norm gain's."""
    db32 = bias_grad(dy2)
    return (_emit_weight_grad(bd, _norm_dw_into(db32), bd), _emit_weight_grad(b4, _norm_dw_into(db32), b4))


class _ParallelOut(torch.autograd.Function):
    """The dense GEMM writes ``bf16(attn @ Wd^T + bf16(bd + b4))`` (bias epilogue, overwrite mode); the
    down-projection GEMM adds ``act @ W4^T`` into the same buffer (accumulate mode).  While an FSDP weight's gather is
    pending, its ``_GatherSpec.gemm`` runs instead and the down-projection's product is added."""

    @staticmethod
    def forward(ctx, attn, act, wd, w4, bd, b4):
        a2 = attn.reshape(-1, attn.shape[-1])
        m2 = act.reshape(-1, act.shape[-1])
        bias = _bias_sum(bd, b4)
        gs = getattr(wd, "_dtg_gather", None)
        if gs is not None and gs.pending():
            out = gs.gemm(a2 if a2.is_contiguous() else a2.contiguous(), True, bias)
        else:
            out = gemm(a2, wd, trans_b=True, bias=bias)
        gs = getattr(w4, "_dtg_gather", None)
        if gs is not None and gs.pending():
            out.add_(gs.gemm(m2 if m2.is_contiguous() else m2.contiguous(), True))
        else:
            gemm(m2, w4, out=out, trans_b=True, accumulate=True)
        ctx.save_for_backward(a2, m2, wd, w4)
        ctx.params = (bd, b4)
        ctx.shapes = (attn.shape, act.shape)
        return out.view(*attn.shape[:-1], wd.shape[0])

    @staticmethod
    def backward(ctx, dy):
        a2, m2, wd, w4 = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1]).contiguous()
        need = ctx.needs_input_grad
        dattn, dwd = _linear_grads(dy2, a2, wd, wd, ctx.shapes[0], need[0], need[2])
        dact, dw4 = _linear_grads(dy2, m2, w4, w4, ctx.shapes[1], need[1], need[3])
        return (dattn, dact, dwd, dw4) + _emit_shared_bias_grad(dy2, *ctx.params)


class _FP8ParallelOut(torch.autograd.Function):
    """``_ParallelOut`` with both GEMMs in fp8 (``_FP8Linear``'s scheme): the dense GEMM with the summed bias in its
    epilogue, the down-projection with ``gemm_fp8(..., accumulate=True)``.  The output gradient is cast to e5m2 once
    for both weights."""

    @staticmethod
    def forward(ctx, attn, act, wd, w4, bd, b4):
        a2 = attn.reshape(-1, attn.shape[-1])
        m2 = act.reshape(-1, act.shape[-1])
        a8, a8t, sa = fp8_cast(a2, torch.float8_e4m3fn)
        m8, m8t, sm = fp8_cast(m2, torch.float8_e4m3fn)
        amax_d, amax_4 = fp8_amax(wd), fp8_amax(w4)
        wd8, _, swd = fp8_cast(wd, torch.float8_e4m3fn, transposed=False, amax=amax_d)
        w48, _, sw4 = fp8_cast(w4, torch.float8_e4m3fn, transposed=False, amax=amax_4)
        out = gemm_fp8(a8, sa, wd8, swd, out_dtype=attn.dtype, bias=_bias_sum(bd, b4))
        gemm_fp8(m8, sm, w48, sw4, out=out, accumulate=True)
        ctx.save_for_backward(a8t, sa, m8t, sm, wd, w4, amax_d, amax_4)
        ctx.params = (bd, b4)
        ctx.shapes = (attn.shape, act.shape)
        return out.view(*attn.shape[:-1], wd.shape[0])

    @staticmethod
    def backward(ctx, dy):
        a8t, sa, m8t, sm, wd, w4, amax_d, amax_4 = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1]).contiguous()
        need = ctx.needs_input_grad
        dy8, dy8t, sdy = fp8_cast(dy2, torch.float8_e5m2, rowwise=need[0] or need[1])
        dattn, dwd = _fp8_linear_grads(dy8, dy8t, sdy, a8t, sa, wd, amax_d, wd, ctx.shapes[0], dy.dtype, need[0],
                                       need[2])
        dact, dw4 = _fp8_linear_grads(dy8, dy8t, sdy, m8t, sm, w4, amax_4, w4, ctx.shapes[1], dy.dtype, need[1],
                                      need[3])
        return (dattn, dact, dwd, dw4) + _emit_shared_bias_grad(dy2, *ctx.params)


def parallel_out(attn, act, wd, w4, bd, b4, fp8=False):
    """GPT-NeoX's layer branch ``attn @ Wd^T + act @ W4^T + bd + b4`` (attention dense + MLP down-projection) as one
    [..., H] tensor.  bf16 CUDA tensors run two wgmma GEMMs into one buffer, with no elementwise pass: the first with
    ``bf16(bd + b4)`` in its epilogue, the second accumulating; backward sums the output gradient once for both
    biases.  ``fp8``: both GEMMs in fp8 (CPU tensors run the same quantisation through ``ops/reference.py``)."""
    if fp8:
        return _FP8ParallelOut.apply(attn, act, wd, w4, bd, b4)
    if _ext.use_cuda_kernel("gemm", attn, act, wd, w4) and attn.dtype == torch.bfloat16:
        return _ParallelOut.apply(attn, act, wd, w4, bd, b4)
    return ref.linear(attn, wd, bd) + ref.linear(act, w4, b4)


# --------------------------------------------------------------------------------------
# Row norms: RMSNorm and LayerNorm (+ fused residual add), OLMo 2's norm-then-add
# --------------------------------------------------------------------------------------
def _norm_dw_into(dw32):
    def into(out, acc):
        if acc:
            out.add_(dw32.to(out.dtype))
        else:
            out.copy_(dw32)
    return into


def _rows(t):
    return t.reshape(-1, t.shape[-1])


def _norm_grads(params, d32):
    """Route the fp32 gain / bias gradients ``d32[i]`` of ``params[i]`` through ``_emit_weight_grad`` (None for an
    absent parameter)."""
    return tuple(None if p is None else _emit_weight_grad(p, _norm_dw_into(d32[i]), p) for i, p in enumerate(params))


class _Norm(torch.autograd.Function):
    """y = norm(h) * w (+ b) with h = x, or (y, h) with h = x + r rounded to bf16, in one pass over the activations.
    ``b`` None: RMSNorm, else LayerNorm; ``r`` None: no residual.  Backward: dx = the norm's backward + dh, the
    gradient of both x and r when h is an output."""

    @staticmethod
    def forward(ctx, x, r, w, b, eps):
        C = _ext.load()
        x2, r2 = _rows(x), (_rows(r) if r is not None else None)
        if b is None:
            y, rstd, h = C.rmsnorm_fwd(x2, w, float(eps), r2)
            stats = (rstd,)
        else:
            y, h, mean, rstd = C.layernorm_fwd(x2, r2, w, b, float(eps))
            stats = (mean, rstd)
        ctx.save_for_backward(x2 if h is None else h, w, *stats)
        ctx.shape = x.shape
        ctx.params = (w, b)
        if h is None:
            return y.view(x.shape)
        return y.view(x.shape), h.view(x.shape)

    @staticmethod
    def backward(ctx, dy, dh=None):
        C = _ext.load()
        h, w, *stats = ctx.saved_tensors
        dy2 = _rows(dy).contiguous()
        dh2 = _rows(dh).contiguous() if dh is not None else None
        bwd = C.rmsnorm_bwd if ctx.params[1] is None else C.layernorm_bwd
        dx, *d32 = bwd(dy2, h, w, *stats, dh2)
        dx = dx.view(ctx.shape)
        return (dx, dx if dh is not None else None) + _norm_grads(ctx.params, d32) + (None,)


def rms_norm(x, w, eps):
    if _ext.use_cuda_kernel("rmsnorm", x, w) and x.dtype == torch.bfloat16:
        return _Norm.apply(x.contiguous(), None, w, None, eps)
    return ref.rms_norm(x, w, eps)


def add_rms_norm(x, residual, w, eps):
    """Fused ``h = x + residual; y = rmsnorm(h) * w`` -> (y, h)."""
    if _ext.use_cuda_kernel("rmsnorm", x, residual, w) and x.dtype == torch.bfloat16:
        return _Norm.apply(x.contiguous(), residual.contiguous(), w, None, eps)
    return ref.add_rms_norm(x, residual, w, eps)


class _RMSNormAdd(torch.autograd.Function):
    """h = r + rmsnorm(x) * w in one pass: the normalised branch is never stored.  Backward: dr = dh, and dx / dw are
    the RMSNorm backward of x (rmsnorm_bwd with h := x, no residual gradient)."""

    @staticmethod
    def forward(ctx, x, r, w, eps):
        C = _ext.load()
        x2 = _rows(x)
        h, rstd = C.rmsnorm_add_fwd(x2, _rows(r), w, float(eps))
        ctx.save_for_backward(x2, w, rstd)
        ctx.shape = x.shape
        ctx.params = (w,)
        return h.view(x.shape)

    @staticmethod
    def backward(ctx, dh):
        C = _ext.load()
        x2, w, rstd = ctx.saved_tensors
        dx, dw32 = C.rmsnorm_bwd(_rows(dh).contiguous(), x2, w, rstd, None)
        return (dx.view(ctx.shape), dh) + _norm_grads(ctx.params, (dw32,)) + (None,)


def rms_norm_add(x, r, w, eps):
    """Norm-then-add (OLMo 2's post-sublayer norms): ``bf16(r + bf16(rmsnorm(x) * w))``, the gain applied in fp32 with
    one rounding (``ref.rms_norm_add``).  bf16 CUDA tensors run the sm_90a kernel, whose output is bit-identical to
    ``rmsnorm_fwd`` followed by a bf16 add; the gain gradient goes through ``_emit_weight_grad``."""
    if _ext.use_cuda_kernel("rmsnorm", x, r, w) and x.dtype == torch.bfloat16:
        return _RMSNormAdd.apply(x.contiguous(), r.contiguous(), w, eps)
    return ref.rms_norm_add(x, r, w, eps)


# --------------------------------------------------------------------------------------
# LayerNorm (+ fused residual add), StarCoder2
# --------------------------------------------------------------------------------------
def layer_norm(x, w, b, eps):
    """``y = (x - mean) * rsqrt(var + eps) * w + b`` over the last dimension with fp32 statistics and one rounding
    (ATen's bf16 ``layer_norm``).  bf16 CUDA tensors run the sm_90a kernels; the gain and bias gradients go through
    ``_emit_weight_grad`` (overwrite on the first write of a step, accumulate after it)."""
    if _ext.use_cuda_kernel("layernorm", x, w, b) and x.dtype == torch.bfloat16:
        return _Norm.apply(x.contiguous(), None, w, b, eps)
    return ref.layer_norm(x, w, b, eps)


def add_layer_norm(x, residual, w, b, eps):
    """Fused ``h = x + residual; y = layer_norm(h, w, b)`` -> (y, h), with ``h`` rounded to the input dtype before it
    is normalised."""
    if _ext.use_cuda_kernel("layernorm", x, residual, w, b) and x.dtype == torch.bfloat16:
        return _Norm.apply(x.contiguous(), residual.contiguous(), w, b, eps)
    h = x + residual
    return ref.layer_norm(h, w, b, eps), h


class _GeluTanh(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return _ext.load().gelu_tanh_fwd(x)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        return _ext.load().gelu_tanh_bwd(dy.contiguous(), x)


def gelu_tanh(x):
    """GELU with the tanh approximation (``F.gelu(x, approximate="tanh")``, StarCoder2's ``gelu_pytorch_tanh``) in
    fp32 with one rounding.  bf16 CUDA tensors run the sm_90a kernels, which keep the pre-activation for the
    backward."""
    if _ext.use_cuda_kernel("gelu", x) and x.dtype == torch.bfloat16:
        return _GeluTanh.apply(x.contiguous())
    return ref.gelu_new(x.float()).to(x.dtype)


class _Gelu(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return _ext.load().gelu_fwd(x)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        return _ext.load().gelu_bwd(dy.contiguous(), x)


def gelu(x):
    """Exact GELU, ``x/2 * (1 + erf(x / sqrt(2)))`` (``F.gelu(x)``, GPT-NeoX's ``hidden_act: "gelu"``), in fp32 with
    one rounding.  bf16 CUDA tensors run the sm_90a kernels, which keep the pre-activation for the backward."""
    if _ext.use_cuda_kernel("gelu", x) and x.dtype == torch.bfloat16:
        return _Gelu.apply(x.contiguous())
    return ref.gelu(x)


# --------------------------------------------------------------------------------------
# two LayerNorms over one residual stream (GPT-NeoX's parallel residual)
# --------------------------------------------------------------------------------------
class _LayerNorm2(torch.autograd.Function):
    """(y1, y2[, h]) = (layernorm(h) * w1 + b1, layernorm(h) * w2 + b2[, h]), h = x + r (x without r), one shared
    statistic.  Backward: one kernel for dx (+ dh as the residual gradient) and the four parameter gradients."""

    @staticmethod
    def forward(ctx, x, r, w1, b1, w2, b2, eps):
        C = _ext.load()
        x2 = _rows(x)
        r2 = _rows(r) if r is not None else None
        y1, y2, h, mean, rstd = C.layernorm2_fwd(x2, r2, w1, b1, w2, b2, float(eps))
        ctx.save_for_backward(h if h is not None else x2, w1, w2, mean, rstd)
        ctx.shape = x.shape
        ctx.params = (w1, b1, w2, b2)
        ctx.has_res = r is not None
        if h is None:
            return y1.view(x.shape), y2.view(x.shape)
        return y1.view(x.shape), y2.view(x.shape), h.view(x.shape)

    @staticmethod
    def backward(ctx, dy1, dy2, dh=None):
        C = _ext.load()
        h, w1, w2, mean, rstd = ctx.saved_tensors
        flat = lambda t: _rows(t).contiguous() if t is not None else torch.zeros_like(h)  # noqa: E731
        dh2 = _rows(dh).contiguous() if dh is not None else None
        dx, d32 = C.layernorm2_bwd(flat(dy1), flat(dy2), h, w1, w2, mean, rstd, dh2)
        dx = dx.view(ctx.shape)
        return (dx, dx if ctx.has_res else None) + _norm_grads(ctx.params, d32) + (None,)


def layer_norm2(x, r, w1, b1, w2, b2, eps):
    """GPT-NeoX's two pre-norms of one residual stream: ``h = x + r`` (rounded to the input dtype; ``x`` itself when
    ``r`` is None), then ``(layer_norm(h, w1, b1), layer_norm(h, w2, b2), h)``.  Both norms share one mean and one
    rstd.  bf16 CUDA tensors run the sm_90a kernels: one read of the row and three writes forward; y1 and y2 are
    bit-identical to ``layer_norm`` with each (w, b).  The four parameter gradients go through ``_emit_weight_grad``."""
    if _ext.use_cuda_kernel("layernorm", x, w1, b1, w2, b2) and x.dtype == torch.bfloat16:
        if r is None:
            y1, y2 = _LayerNorm2.apply(x.contiguous(), None, w1, b1, w2, b2, eps)
            return y1, y2, x
        return _LayerNorm2.apply(x.contiguous(), r.contiguous(), w1, b1, w2, b2, eps)
    return ref.layer_norm2(x, r, w1, b1, w2, b2, eps)


# --------------------------------------------------------------------------------------
# RoPE, applied in place on the q and k heads of the fused qkv activation
# --------------------------------------------------------------------------------------
class _RopeQKV(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, cos, sin, n_rot_heads, rotary_dim=None):
        # qkv: [B, S, n_total_heads, d]; the first n_rot_heads heads (q then k) are rotated
        C = _ext.load()
        ctx.save_for_backward(cos, sin)
        ctx.n_rot = n_rot_heads
        ctx.rotary_dim = rotary_dim
        C.rope_inplace(qkv, cos, sin, n_rot_heads, False, rot_dim=rotary_dim)
        # physically in place, but handed to autograd as a fresh tensor aliasing the same
        # storage: the producer GEMM never re-reads its output, so nothing observes the write
        return qkv.detach()

    @staticmethod
    def backward(ctx, dqkv):
        C = _ext.load()
        cos, sin = ctx.saved_tensors
        if not dqkv.is_contiguous():
            dqkv = dqkv.contiguous()
        C.rope_inplace(dqkv, cos, sin, ctx.n_rot, True, rot_dim=ctx.rotary_dim)  # inverse rotation, in place
        return dqkv, None, None, None, None


def rope_qkv_(qkv, cos, sin, n_rot_heads, rotary_dim=None):
    """Rotate heads [0, n_rot_heads) of ``qkv`` [B,S,heads,d] with cos/sin [S,r/2] or [B,S,r/2] (fp32), r =
    ``rotary_dim`` (None: the whole head, r = d).  A partial rotary_dim (GPT-NeoX) rotates the pairs (j, j + r/2),
    j < r/2, and leaves elements [r, d) of every head untouched; it must be a multiple of 16."""
    if rotary_dim is not None and rotary_dim == qkv.shape[-1]:
        rotary_dim = None
    if _ext.use_cuda_kernel("rope", qkv) and qkv.dtype == torch.bfloat16:
        # views produced by a GEMM are fresh tensors, in-place is safe for autograd via mark_dirty
        return _RopeQKV.apply(qkv, cos.contiguous(), sin.contiguous(), n_rot_heads, rotary_dim)
    if rotary_dim is None:
        rot = ref.rope_apply(qkv[:, :, :n_rot_heads], cos, sin)
    else:
        qk = qkv[:, :, :n_rot_heads]
        rot = torch.cat([ref.rope_apply(qk[..., :rotary_dim], cos, sin), qk[..., rotary_dim:]], dim=-1)
    return torch.cat([rot, qkv[:, :, n_rot_heads:]], dim=2)


class _QKNormRope(torch.autograd.Function):
    """QK-norm + RoPE in place on qkv's q|k heads: per head (Qwen3) or, with ``full``, over each token's whole q and k
    regions (OLMo 2)."""

    @staticmethod
    def forward(ctx, qkv, q_w, k_w, cos, sin, nh, nkv, eps, full):
        C = _ext.load()
        fwd = C.qk_norm_full_rope_fwd if full else C.qk_norm_rope_fwd
        x_save, rstd = fwd(qkv, q_w, k_w, cos, sin, nh, nkv, float(eps))
        ctx.save_for_backward(x_save, rstd, q_w, k_w, cos, sin)
        ctx.heads = (nh, nkv)
        ctx.full = full
        ctx.w_params = (q_w, k_w)
        return qkv.detach()   # in place, handed to autograd as a fresh tensor (see _RopeQKV)

    @staticmethod
    def backward(ctx, dqkv):
        C = _ext.load()
        x_save, rstd, q_w, k_w, cos, sin = ctx.saved_tensors
        if not dqkv.is_contiguous():
            dqkv = dqkv.contiguous()
        bwd = C.qk_norm_full_rope_bwd if ctx.full else C.qk_norm_rope_bwd
        dw32 = bwd(dqkv, x_save, rstd, q_w, k_w, cos, sin, *ctx.heads).view(-1)   # in place on dqkv's q|k; q then k
        nq = q_w.numel()
        dq = _emit_weight_grad(ctx.w_params[0], _norm_dw_into(dw32[:nq]), q_w)
        dk = _emit_weight_grad(ctx.w_params[1], _norm_dw_into(dw32[nq:]), k_w)
        return dqkv, dq, dk, None, None, None, None, None, None


def qk_norm_rope_(qkv, q_w, k_w, cos, sin, nh, nkv, eps):
    """Qwen3's QK-norm then RoPE on ``qkv`` [B,S,nh+2*nkv,d]: every q head is RMS-normalised over its d elements
    and scaled by ``q_w`` [d], every k head likewise with ``k_w``, with ``ref.rms_norm``'s rounding points; then
    heads [0, nh+nkv) are rotated as ``rope_qkv_`` does, with cos/sin [S,d/2] or [B,S,d/2] (fp32).  V is untouched.

    bf16 CUDA tensors with d = 128 run the sm_90a kernels in place on ``qkv``; anything else composes
    ``ref.rms_norm`` and ``ref.rope_apply``.  The kernel path keeps the pre-norm q|k heads (bf16) and one fp32 rstd
    per head for the backward: (nh + nkv) * 128 * 2 bytes per token, 42 MB per layer for Qwen3-8B (32 + 8 heads)
    at 4096 tokens.  The gain gradients go through ``_emit_weight_grad``, so flat-buffer parameters are overwritten
    on their first use in a step and accumulated on later ones."""
    if (_ext.use_cuda_kernel("qk_norm_rope", qkv, q_w, k_w) and qkv.dtype == torch.bfloat16
            and qkv.shape[-1] == 128):
        return _QKNormRope.apply(qkv, q_w, k_w, cos.contiguous(), sin.contiguous(), nh, nkv, eps, False)
    q = ref.rms_norm(qkv[:, :, :nh], q_w, eps)
    k = ref.rms_norm(qkv[:, :, nh:nh + nkv], k_w, eps)
    rot = ref.rope_apply(torch.cat([q, k], dim=2), cos, sin)
    return torch.cat([rot, qkv[:, :, nh + nkv:]], dim=2)


def olmo_qk_norm_rope_(qkv, q_w, k_w, cos, sin, nh, nkv, eps):
    """OLMo 2's full-width QK-norm then RoPE on ``qkv`` [B,S,nh+2*nkv,d]: each token's q heads are RMS-normalised
    together, over all nh*d elements, and scaled by ``q_w`` [nh*d]; its k heads likewise with ``k_w`` [nkv*d]; the
    gain is applied in fp32 with one rounding (``ref.rms_norm_one_rounding``).  Then heads [0, nh+nkv) are rotated as
    ``rope_qkv_`` does, with cos/sin [S,d/2] or [B,S,d/2] (fp32).  V is untouched.

    bf16 CUDA tensors with d = 128 run the sm_90a kernels in place on ``qkv``; anything else composes
    ``ref.rms_norm_one_rounding`` and ``ref.rope_apply``.  The kernel path keeps the pre-norm q|k heads (bf16) and
    two fp32 rstd per token for the backward.  The gain gradients go through ``_emit_weight_grad``, so flat-buffer
    parameters are overwritten on their first use in a step and accumulated on later ones."""
    if (_ext.use_cuda_kernel("qk_norm_rope", qkv, q_w, k_w) and qkv.dtype == torch.bfloat16
            and qkv.shape[-1] == 128):
        return _QKNormRope.apply(qkv, q_w, k_w, cos.contiguous(), sin.contiguous(), nh, nkv, eps, True)
    B, S, _, d = qkv.shape
    q = ref.rms_norm_one_rounding(qkv[:, :, :nh].reshape(B, S, nh * d), q_w, eps).view(B, S, nh, d)
    k = ref.rms_norm_one_rounding(qkv[:, :, nh:nh + nkv].reshape(B, S, nkv * d), k_w, eps).view(B, S, nkv, d)
    rot = ref.rope_apply(torch.cat([q, k], dim=2), cos, sin)
    return torch.cat([rot, qkv[:, :, nh + nkv:]], dim=2)


# --------------------------------------------------------------------------------------
# causal flash attention on the fused qkv buffer
# --------------------------------------------------------------------------------------
class _AttentionQKV(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qkv, nh, nkv, scale, doc_start=None, window=None):
        C = _ext.load()
        head_dim = qkv.shape[-1]
        o, lse = C.attn_fwd(qkv, nh, nkv, float(scale), doc_start=doc_start, window=window, head_dim=head_dim)
        ctx.save_for_backward(qkv, o, lse, doc_start)
        ctx.meta = (nh, nkv, scale, window, head_dim)
        return o

    @staticmethod
    def backward(ctx, do):
        C = _ext.load()
        qkv, o, lse, doc_start = ctx.saved_tensors
        nh, nkv, scale, window, head_dim = ctx.meta
        dqkv = C.attn_bwd(do.contiguous(), qkv, o, lse, nh, nkv, float(scale), doc_start=doc_start, window=window,
                          head_dim=head_dim)
        return dqkv, None, None, None, None, None


def document_starts(position_ids):
    """Document masking convention: a document starts at every token whose position id is 0, and at the first
    token of every row.  ``position_ids`` [B, S] -> int32 [B, S]: for each token, the index within its row of the
    first token of its document.  Non-decreasing along a row and never above the token's own index.  One cummax on
    the device, no host synchronisation.  The attention kernels let query q see key k iff start[q] <= k <= q."""
    B, S = position_ids.shape
    idx = torch.arange(S, device=position_ids.device, dtype=torch.int32).expand(B, S)
    is_start = position_ids == 0
    is_start[:, 0] = True
    return torch.where(is_start, idx, torch.zeros_like(idx)).cummax(dim=1).values.to(torch.int32).contiguous()


def attention_qkv(qkv, nh, nkv, scale=None, doc_start=None, window=None):
    """Causal self-attention. qkv: [B,S,nh+2*nkv,d] (q heads | k heads | v heads) -> [B,S,nh,d].
    ``doc_start`` (int32 [B,S] from ``document_starts``, or None): document masking, query q sees key k iff
    ``doc_start[q] <= k <= q``.  ``window`` (an int >= 1, or None): sliding-window attention (Mistral), query q also
    sees only the ``window`` most recent keys, ``k > q - window``; a window of S or more changes nothing.  ``scale``
    (None = 1/sqrt(d)) must be finite and > 0 on every path.  bf16 CUDA tensors with d = 64 or 128 and S a multiple
    of 128 run the sm_90a kernels."""
    d = qkv.shape[-1]
    scale = scale if scale is not None else 1.0 / math.sqrt(d)
    if isinstance(scale, bool) or not math.isfinite(scale) or scale <= 0:
        raise ValueError(f"scale must be finite and > 0 or None, got {scale!r}")
    if window is not None:
        if isinstance(window, bool) or int(window) != window or window < 1:
            raise ValueError(f"window must be an int >= 1 or None, got {window!r}")
        window = None if window >= qkv.shape[1] else int(window)
    if (_ext.use_cuda_kernel("attention", qkv) and qkv.dtype == torch.bfloat16 and d in (64, 128)
            and qkv.shape[1] % 128 == 0):
        if doc_start is not None:
            return _AttentionQKV.apply(qkv, nh, nkv, scale, doc_start.to(torch.int32).contiguous(), window)
        if window is not None:
            return _AttentionQKV.apply(qkv, nh, nkv, scale, None, window)
        return _AttentionQKV.apply(qkv, nh, nkv, scale)
    q, k, v = qkv[:, :, :nh], qkv[:, :, nh:nh + nkv], qkv[:, :, nh + nkv:]
    if qkv.is_cuda:
        # head dims other than 64 and 128 (toy configs) and sequence lengths that are not a multiple of the
        # 128-row tile are outside the sm_90a kernels' scope; use the library kernel rather than the
        # O(S^2)-memory reference
        if doc_start is not None or window is not None:
            mask = ref.document_mask(doc_start, qkv.shape[1], window, device=qkv.device)[:, None]  # [B|1, 1, S, S]
            o = torch.nn.functional.scaled_dot_product_attention(
                q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), attn_mask=mask, scale=scale,
                enable_gqa=(nh != nkv))
        else:
            o = torch.nn.functional.scaled_dot_product_attention(
                q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), is_causal=True, scale=scale,
                enable_gqa=(nh != nkv))
        return o.transpose(1, 2)
    return ref.attention(q, k, v, causal=True, scale=scale, doc_start=doc_start, window=window)


# --------------------------------------------------------------------------------------
# SwiGLU on the fused [gate | up] activation
# --------------------------------------------------------------------------------------
class _SwiGLU(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gu):
        C = _ext.load()
        gu2 = gu.reshape(-1, gu.shape[-1])
        ctx.save_for_backward(gu2)
        ctx.shape = gu.shape
        return C.swiglu_fwd(gu2).view(*gu.shape[:-1], gu.shape[-1] // 2)

    @staticmethod
    def backward(ctx, dh):
        C = _ext.load()
        (gu2,) = ctx.saved_tensors
        dh2 = dh.reshape(-1, dh.shape[-1]).contiguous()
        return C.swiglu_bwd(dh2, gu2).view(ctx.shape)


def swiglu(gu):
    if _ext.use_cuda_kernel("swiglu", gu) and gu.dtype == torch.bfloat16:
        return _SwiGLU.apply(gu)
    return ref.swiglu(gu)


# --------------------------------------------------------------------------------------
# cross entropy (forward computes the loss and leaves dlogits in place of the logits)
# --------------------------------------------------------------------------------------
class _CrossEntropy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, targets):
        C = _ext.load()
        # one pass: per-row logsumexp -> loss; second pass overwrites logits with
        # (softmax - onehot) / n_valid so backward is free of [T,V] temporaries.
        loss = C.cross_entropy_fwd_bwd(logits, targets)  # logits storage now holds dlogits
        ctx.save_for_backward(logits.detach())
        return loss

    @staticmethod
    def backward(ctx, dloss):
        (dlogits,) = ctx.saved_tensors
        # dloss is a scalar; the common case (== 1) costs nothing
        C = _ext.load()
        C.scale_inplace(dlogits, dloss.reshape(1).float())
        return dlogits, None


def cross_entropy(logits, targets):
    """Mean CE over targets != -100. logits [T,V] (consumed in place on CUDA), targets [T] int64."""
    if _ext.use_cuda_kernel("cross_entropy", logits, targets) and logits.dtype == torch.bfloat16:
        return _CrossEntropy.apply(logits, targets.contiguous())
    return ref.cross_entropy(logits, targets)


# --------------------------------------------------------------------------------------
# embedding
# --------------------------------------------------------------------------------------
class _Embedding(torch.autograd.Function):
    @staticmethod
    def forward(ctx, ids, w):
        C = _ext.load()
        ctx.save_for_backward(ids)
        ctx.w_param = w
        return C.embedding_fwd(ids.reshape(-1), w).view(*ids.shape, w.shape[1])

    @staticmethod
    def backward(ctx, dout):
        C = _ext.load()
        (ids,) = ctx.saved_tensors
        w = ctx.w_param
        d2 = dout.reshape(-1, dout.shape[-1]).contiguous()

        def into(out, acc):
            flat = ids.reshape(-1)
            if torch.are_deterministic_algorithms_enabled():
                # --deterministic: sorted runs summed in token order, no atomics (bit-identical run to run)
                if not acc:
                    out.zero_()
                srt, perm = torch.sort(flat, stable=True)
                C.embedding_bwd_sorted(d2, srt.contiguous(), perm.contiguous(), out, True)
                return
            # each row summed in fp32 and rounded once; overwrite mode zeroes the rows of absent ids too
            C.embedding_bwd(d2, flat, out, acc)

        return None, _emit_weight_grad(w, into, w)


def embedding(ids, w):
    if _ext.use_cuda_kernel("embedding", ids, w) and w.dtype == torch.bfloat16:
        return _Embedding.apply(ids, w)
    return ref.embedding(ids, w)
