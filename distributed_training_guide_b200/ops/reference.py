"""Plain-PyTorch fp32 reference implementations of every op.

These serve two roles and are never a second GPU backend:
  * the CPU execution path (chapter 01's GPT-2 plumbing config, all ``gloo`` tests);
  * the numerics oracle the CUDA kernels are tested against (``tests/test_gpu_elementwise.py``,
    ``tests/test_gpu_attention.py``, ``tests/test_gpu_gemm.py``; ``tests/test_gpu_step_reference.py`` runs a
    whole fp32 model on them against the training step).

Semantics follow what the reference guide gets from ``transformers`` (SURVEY.md §3.2 /
K1-K9): RMSNorm with fp32 statistics, half-rotation RoPE, causal softmax attention
with GQA (optionally document-masked and / or sliding-window), SwiGLU, shifted-label mean cross-entropy with ``ignore_index=-100``.  The fp8 functions define the
quantisation of ``ops.linear(..., fp8=True)`` (per-tensor current scaling) exactly, so the cast kernels are tested bit for bit.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def linear(x, w, bias=None):
    return F.linear(x, w, bias)


def rms_norm(x, w, eps):
    xf = x.float()
    rstd = torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    return ((xf * rstd).to(x.dtype) * w).to(x.dtype)


def rms_norm_one_rounding(x, w, eps):
    """RMSNorm with the gain applied in fp32 and one rounding to ``x.dtype`` (transformers' ``Olmo2RMSNorm``, and what
    the rmsnorm kernels compute): ``(w * (x * rsqrt(mean(x^2) + eps))).to(x.dtype)``."""
    xf = x.float()
    rstd = torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)
    return (w.float() * (xf * rstd)).to(x.dtype)


def rms_norm_add(x, r, w, eps):
    """Norm-then-add (OLMo 2's post-sublayer norms): ``r + rms_norm_one_rounding(x, w, eps)``, the normalised branch
    rounded to ``x.dtype`` before the add and the sum rounded again."""
    return r + rms_norm_one_rounding(x, w, eps)


def layer_norm(x, w, b, eps):
    """LayerNorm over the last dimension in fp32 with one rounding to ``x.dtype`` (what ATen's bf16 ``layer_norm`` and
    the layernorm kernels compute): ``((x - mean) * rsqrt(var + eps) * w + b).to(x.dtype)``, biased variance."""
    return F.layer_norm(x.float(), (x.shape[-1],), w.float(), b.float(), eps).to(x.dtype)


def layer_norm2(x, r, w1, b1, w2, b2, eps):
    """GPT-NeoX's two LayerNorms over one residual stream: ``h = x + r`` (``x`` when ``r`` is None), then
    ``(layer_norm(h, w1, b1), layer_norm(h, w2, b2), h)``."""
    h = x if r is None else x + r
    return layer_norm(h, w1, b1, eps), layer_norm(h, w2, b2, eps), h


def add_rms_norm(x, residual, w, eps):
    """returns (normed, new_residual) with new_residual = x + residual."""
    h = x + residual
    return rms_norm(h, w, eps), h


def rope_tables(positions, head_dim, theta, scaling=None, dtype=torch.float32):
    """cos/sin tables [*positions.shape, head_dim//2] in fp32 (llama3 scaling supported)."""
    inv_freq = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.float32, device=positions.device) / head_dim))
    if scaling and scaling.get("rope_type", scaling.get("type")) == "llama3":
        factor = scaling["factor"]
        lo, hi = scaling["low_freq_factor"], scaling["high_freq_factor"]
        old = scaling["original_max_position_embeddings"]
        wavelen = 2 * math.pi / inv_freq
        smooth = (old / wavelen - lo) / (hi - lo)
        scaled = torch.where(wavelen > old / lo, inv_freq / factor, inv_freq)
        mid = (1 - smooth) * inv_freq / factor + smooth * inv_freq
        is_mid = (wavelen <= old / lo) & (wavelen >= old / hi)
        inv_freq = torch.where(is_mid, mid, scaled)
    ang = positions.to(torch.float32)[..., None] * inv_freq
    return ang.cos().to(dtype), ang.sin().to(dtype)


def rope_apply(x, cos, sin, inverse=False):
    """x: [B, S, nheads, d]; cos/sin: [S, d/2] or [B, S, d/2]. Half-rotation (HF Llama) layout."""
    d2 = x.shape[-1] // 2
    xf = x.float()
    x1, x2 = xf[..., :d2], xf[..., d2:]
    if cos.dim() == 2:
        c, s = cos[None, :, None, :], sin[None, :, None, :]
    else:
        c, s = cos[:, :, None, :], sin[:, :, None, :]
    if inverse:
        s = -s
    out = torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], dim=-1)
    return out.to(x.dtype)


def document_mask(doc_start, S, window=None, device=None):
    """bool [B, S, S]: query q may see key k iff ``max(doc_start[b, q], q - window + 1) <= k <= q`` (causal attention
    inside each document and inside the sliding window; ``doc_start`` as ``ops.document_starts`` returns it).
    ``doc_start`` None means one document per row and gives a [1, S, S] mask on ``device``; ``window`` None means no
    window."""
    k = torch.arange(S, device=doc_start.device if doc_start is not None else device)
    mask = (k[None, :] <= k[:, None])[None]
    if doc_start is not None:
        mask = mask & (k[None, None, :] >= doc_start.long()[:, :, None])
    if window is not None:
        mask = mask & (k[None, :] > k[:, None] - window)[None]
    return mask


def attention(q, k, v, causal=True, scale=None, doc_start=None, window=None):
    """q: [B, S, nh, d]; k, v: [B, S, nkv, d] -> [B, S, nh, d]. fp32 softmax.  ``doc_start`` (int [B, S]) and
    ``window`` (int >= 1): document masking and a sliding window on top of the causal mask (see ``document_mask``)."""
    B, S, nh, d = q.shape
    nkv = k.shape[2]
    scale = scale if scale is not None else 1.0 / math.sqrt(d)
    qf = q.float().permute(0, 2, 1, 3)
    kf = k.float().permute(0, 2, 1, 3)
    vf = v.float().permute(0, 2, 1, 3)
    if nkv != nh:
        rep = nh // nkv
        kf = kf.repeat_interleave(rep, dim=1)
        vf = vf.repeat_interleave(rep, dim=1)
    s = torch.matmul(qf, kf.transpose(-1, -2)) * scale
    if doc_start is not None or window is not None:
        s = s.masked_fill(~document_mask(doc_start, S, window, device=q.device)[:, None], float("-inf"))
    elif causal:
        mask = torch.ones(S, k.shape[1], dtype=torch.bool, device=q.device).tril()
        s = s.masked_fill(~mask, float("-inf"))
    p = torch.softmax(s, dim=-1)
    o = torch.matmul(p, vf)
    return o.permute(0, 2, 1, 3).to(q.dtype)


def swiglu(gu):
    """gu: [..., 2*I] laid out as [gate | up] -> silu(gate) * up."""
    g, u = gu.chunk(2, dim=-1)
    return (F.silu(g.float()) * u.float()).to(gu.dtype)


def moe_route(x, gate_w, k, norm_topk_prob=False):
    """The MoE router in fp32: ``(p, w, idx)`` with p = softmax(x @ gate_w.T) [T, E], and w, idx [T, k] the top-k
    probabilities and their experts.  w is kept raw (OLMoE, ``norm_topk_prob: false``) or divided by its row sum in
    fp32 (Qwen3-MoE's ``norm_topk_prob: true``, as ``Qwen3MoeTopKRouter`` does it)."""
    p = torch.softmax(x.float() @ gate_w.float().t(), dim=-1)
    w, idx = torch.topk(p, k, dim=-1)
    if norm_topk_prob:
        w = w / w.sum(dim=-1, keepdim=True)
    return p, w, idx


def moe(x, gate_w, gate_up, down, k, norm_topk_prob=False):
    """The sparse MLP of OLMoE and Qwen3-MoE in fp32, one expert at a time: ``sum_slot w[t, slot] * expert_idx[t, slot](x_t)`` with
    ``expert_e(x) = down[e] @ (silu(g) * u)``, ``[g | u] = gate_up[e] @ x``.  x [T, H], gate_w [E, H], gate_up
    [E, 2I, H], down [E, H, I].  Returns ``(y in x.dtype, p)`` with p the fp32 router probabilities [T, E]."""
    xf = x.float()
    p, w, idx = moe_route(xf, gate_w, k, norm_topk_prob)
    out = torch.zeros_like(xf)
    for e in range(gate_up.shape[0]):
        tok, slot = (idx == e).nonzero(as_tuple=True)
        if tok.numel() == 0:
            continue
        g, u = (xf[tok] @ gate_up[e].float().t()).chunk(2, dim=-1)
        y = (F.silu(g) * u) @ down[e].float().t()
        out = out.index_add(0, tok, y * w[tok, slot, None])
    return out.to(x.dtype), p


def router_aux_loss(counts, psums, n_tokens, num_experts):
    """The Switch load-balancing loss of transformers' ``load_balancing_loss_func`` over the concatenated tokens of
    every layer: ``E * sum_e f_e * P_e`` with f_e = (top-k assignments to e) / tokens and P_e the mean router
    probability of e.  ``counts`` and ``psums`` hold one [E] tensor per layer (assignment counts and column sums of
    p); ``n_tokens`` is the token count of one layer."""
    n = float(n_tokens * len(psums))
    f = torch.stack([c.float() for c in counts]).sum(0) / n
    P = torch.stack(list(psums)).sum(0) / n
    return num_experts * (f * P).sum()


def gelu_new(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x.pow(3))))


def gelu(x):
    """Exact (erf) GELU, ``x/2 * (1 + erf(x / sqrt(2)))``, in fp32 with one rounding to ``x.dtype``."""
    return F.gelu(x.float()).to(x.dtype)


def shift_labels(labels):
    """HF causal-LM convention: token t predicts label t+1; last position ignored."""
    pad = torch.full_like(labels[..., :1], -100)
    return torch.cat([labels[..., 1:], pad], dim=-1)


def drop_cross_document_targets(shifted, doc_start, ignore_index=-100):
    """``shifted`` [B, S] targets after ``shift_labels``: the target of token t is token t+1.  Where token t+1 starts
    a document (``doc_start[t+1] == t+1``), the target becomes ``ignore_index``, so the last token of one document
    is not trained to predict the first token of the next."""
    S = doc_start.shape[-1]
    first = doc_start == torch.arange(S, device=doc_start.device, dtype=doc_start.dtype)
    nxt = torch.zeros_like(first)
    nxt[..., :-1] = first[..., 1:]
    return shifted.masked_fill(nxt, ignore_index)


def cross_entropy(logits, targets, ignore_index=-100):
    """logits [T, V] (any float dtype), targets [T] already shifted -> mean loss (fp32) over the targets that are
    not ``ignore_index``.  With none left (a chunk of padding) the loss is 0 with a zero gradient, as in the CUDA
    kernel, where ``reduction="mean"`` would give NaN."""
    total = F.cross_entropy(logits.float(), targets, ignore_index=ignore_index, reduction="sum")
    return total / (targets != ignore_index).sum().clamp(min=1)


def embedding(ids, w):
    return F.embedding(ids, w)


def fp8_quantize(t, dtype, amax=None):
    """Per-tensor current scaling of ``t`` to ``dtype`` (``torch.float8_e4m3fn`` or ``torch.float8_e5m2``), as the
    fp8 cast kernels compute it: ``amax = max|t|``, ``scale = FP8_MAX / amax`` in fp32 (1 when amax is 0) clamped
    to FLT_MAX, ``t8 = round_to_nearest_even(t * scale)`` saturated at +-FP8_MAX.  The clamp matters for a finite
    ``0 < amax < FP8_MAX / FLT_MAX`` (about 1.3e-36 for e4m3, 1.7e-34 for e5m2), where the division overflows: an
    Inf scale would turn every zero into NaN and every other element into +-FP8_MAX; it keeps a NaN scale NaN.
    torch's cast of an out-of-range value gives NaN (e4m3) or Inf (e5m2) instead of saturating, hence the clamp of
    ``t * scale``, which keeps NaN.  A non-finite amax makes the scale 0 or NaN, so ``t8`` holds NaN and the
    non-finite value reaches whatever consumes it.
    ``amax`` (a one-element fp32 tensor) is computed from ``t`` when not given.
    Returns ``(t8, scale_inv)`` with ``scale_inv = 1 / scale`` as a one-element fp32 tensor (2^-128, a subnormal,
    for the clamped scale)."""
    fp8_max = torch.finfo(dtype).max
    flt_max = torch.finfo(torch.float32).max
    tf = t.float()
    amax = tf.abs().max().reshape(1) if amax is None else amax.float().reshape(1)
    scale = torch.where(amax == 0, torch.ones_like(amax), torch.full_like(amax, fp8_max) / amax)
    scale = torch.where(scale > flt_max, torch.full_like(scale, flt_max), scale)
    t8 = (tf * scale).clamp(-fp8_max, fp8_max).to(dtype)
    return t8, torch.ones_like(scale) / scale


def fp8_gemm(a8, scale_inv_a, b8, scale_inv_b):
    """fp32 ``(a8 * scale_inv_a) @ (b8 * scale_inv_b).T`` of fp8 operands stored [M, K] and [N, K]."""
    return (a8.float() * scale_inv_a) @ (b8.float() * scale_inv_b).t()


def clip_coefficient(norm, max_norm):
    """``torch.nn.utils.clip_grad_norm_``'s factor for a gradient of global L2 norm ``norm`` (an fp32 tensor):
    ``min(1, max_norm / (norm + 1e-6))`` in fp32.  A NaN norm gives NaN and an Inf norm 0, as in torch: the step
    goes non-finite rather than being skipped."""
    norm = torch.as_tensor(norm, dtype=torch.float32)
    return (torch.tensor(max_norm, dtype=torch.float32, device=norm.device) / (norm + 1e-6)).clamp(max=1.0)


def adamw_step(p, g, m, v, lr, beta1, beta2, eps, weight_decay, step, grad_scale=1.0, coef=None):
    """Single-tensor AdamW with fp32 math on (possibly bf16) storage, matching
    ``torch.optim.AdamW`` (decoupled decay, bias correction).  ``coef`` (gradient clipping, ``clip_coefficient``)
    multiplies the gradient first, as the clipping kernels do."""
    gf = g.float() if coef is None else g.float() * torch.as_tensor(coef, dtype=torch.float32).to(g.device)
    pf, gf, mf, vf = p.float(), gf * grad_scale, m.float(), v.float()
    pf = pf * (1 - lr * weight_decay)
    mf = beta1 * mf + (1 - beta1) * gf
    vf = beta2 * vf + (1 - beta2) * gf * gf
    bc1 = 1 - beta1 ** step
    bc2 = 1 - beta2 ** step
    denom = (vf.sqrt() / math.sqrt(bc2)) + eps
    pf = pf - (lr / bc1) * mf / denom
    p.copy_(pf)
    m.copy_(mf)
    v.copy_(vf)
