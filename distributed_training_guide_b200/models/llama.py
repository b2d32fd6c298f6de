"""Llama-family causal LM built on the sm_90a op layer (Llama; Mistral: Llama plus a sliding attention window; Qwen3:
Llama plus QK-norm, with a head_dim of its own; Qwen2: Llama plus q/k/v biases; OLMo 2: Llama with a full-width
QK-norm and RMSNorms after each sublayer instead of before it, ``Olmo2DecoderLayer``; StarCoder2: Llama with
LayerNorms, a c_fc -> GELU-tanh -> c_proj MLP and a bias on every projection, ``Starcoder2DecoderLayer``; GPT-NeoX:
StarCoder2's parameters with a parallel residual, partial rotary embeddings and an exact GELU, ``GPTNeoXDecoderLayer``).

Same module tree and parameter names as ``transformers``' ``LlamaForCausalLM`` (what
the reference instantiates at e.g. ``02-distributed-data-parallel/train_llm.py:57-58``)
so checkpoints keep meaningful keys: ``model.embed_tokens.weight``,
``model.layers.{i}.self_attn.{q,k,v,o}_proj.weight``, ``model.layers.{i}.mlp.
{gate,up,down}_proj.weight``, ``...{input,post_attention}_layernorm.weight``,
``model.norm.weight``, ``lm_head.weight``; Qwen3 adds ``...self_attn.{q,k}_norm.weight``, Qwen2
``...self_attn.{q,k,v}_proj.bias``; OLMo 2 has ``...self_attn.{q,k}_norm.weight`` ([nh*d], [nkv*d]) and
``...post_{attention,feedforward}_layernorm.weight`` and no ``input_layernorm``; StarCoder2 ``...mlp.{c_fc,c_proj}.{weight,bias}``,
``...self_attn.{q,k,v,o}_proj.bias`` and a ``.bias`` beside every norm gain; GPT-NeoX StarCoder2's names (its
checkpoint names and per-head interleaved q|k|v live in ``models/gpt_neox_layout.py``).

What is *different* from the HF module code (SURVEY.md §3.2) is the execution plan:
  * q/k/v (and gate/up) projections run as ONE wgmma GEMM over a fused weight that is
    just the adjacent placement of the three (two) parameters in the layer's flat buffer;
  * RoPE rotates the q and k heads in place inside the fused qkv activation, attention
    reads q/k/v straight out of that buffer through strided TMA descriptors (no
    transpose/contiguous/repeat_kv copies);
  * the residual add is deferred and fused into the following RMSNorm kernel;
  * the loss kernel leaves dlogits in place of the logits (no fp32 [T,V] copy).
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Optional

import torch
from torch import nn

from .. import _ext, ops
from ..ops import reference as ref
from .configs import ModelConfig


def _name_seed(seed: int, name: str) -> int:
    import zlib

    return (int(seed) * 1000003 + zlib.crc32(name.encode())) % (2**63 - 1)


@torch.no_grad()
def init_parameter_(p, name: str, seed: int, std: float = 0.02, full_shape=None, shard_dim=None, shard_index=0,
                    shard_count=1):
    """Fill ``p`` (possibly a tensor-parallel slice of a ``full_shape`` parameter) deterministically."""
    if name.endswith("norm.weight") or name.endswith("layernorm.weight"):
        p.fill_(1.0)
        return
    if name.endswith(".bias"):   # projection biases start at zero, as in transformers
        p.zero_()
        return
    gen = torch.Generator(device=p.device)
    gen.manual_seed(_name_seed(seed, name))
    shape = tuple(full_shape) if full_shape is not None else tuple(p.shape)
    full = torch.empty(shape, dtype=torch.float32, device=p.device).normal_(0.0, std, generator=gen)
    if shard_dim is not None and shard_count > 1:
        full = full.chunk(shard_count, dim=shard_dim)[shard_index]
    p.copy_(full.to(p.dtype))


#: which dimension of each parameter tensor parallelism splits (None = replicated); a projection's bias (q/k/v, Qwen2)
#: is split with its output features, dimension 0
TP_SHARD_DIM = {"q_proj": 0, "k_proj": 0, "v_proj": 0, "gate_proj": 0, "up_proj": 0, "o_proj": 1, "down_proj": 1,
                "embed_tokens": 1, "lm_head": 0}


def tp_shard_spec(name: str, p, tp_size: int, tp_rank: int) -> dict:
    """init_parameter_ kwargs that make rank ``tp_rank`` hold its slice of the full parameter."""
    if tp_size == 1:
        return {}
    for key, dim in TP_SHARD_DIM.items():
        if f"{key}.weight" in name or (f"{key}.bias" in name and dim == 0):
            full = list(p.shape)
            full[dim] *= tp_size
            return dict(full_shape=full, shard_dim=dim, shard_index=tp_rank, shard_count=tp_size)
    return {}


class Linear(nn.Module):
    """Projection holding ``weight`` [out, in] and, with ``bias=True``, ``bias`` [out] (HF naming)."""

    def __init__(self, in_features, out_features, dtype=None, device=None, bias=False):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.weight = nn.Parameter(torch.empty(out_features, in_features, dtype=dtype, device=device))
        self.bias = nn.Parameter(torch.zeros(out_features, dtype=dtype, device=device)) if bias else None

    def forward(self, x):
        return ops.linear(x, self.weight, self.bias)

    def reset_parameters(self, std=0.02):
        nn.init.normal_(self.weight, mean=0.0, std=std)
        if self.bias is not None:
            nn.init.zeros_(self.bias)


class RMSNorm(nn.Module):
    def __init__(self, hidden, eps, dtype=None, device=None):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(hidden, dtype=dtype, device=device))

    def forward(self, x, residual=None):
        if residual is None:
            return ops.rms_norm(x, self.weight, self.eps), x
        return ops.add_rms_norm(x, residual, self.weight, self.eps)

    def reset_parameters(self):
        nn.init.ones_(self.weight)


class LayerNorm(nn.Module):
    """LayerNorm with a gain ``weight`` and a ``bias`` (HF names), StarCoder2's norm."""

    def __init__(self, hidden, eps, dtype=None, device=None):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(hidden, dtype=dtype, device=device))
        self.bias = nn.Parameter(torch.zeros(hidden, dtype=dtype, device=device))

    def forward(self, x, residual=None):
        if residual is None:
            return ops.layer_norm(x, self.weight, self.bias, self.eps), x
        return ops.add_layer_norm(x, residual, self.weight, self.bias, self.eps)

    def reset_parameters(self):
        nn.init.ones_(self.weight)
        nn.init.zeros_(self.bias)


class Embedding(nn.Module):
    def __init__(self, n, dim, dtype=None, device=None):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(n, dim, dtype=dtype, device=device))

    def forward(self, ids):
        return ops.embedding(ids, self.weight)

    def reset_parameters(self, std=0.02):
        nn.init.normal_(self.weight, mean=0.0, std=std)


class RotaryEmbedding(nn.Module):
    """cos/sin tables in fp32.  ``inv_freq`` is a non-persistent buffer like HF's (the
    reference has to re-create / broadcast it by hand: ``04:36-40``, ``05:131-139``);
    here it is recomputed from the config on demand so meta-device init needs no patch."""

    def __init__(self, config: ModelConfig):
        super().__init__()
        self.head_dim = config.rotary_dim   # the rotated share of each head (all of it but for GPT-NeoX)
        self.theta = config.rope_theta
        self.scaling = config.rope_scaling
        self._cache = {}

    def forward(self, positions):
        return ref.rope_tables(positions, self.head_dim, self.theta, self.scaling)

    def tables(self, seq_len, device):
        key = (seq_len, str(device))
        if key not in self._cache:
            pos = torch.arange(seq_len, device=device)
            self._cache = {key: self.forward(pos)}
        return self._cache[key]


class LlamaAttention(nn.Module):
    def __init__(self, config: ModelConfig, dtype=None, device=None, tp_size=1):
        super().__init__()
        h, d = config.hidden_size, config.head_dim
        assert config.num_attention_heads % tp_size == 0 and config.num_key_value_heads % tp_size == 0
        self.num_heads = config.num_attention_heads // tp_size
        self.num_kv_heads = config.num_key_value_heads // tp_size
        self.head_dim = d
        #: the rotated share of each q/k head: all of it but for GPT-NeoX's partial rotary
        self.rotary_dim = config.rotary_dim
        #: sliding-window attention (Mistral): None, or W >= 1 with query q seeing keys k > q - W only
        self.sliding_window = config.sliding_window
        #: q/k/v biases (Qwen2, StarCoder2), split with their heads under tensor parallelism; an o_proj bias
        #: (StarCoder2) only without it
        qkv_bias = config.qkv_bias or config.all_bias
        self.q_proj = Linear(h, self.num_heads * d, dtype, device, bias=qkv_bias)
        self.k_proj = Linear(h, self.num_kv_heads * d, dtype, device, bias=qkv_bias)
        self.v_proj = Linear(h, self.num_kv_heads * d, dtype, device, bias=qkv_bias)
        self.o_proj = Linear(self.num_heads * d, h, dtype, device, bias=config.all_bias)
        #: QK-norm (Qwen3): [head_dim] gains, replicated under tensor parallelism (every rank normalises its heads)
        self.q_norm = RMSNorm(d, config.rms_norm_eps, dtype, device) if config.qk_norm else None
        self.k_norm = RMSNorm(d, config.rms_norm_eps, dtype, device) if config.qk_norm else None
        #: full-width QK-norm (OLMo 2): [nh * head_dim] and [nkv * head_dim] gains, one statistic over all of a
        #: token's q (k) heads, so tensor parallelism cannot split them (it is refused for OLMo 2)
        self.full_qk_norm = config.full_qk_norm
        if self.full_qk_norm:
            self.q_norm = RMSNorm(self.num_heads * d, config.rms_norm_eps, dtype, device)
            self.k_norm = RMSNorm(self.num_kv_heads * d, config.rms_norm_eps, dtype, device)

    def position_qk_(self, qkv, cos, sin):
        """RoPE (after QK-norm, when the layer has it) on the q and k heads of ``qkv`` [B,S,heads,d], in place on
        the kernel path."""
        if self.q_norm is None:
            return ops.rope_qkv_(qkv, cos, sin, self.num_heads + self.num_kv_heads, self.rotary_dim)
        if self.full_qk_norm:
            return ops.olmo_qk_norm_rope_(qkv, self.q_norm.weight, self.k_norm.weight, cos, sin, self.num_heads,
                                          self.num_kv_heads, self.q_norm.eps)
        return ops.qk_norm_rope_(qkv, self.q_norm.weight, self.k_norm.weight, cos, sin, self.num_heads,
                                 self.num_kv_heads, self.q_norm.eps)


class LlamaMLP(nn.Module):
    def __init__(self, config: ModelConfig, dtype=None, device=None, tp_size=1):
        super().__init__()
        h, i = config.hidden_size, config.intermediate_size
        assert i % tp_size == 0
        self.gate_proj = Linear(h, i // tp_size, dtype, device)
        self.up_proj = Linear(h, i // tp_size, dtype, device)
        self.down_proj = Linear(i // tp_size, h, dtype, device)


class Starcoder2MLP(nn.Module):
    """StarCoder2's MLP: ``c_proj(gelu_tanh(c_fc(x)))``, both projections with a bias."""

    def __init__(self, config: ModelConfig, dtype=None, device=None):
        super().__init__()
        h, i = config.hidden_size, config.intermediate_size
        self.c_fc = Linear(h, i, dtype, device, bias=True)
        self.c_proj = Linear(i, h, dtype, device, bias=True)


class FusedWeight:
    """A fused [q|k|v] or [gate|up] weight: adjacent parameters of a flat buffer seen as one
    matrix, plus the matching view of the flat gradient buffer (see ops._emit_weight_grad)."""

    def __init__(self, data, grad):
        self.data = data
        self._dtg_grad = grad
        self._dtg_writes = 0
        self._dtg_ready_hook = None


class LlamaDecoderLayer(nn.Module):
    #: parameter order inside a Llama / Mistral layer's flat buffer; adjacency is what makes fusion free
    FLAT_ORDER = (
        "self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight",
        "self_attn.o_proj.weight", "mlp.gate_proj.weight", "mlp.up_proj.weight",
        "mlp.down_proj.weight", "input_layernorm.weight", "post_attention_layernorm.weight",
    )
    #: appended with QK-norm: after the layer norms, so the matrices stay first (FSDP's chunked layout) and every
    #: replicated gain sits in one run at the end (TP sums their gradients over the group in one launch)
    QK_NORM_ORDER = ("self_attn.q_norm.weight", "self_attn.k_norm.weight")
    #: appended with q/k/v biases (Qwen2), also after the layer norms: adjacent, and each a multiple of 8 elements, so
    #: they form one [(nh + 2 nkv) d] q|k|v bias (``fused_view_1d``) next to the fused q|k|v weight
    QKV_BIAS_ORDER = ("self_attn.q_proj.bias", "self_attn.k_proj.bias", "self_attn.v_proj.bias")
    FUSED = {"qkv": FLAT_ORDER[0:3], "gate_up": FLAT_ORDER[4:6]}

    def __init__(self, config: ModelConfig, layer_idx: int, dtype=None, device=None, tp_size=1):
        super().__init__()
        self.layer_idx = layer_idx
        self.self_attn = LlamaAttention(config, dtype, device, tp_size)
        self.mlp = LlamaMLP(config, dtype, device, tp_size)
        self.input_layernorm = RMSNorm(config.hidden_size, config.rms_norm_eps, dtype, device)
        self.post_attention_layernorm = RMSNorm(config.hidden_size, config.rms_norm_eps, dtype, device)
        #: this layer's parameter order in its flat buffer (parallel/flat.py, parallel/fsdp.py); a parameter missing
        #: here would get no gradient buffer and no optimizer update
        self.flat_order = (self.FLAT_ORDER + (self.QK_NORM_ORDER if config.qk_norm else ())
                           + (self.QKV_BIAS_ORDER if config.qkv_bias else ()))
        self._fused = {}  # name -> FusedWeight, installed by parallel.flat.FlatParamGroup
        self.tp = None  # installed by parallel.tp.apply_tensor_parallel
        self.fp8 = False  # set through LlamaForCausalLM.fp8: the four projections run ops.fp8_linear

    # fused weights -------------------------------------------------------------------
    def _qkv_weight(self):
        f = self._fused.get("qkv")
        if f is not None and _ext.use_cuda_kernel("gemm", f.data):
            return f.data, f
        a = self.self_attn
        return torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], dim=0), None

    def _qkv_bias(self):
        """(fused q|k|v bias, its flat-gradient owner) or (None, None) without biases."""
        a = self.self_attn
        if a.q_proj.bias is None:
            return None, None
        f = self._fused.get("qkv_bias")
        if f is not None and _ext.use_cuda_kernel("gemm", f.data):
            return f.data, f
        return torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias]), None

    def _gate_up_weight(self):
        f = self._fused.get("gate_up")
        if f is not None and _ext.use_cuda_kernel("gemm", f.data):
            return f.data, f
        return torch.cat([self.mlp.gate_proj.weight, self.mlp.up_proj.weight], dim=0), None

    # forward ---------------------------------------------------------------------------
    def forward(self, x, residual, cos, sin, doc_start=None):
        """x: [B,S,H] branch output of the previous layer (or the embeddings);
        residual: running residual stream *before* adding x (None for the first layer);
        doc_start: None or int32 [B,S] from ``ops.document_starts`` (attention stays inside each document).
        Returns (mlp_out, residual) with the final add again deferred to the consumer."""
        att = self.self_attn
        B, S, _ = x.shape
        fused_linear = ops.fp8_linear if self.fp8 else ops.fused_linear
        y, h = self.input_layernorm(x, residual)
        w, owner = self._qkv_weight()
        b, b_owner = self._qkv_bias()
        qkv = fused_linear(y, w, owner, b, b_owner).view(B, S, att.num_heads + 2 * att.num_kv_heads, att.head_dim)
        qkv = att.position_qk_(qkv, cos, sin)
        a = ops.attention_qkv(qkv, att.num_heads, att.num_kv_heads, doc_start=doc_start, window=att.sliding_window)
        a = a.reshape(B, S, att.num_heads * att.head_dim)
        a = ops.fp8_linear(a, att.o_proj.weight) if self.fp8 else att.o_proj(a)
        y, h = self.post_attention_layernorm(a, h)
        w, owner = self._gate_up_weight()
        act = ops.swiglu(fused_linear(y, w, owner))
        down = ops.fp8_linear(act, self.mlp.down_proj.weight) if self.fp8 else self.mlp.down_proj(act)
        return down, h


class Olmo2DecoderLayer(LlamaDecoderLayer):
    """OLMo 2's layer: the Llama layer with full-width QK-norm and RMSNorms after each sublayer instead of before it:
    ``h1 = h + norm_pa(o_proj(attn(h)))``, ``h2 = h1 + norm_pf(mlp(h1))``; there is no ``input_layernorm``."""

    #: matrices first in the Llama order (FSDP's chunked layout; ``FUSED``'s q|k|v and gate|up), then the gains
    FLAT_ORDER = LlamaDecoderLayer.FLAT_ORDER[:7] + (
        "post_attention_layernorm.weight", "post_feedforward_layernorm.weight", "self_attn.q_norm.weight",
        "self_attn.k_norm.weight",
    )

    def __init__(self, config: ModelConfig, layer_idx: int, dtype=None, device=None, tp_size=1):
        nn.Module.__init__(self)
        self.layer_idx = layer_idx
        self.self_attn = LlamaAttention(config, dtype, device, tp_size)
        self.mlp = LlamaMLP(config, dtype, device, tp_size)
        self.post_attention_layernorm = RMSNorm(config.hidden_size, config.rms_norm_eps, dtype, device)
        self.post_feedforward_layernorm = RMSNorm(config.hidden_size, config.rms_norm_eps, dtype, device)
        self.flat_order = self.FLAT_ORDER
        self._fused = {}
        self.tp = None
        self.fp8 = False

    def forward(self, x, residual, cos, sin, doc_start=None):
        """x: [B,S,H] the residual stream (the embeddings for the first layer); residual: None.  The pending add
        needs this layer's post_feedforward_layernorm gain, which FSDP may reshard before the next layer runs, so the
        layer completes its stream and returns (h2, None): every layer sees ``residual = None``."""
        assert residual is None, "an OLMo 2 layer takes the complete residual stream"
        att = self.self_attn
        B, S, _ = x.shape
        fused_linear = ops.fp8_linear if self.fp8 else ops.fused_linear
        w, owner = self._qkv_weight()
        qkv = fused_linear(x, w, owner).view(B, S, att.num_heads + 2 * att.num_kv_heads, att.head_dim)
        qkv = att.position_qk_(qkv, cos, sin)
        a = ops.attention_qkv(qkv, att.num_heads, att.num_kv_heads, doc_start=doc_start, window=att.sliding_window)
        a = a.reshape(B, S, att.num_heads * att.head_dim)
        a = ops.fp8_linear(a, att.o_proj.weight) if self.fp8 else att.o_proj(a)
        n = self.post_attention_layernorm
        h1 = ops.rms_norm_add(a, x, n.weight, n.eps)
        w, owner = self._gate_up_weight()
        act = ops.swiglu(fused_linear(h1, w, owner))
        down = ops.fp8_linear(act, self.mlp.down_proj.weight) if self.fp8 else self.mlp.down_proj(act)
        n = self.post_feedforward_layernorm
        return ops.rms_norm_add(down, h1, n.weight, n.eps), None


class Starcoder2DecoderLayer(LlamaDecoderLayer):
    """StarCoder2's layer: the Llama layer with LayerNorms, a c_fc -> GELU-tanh -> c_proj MLP and a bias on every
    projection.  The residual add stays deferred: the layer returns ``(c_proj_out, h)``."""

    #: matrices first (FSDP's chunked layout; ``FUSED``'s q|k|v), then the norm gains and biases, then the adjacent
    #: q|k|v biases (one 1-D view, ``fused_view_1d``), then the o_proj, c_fc and c_proj biases
    FLAT_ORDER = LlamaDecoderLayer.FLAT_ORDER[:4] + (
        "mlp.c_fc.weight", "mlp.c_proj.weight", "input_layernorm.weight", "input_layernorm.bias",
        "post_attention_layernorm.weight", "post_attention_layernorm.bias",
    ) + LlamaDecoderLayer.QKV_BIAS_ORDER + ("self_attn.o_proj.bias", "mlp.c_fc.bias", "mlp.c_proj.bias")
    FUSED = {"qkv": FLAT_ORDER[0:3]}

    def __init__(self, config: ModelConfig, layer_idx: int, dtype=None, device=None, tp_size=1):
        nn.Module.__init__(self)
        assert tp_size == 1, "StarCoder2 layers are not tensor-parallel"
        self.layer_idx = layer_idx
        self.self_attn = LlamaAttention(config, dtype, device)   # q, k, v and o with biases (``all_bias``)
        h = config.hidden_size
        self.mlp = Starcoder2MLP(config, dtype, device)
        self.input_layernorm = LayerNorm(h, config.layer_norm_epsilon, dtype, device)
        self.post_attention_layernorm = LayerNorm(h, config.layer_norm_epsilon, dtype, device)
        self.flat_order = self.FLAT_ORDER
        self._fused = {}
        self.tp = None
        self.fp8 = False

    def forward(self, x, residual, cos, sin, doc_start=None):
        att = self.self_attn
        B, S, _ = x.shape
        fused_linear = ops.fp8_linear if self.fp8 else ops.fused_linear
        y, h = self.input_layernorm(x, residual)
        w, owner = self._qkv_weight()
        b, b_owner = self._qkv_bias()
        qkv = fused_linear(y, w, owner, b, b_owner).view(B, S, att.num_heads + 2 * att.num_kv_heads, att.head_dim)
        qkv = att.position_qk_(qkv, cos, sin)
        a = ops.attention_qkv(qkv, att.num_heads, att.num_kv_heads, doc_start=doc_start, window=att.sliding_window)
        a = a.reshape(B, S, att.num_heads * att.head_dim)
        a = ops.fp8_linear(a, att.o_proj.weight, None, att.o_proj.bias) if self.fp8 else att.o_proj(a)
        y, h = self.post_attention_layernorm(a, h)
        mlp = self.mlp
        up = ops.fp8_linear(y, mlp.c_fc.weight, None, mlp.c_fc.bias) if self.fp8 else mlp.c_fc(y)
        act = ops.gelu_tanh(up)
        down = ops.fp8_linear(act, mlp.c_proj.weight, None, mlp.c_proj.bias) if self.fp8 else mlp.c_proj(act)
        return down, h


class GPTNeoXDecoderLayer(Starcoder2DecoderLayer):
    """GPT-NeoX's layer: StarCoder2's parameters (names, ``FLAT_ORDER``, fused q|k|v weight and bias) with a parallel
    residual, ``h' = h + attn(ln1(h)) + mlp(ln2(h))``, RoPE on the first ``rotary_dim`` elements of each q/k head and
    an exact GELU.  Both norms read the same h (``ops.layer_norm2``); the attention dense and the MLP down-projection
    write one branch (``ops.parallel_out``), and the residual add stays deferred: the layer returns ``(branch, h)``."""

    def __init__(self, config: ModelConfig, layer_idx: int, dtype=None, device=None, tp_size=1):
        assert tp_size == 1, "GPT-NeoX layers are not tensor-parallel"
        super().__init__(config, layer_idx, dtype, device, tp_size)

    def forward(self, x, residual, cos, sin, doc_start=None):
        att = self.self_attn
        B, S, _ = x.shape
        fused_linear = ops.fp8_linear if self.fp8 else ops.fused_linear
        n1, n2 = self.input_layernorm, self.post_attention_layernorm
        y1, y2, h = ops.layer_norm2(x, residual, n1.weight, n1.bias, n2.weight, n2.bias, n1.eps)
        w, owner = self._qkv_weight()
        b, b_owner = self._qkv_bias()
        qkv = fused_linear(y1, w, owner, b, b_owner).view(B, S, att.num_heads + 2 * att.num_kv_heads, att.head_dim)
        qkv = att.position_qk_(qkv, cos, sin)
        a = ops.attention_qkv(qkv, att.num_heads, att.num_kv_heads, doc_start=doc_start, window=att.sliding_window)
        a = a.reshape(B, S, att.num_heads * att.head_dim)
        mlp = self.mlp
        up = ops.fp8_linear(y2, mlp.c_fc.weight, None, mlp.c_fc.bias) if self.fp8 else mlp.c_fc(y2)
        act = ops.gelu(up)
        out = ops.parallel_out(a, act, att.o_proj.weight, mlp.c_proj.weight, att.o_proj.bias, mlp.c_proj.bias,
                               fp8=self.fp8)
        return out, h


class LlamaModel(nn.Module):
    def __init__(self, config: ModelConfig, dtype=None, device=None, tp_size=1):
        super().__init__()
        assert config.hidden_size % tp_size == 0
        # tensor parallel: the table is sharded over the hidden dimension (reference: ColwiseParallel on
        # nn.Embedding, 06-tensor-parallel/train_llm.py:82)
        self.embed_tokens = Embedding(config.vocab_size, config.hidden_size // tp_size, dtype, device)
        layer_cls = (Olmo2DecoderLayer if config.post_norm else
                     GPTNeoXDecoderLayer if config.parallel_residual else
                     Starcoder2DecoderLayer if config.arch == "starcoder2" else LlamaDecoderLayer)
        self.layers = nn.ModuleList(
            [layer_cls(config, i, dtype, device, tp_size) for i in range(config.num_hidden_layers)]
        )
        if config.layer_norm:
            self.norm = LayerNorm(config.hidden_size, config.layer_norm_epsilon, dtype, device)
        else:
            self.norm = RMSNorm(config.hidden_size, config.rms_norm_eps, dtype, device)
        self.rotary_emb = RotaryEmbedding(config)


class LlamaForCausalLM(nn.Module):
    def __init__(self, config: ModelConfig, dtype=None, device=None, tp_size=1):
        super().__init__()
        self.config = config
        self.tp_size = tp_size
        self.tp_rank = 0  # set by the tensor-parallel strategy before init_weights
        self.model = LlamaModel(config, dtype, device, tp_size)
        assert config.vocab_size % tp_size == 0
        vocab_local = config.vocab_size // tp_size  # vocabulary-sharded head (loss-parallel)
        self.lm_head = Linear(config.hidden_size, vocab_local, dtype, device)
        if config.tie_word_embeddings:
            assert tp_size == 1, "tied embeddings cannot be tensor-parallel (vocabulary- vs hidden-sharded)"
            self.lm_head.weight = self.model.embed_tokens.weight
        #: parallel engine (parallel/ddp.py, fsdp.py): called around every decoder layer and the
        #: head so it can insert autograd boundaries, prefetch shards and launch bucket kernels
        self.engine = None
        self.activation_checkpointing = False
        self.tp = None
        self.fp8 = False
        #: packed documents (``--document-masking``): with ``position_ids`` given, a document starts at every token
        #: whose position id is 0 (``ops.document_starts``); attention stays inside each document and the last token
        #: of a document is not trained to predict the first token of the next.  Off: ``position_ids`` only feeds RoPE.
        self.document_masking = False

    @property
    def fp8(self) -> bool:
        """Run the decoder-layer projections (q|k|v, o, gate|up, down) through ``ops.fp8_linear``: fp8 GEMMs with
        per-tensor current scaling.  The lm_head, embedding, attention, norms and loss stay bf16."""
        return self._fp8

    @fp8.setter
    def fp8(self, on: bool):
        self._fp8 = bool(on)
        for layer in self.model.layers:
            layer.fp8 = self._fp8

    # -- initialisation -----------------------------------------------------------------
    @torch.no_grad()
    def init_weights(self, std: float = 0.02, seed: Optional[int] = None):
        """Random init: normal(0, 0.02) matrices, unit norm gains.  Every parameter draws from its
        own generator seeded by (seed, parameter name), so the same seed gives the same weights under
        any placement: replicated, flat-sharded (FSDP builds one layer at a time) or tensor-parallel
        (each rank generates the full tensor and keeps its slice)."""
        seed = torch.initial_seed() if seed is None else seed
        self._init_seed = seed
        for name, p in self.named_parameters():
            if not p.is_meta:
                init_parameter_(p, name, seed, std, **tp_shard_spec(name, p, self.tp_size, getattr(self, "tp_rank", 0)))

    def num_parameters(self) -> int:
        return sum(p.numel() for p in self.parameters())

    # -- loss (kept as an attribute like HF's ``model.loss_function``) ---------------------
    @staticmethod
    def loss_function(logits, labels, vocab_size=None):
        tgt = ref.shift_labels(labels).reshape(-1)
        return ops.cross_entropy(logits.reshape(-1, logits.shape[-1]), tgt)

    # -- forward --------------------------------------------------------------------------
    def forward(self, input_ids, attention_mask=None, labels=None, position_ids=None, return_logits=None):
        """``attention_mask`` is accepted for API parity; the data pipeline only produces full
        (unpadded) chunks so only the causal mask is applied (the reference's all-ones mask
        collapses to the same thing inside transformers, SURVEY.md K3).  With ``document_masking``
        and ``position_ids``, attention and targets stay inside each packed document."""
        if self.tp is not None:
            return self.tp.model_forward(self, input_ids, labels, position_ids)
        B, S = input_ids.shape
        m = self.model
        if position_ids is None:
            cos, sin = m.rotary_emb.tables(S, input_ids.device)
        else:
            cos, sin = m.rotary_emb(position_ids)
        doc_start = None
        if self.document_masking and position_ids is not None:
            doc_start = ops.document_starts(position_ids)
        eng = self.engine
        if eng is not None:
            eng.pre_forward(self)
        x = m.embed_tokens(input_ids)
        residual = None
        for i, layer in enumerate(m.layers):
            if eng is not None:
                x, residual = eng.pre_layer(i, layer, x, residual)
            if self.activation_checkpointing and torch.is_grad_enabled():
                from ..parallel.act_ckpt import checkpoint_layer

                x, residual = checkpoint_layer(layer, x, residual, cos, sin, doc_start)
            else:
                x, residual = layer(x, residual, cos, sin, doc_start)
            if eng is not None:
                x, residual = eng.post_layer(i, layer, x, residual)
        if eng is not None:
            x, residual = eng.pre_head(x, residual)
        y, _ = m.norm(x, residual)
        logits = self.lm_head(y.reshape(B * S, -1))  # [T, V], a fresh tensor the loss may consume
        loss = None
        if labels is not None:
            tgt = ref.shift_labels(labels)
            if doc_start is not None:
                tgt = ref.drop_cross_document_targets(tgt, doc_start)
            tgt = tgt.reshape(-1)
            if return_logits:
                loss = ops.cross_entropy(logits.clone(), tgt)
            else:
                loss = ops.cross_entropy(logits, tgt)
                logits = None  # its storage now holds dlogits (CUDA path)
        if logits is not None:
            logits = logits.view(B, S, -1)
        return SimpleNamespace(loss=loss, logits=logits)


def build_llama(config: ModelConfig, dtype=torch.bfloat16, device=None, tp_size=1, init=True, seed=None):
    if seed is not None:
        torch.manual_seed(seed)
    model = LlamaForCausalLM(config, dtype=dtype, device=device, tp_size=tp_size)
    if init and (device is None or torch.device(device).type != "meta"):
        model.init_weights()
    return model
