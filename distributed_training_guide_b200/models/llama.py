"""Llama-family causal LM built on the sm_90a op layer (Llama; Mistral: Llama plus a sliding attention window; Qwen3:
Llama plus QK-norm, with a head_dim of its own; Qwen2: Llama plus q/k/v biases; OLMo 2: Llama with a full-width
QK-norm and RMSNorms after each sublayer instead of before it; StarCoder2: Llama with LayerNorms, a c_fc -> GELU-tanh
-> c_proj MLP and a bias on every projection; GPT-NeoX: StarCoder2's parameters with a parallel residual, partial
rotary embeddings and an exact GELU; OLMoE: Llama with OLMo 2's full-width QK-norm and a mixture-of-experts MLP; Qwen3-MoE: Qwen3 with OLMoE's
mixture-of-experts MLP, its routing weights optionally renormalised).  One ``LlamaDecoderLayer`` builds every family's layer from its
``ModelConfig``, and ``decoder_layout`` fixes its flat-buffer layout.

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

    def attend(self, qkv, cos, sin, doc_start=None):
        """Attention from the fused q|k|v projection ``qkv`` [B,S,(nh + 2 nkv) d]: position the q and k heads, then
        attend.  Returns [B, S, nh d]."""
        B, S, _ = qkv.shape
        qkv = self.position_qk_(qkv.view(B, S, self.num_heads + 2 * self.num_kv_heads, self.head_dim), cos, sin)
        a = ops.attention_qkv(qkv, self.num_heads, self.num_kv_heads, doc_start=doc_start, window=self.sliding_window)
        return a.reshape(B, S, self.num_heads * self.head_dim)


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


class OlmoeExperts(nn.Module):
    """Every expert's SwiGLU weights in two 3-D parameters (transformers 5's layout): ``gate_up_proj`` [E, 2I, H]
    (each expert's gate rows, then its up rows) and ``down_proj`` [E, H, I]."""

    def __init__(self, config: ModelConfig, dtype=None, device=None):
        super().__init__()
        e, h, i = config.num_experts, config.hidden_size, config.intermediate_size
        self.gate_up_proj = nn.Parameter(torch.empty(e, 2 * i, h, dtype=dtype, device=device))
        self.down_proj = nn.Parameter(torch.empty(e, h, i, dtype=dtype, device=device))


class OlmoeMoE(nn.Module):
    """The sparse MLP of OLMoE and Qwen3-MoE (the same parameters): the router ``gate`` [E, H] and the experts
    (``ops.moe``); Qwen3-MoE may renormalise each token's routing weights (``norm_topk_prob``)."""

    def __init__(self, config: ModelConfig, dtype=None, device=None):
        super().__init__()
        self.top_k = config.num_experts_per_tok
        self.norm_topk_prob = config.norm_topk_prob
        self.gate = Linear(config.hidden_size, config.num_experts, dtype, device)
        self.experts = OlmoeExperts(config, dtype, device)


class FusedWeight:
    """A fused [q|k|v] or [gate|up] weight: adjacent parameters of a flat buffer seen as one
    matrix, plus the matching view of the flat gradient buffer (see ops._emit_weight_grad)."""

    def __init__(self, data, grad):
        self.data = data
        self._dtg_grad = grad
        self._dtg_writes = 0
        self._dtg_ready_hook = None


def decoder_layout(config: ModelConfig):
    """``(flat_order, fused)`` of a decoder layer of ``config``.

    ``flat_order`` is the layer's parameter order in its flat buffer (parallel/flat.py, parallel/fsdp.py), which also
    fixes FSDP's shard boundaries and the sharded checkpoint layout; a parameter missing from it would get
    no gradient buffer and no optimizer update.  The matrices come first, with q|k|v and gate|up adjacent so that
    their fused weights are views of the buffer.  The norms' gains (and LayerNorm biases) follow, then the QK-norm
    gains, so every replicated gain sits in one run after the matrices (TP sums their
    gradients over the group in one launch).  Then the q|k|v biases: adjacent, and each a multiple of 8 elements, so
    they form one [(nh + 2 nkv) d] bias (``fused_view_1d``) next to the fused q|k|v weight.  The o_proj and MLP
    biases come last.

    ``fused`` maps each fused weight (``qkv``, ``gate_up`` with the SwiGLU MLP, ``qkv_bias`` with q/k/v biases) to
    its member parameter names."""
    qkv = ("self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight")
    if config.gelu_mlp:
        mlp, mlp_bias = ("mlp.c_fc.weight", "mlp.c_proj.weight"), ("mlp.c_fc.bias", "mlp.c_proj.bias")
    elif config.moe:
        mlp, mlp_bias = ("mlp.gate.weight", "mlp.experts.gate_up_proj", "mlp.experts.down_proj"), ()
    else:
        mlp, mlp_bias = ("mlp.gate_proj.weight", "mlp.up_proj.weight", "mlp.down_proj.weight"), ()
    norms = (("post_attention_layernorm", "post_feedforward_layernorm") if config.post_norm else
             ("input_layernorm", "post_attention_layernorm"))
    gains = tuple(f"{n}.{p}" for n in norms for p in (("weight", "bias") if config.layer_norm else ("weight",)))
    qk_norm = ("self_attn.q_norm.weight", "self_attn.k_norm.weight") if config.qk_norm or config.full_qk_norm else ()
    qkv_bias = (("self_attn.q_proj.bias", "self_attn.k_proj.bias", "self_attn.v_proj.bias")
                if config.qkv_bias or config.all_bias else ())
    o_bias = ("self_attn.o_proj.bias",) if config.all_bias else ()
    fused = {"qkv": qkv}
    if not config.gelu_mlp and not config.moe:
        fused["gate_up"] = mlp[:2]
    if qkv_bias:
        fused["qkv_bias"] = qkv_bias
    return qkv + ("self_attn.o_proj.weight",) + mlp + gains + qk_norm + qkv_bias + o_bias + mlp_bias, fused


class LlamaDecoderLayer(nn.Module):
    """The decoder layer of every family, built from its config: RMSNorms or LayerNorms (``layer_norm``), the SwiGLU
    ``LlamaMLP`` or the c_fc -> GELU -> c_proj ``Starcoder2MLP`` (``gelu_mlp``), and one of three residual schemes:

      * pre-norm (Llama, Mistral, Qwen2.5, Qwen3, StarCoder2): ``h1 = h + attn(norm_in(h))``,
        ``h2 = h1 + mlp(norm_pa(h1))``, each add deferred into the next norm's kernel;
      * ``post_norm`` (OLMo 2): no ``input_layernorm``, ``h1 = h + norm_pa(attn(h))``, ``h2 = h1 + norm_pf(mlp(h1))``;
      * ``parallel_residual`` (GPT-NeoX): ``h' = h + attn(ln1(h)) + mlp(ln2(h))``, both norms of the same h."""

    def __init__(self, config: ModelConfig, layer_idx: int, dtype=None, device=None, tp_size=1):
        super().__init__()
        self.layer_idx = layer_idx
        self.self_attn = LlamaAttention(config, dtype, device, tp_size)
        if config.gelu_mlp:
            assert tp_size == 1, f"{config.arch} layers are not tensor-parallel"
            self.mlp = Starcoder2MLP(config, dtype, device)
        elif config.moe:
            assert tp_size == 1, f"{config.arch} layers are not tensor-parallel"
            self.mlp = OlmoeMoE(config, dtype, device)
        else:
            self.mlp = LlamaMLP(config, dtype, device, tp_size)
        Norm, eps = (LayerNorm, config.layer_norm_epsilon) if config.layer_norm else (RMSNorm, config.rms_norm_eps)
        if not config.post_norm:
            self.input_layernorm = Norm(config.hidden_size, eps, dtype, device)
        self.post_attention_layernorm = Norm(config.hidden_size, eps, dtype, device)
        if config.post_norm:
            self.post_feedforward_layernorm = Norm(config.hidden_size, eps, dtype, device)
        self.post_norm, self.parallel_residual, self.gelu_exact = (config.post_norm, config.parallel_residual,
                                                                   config.gelu_exact)
        self.flat_order, self.fused = decoder_layout(config)
        self._fused = {}  # name -> FusedWeight, installed by parallel.flat.install_fused_views
        self.tp = None  # set through LlamaForCausalLM.tp: the layer runs TensorParallelRuntime.layer_forward
        self.fp8 = False  # set through LlamaForCausalLM.fp8: the projections run in fp8
        #: OLMoE: (assignments per expert int32 [E], router probability column sums fp32 [E]) of the forward in flight;
        #: the model's forward takes them and sets this back to None
        self.router_stats = None

    def fused_weight(self, name):
        """(fused weight ``name``, its flat-gradient owner).  That is the ``FusedWeight`` view the flat group
        installed wherever the projection writes the flat gradient through it: the wgmma GEMM, and the
        tensor-parallel projections, which route it on the CPU too.  Otherwise it is the members concatenated, with no
        owner, so that autograd reaches them.  (None, None) for a fused weight the layer does not have."""
        members = self.fused.get(name)
        if members is None:
            return None, None
        f = self._fused.get(name)
        if f is not None and (self.tp is not None or _ext.use_cuda_kernel("gemm", f.data)):
            return f.data, f
        return torch.cat([self.get_parameter(m) for m in members]), None

    def _proj(self, x, w, bias=None, owner=None, bias_owner=None):
        """Every projection of the layer, in fp8 or bf16."""
        return ops.linear(x, w, bias, owner, bias_owner, fp8=self.fp8)

    def _attention(self, y, cos, sin, doc_start):
        """Attention of the normed stream ``y`` [B,S,H] up to the o_proj: [B, S, nh d]."""
        w, owner = self.fused_weight("qkv")
        b, b_owner = self.fused_weight("qkv_bias")
        return self.self_attn.attend(self._proj(y, w, b, owner, b_owner), cos, sin, doc_start)

    def _mlp_act(self, y):
        """The MLP up to its down-projection: SwiGLU on the fused gate|up, or c_fc -> GELU (exact for GPT-NeoX, the
        tanh form for StarCoder2)."""
        if isinstance(self.mlp, LlamaMLP):
            w, owner = self.fused_weight("gate_up")
            return ops.swiglu(self._proj(y, w, owner=owner))
        up = self._proj(y, self.mlp.c_fc.weight, self.mlp.c_fc.bias)
        return ops.gelu(up) if self.gelu_exact else ops.gelu_tanh(up)

    def _mlp(self, y):
        if isinstance(self.mlp, OlmoeMoE):
            m = self.mlp
            out, psum, counts = ops.moe(y, m.gate.weight, m.experts.gate_up_proj, m.experts.down_proj, m.top_k,
                                        m.norm_topk_prob)
            self.router_stats = (counts, psum)
            return out
        down = self.mlp.down_proj if isinstance(self.mlp, LlamaMLP) else self.mlp.c_proj
        return self._proj(self._mlp_act(y), down.weight, down.bias)

    def forward(self, x, residual, cos, sin, doc_start=None):
        """x: [B,S,H] branch output of the previous layer (or the embeddings);
        residual: running residual stream *before* adding x (None for the first layer);
        doc_start: None or int32 [B,S] from ``ops.document_starts`` (attention stays inside each document).
        Returns (branch, residual) with the final add again deferred to the consumer."""
        if self.tp is not None:
            return self.tp.layer_forward(self, x, residual, cos, sin)
        o = self.self_attn.o_proj
        if self.post_norm:
            # the pending add would need this layer's post_feedforward_layernorm gain, which FSDP may reshard before
            # the next layer runs, so the layer completes its stream and returns (h2, None): every layer sees
            # residual = None
            assert residual is None, "an OLMo 2 layer takes the complete residual stream"
            n1, n2 = self.post_attention_layernorm, self.post_feedforward_layernorm
            h1 = ops.rms_norm_add(self._proj(self._attention(x, cos, sin, doc_start), o.weight), x, n1.weight, n1.eps)
            return ops.rms_norm_add(self._mlp(h1), h1, n2.weight, n2.eps), None
        if self.parallel_residual:
            # the attention dense and the MLP down-projection write one branch
            n1, n2, c_proj = self.input_layernorm, self.post_attention_layernorm, self.mlp.c_proj
            y1, y2, h = ops.layer_norm2(x, residual, n1.weight, n1.bias, n2.weight, n2.bias, n1.eps)
            a = self._attention(y1, cos, sin, doc_start)
            out = ops.parallel_out(a, self._mlp_act(y2), o.weight, c_proj.weight, o.bias, c_proj.bias, fp8=self.fp8)
            return out, h
        y, h = self.input_layernorm(x, residual)
        a = self._attention(y, cos, sin, doc_start)
        y, h = self.post_attention_layernorm(self._proj(a, o.weight, o.bias), h)
        return self._mlp(y), h


class LlamaModel(nn.Module):
    def __init__(self, config: ModelConfig, dtype=None, device=None, tp_size=1):
        super().__init__()
        assert config.hidden_size % tp_size == 0
        # tensor parallel: the table is sharded over the hidden dimension (reference: ColwiseParallel on
        # nn.Embedding, 06-tensor-parallel/train_llm.py:82)
        self.embed_tokens = Embedding(config.vocab_size, config.hidden_size // tp_size, dtype, device)
        self.layers = nn.ModuleList(
            [LlamaDecoderLayer(config, i, dtype, device, tp_size) for i in range(config.num_hidden_layers)]
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
        #: OLMoE load balancing (``--router-aux-loss-coef``): loss = CE + coef * ``ref.router_aux_loss`` over every
        #: layer's tokens; 0 trains on the cross entropy alone
        self.router_aux_loss_coef = 0.0

    @property
    def fp8(self) -> bool:
        """Run the decoder-layer projections (q|k|v, o, gate|up, down) in fp8 (``ops.linear(..., fp8=True)``): fp8
        GEMMs with per-tensor current scaling.  The lm_head, embedding, attention, norms and loss stay bf16."""
        return self._fp8

    @fp8.setter
    def fp8(self, on: bool):
        self._fp8 = bool(on)
        for layer in self.model.layers:
            layer.fp8 = self._fp8

    @property
    def tp(self):
        """The ``parallel.tp.TensorParallelRuntime`` that runs the model's and its layers' forward, or None."""
        return self._tp

    @tp.setter
    def tp(self, runtime):
        self._tp = runtime
        for layer in self.model.layers:
            layer.tp = runtime

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
    def decoder(self, input_ids, cos, sin, doc_start=None, embed=None):
        """The embedding, every decoder layer and the final norm, with the engine's hooks around them and activation
        checkpointing.  ``embed`` replaces the embedding lookup (tensor parallelism's hidden-parallel one).  Returns
        the final norm's output."""
        m, eng = self.model, self.engine
        if eng is not None:
            eng.pre_forward(self)
        x = (embed or m.embed_tokens)(input_ids)
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
        return m.norm(x, residual)[0]

    def forward(self, input_ids, attention_mask=None, labels=None, position_ids=None, return_logits=None):
        """``attention_mask`` is accepted for API parity; the data pipeline only produces full
        (unpadded) chunks so only the causal mask is applied (the reference's all-ones mask
        collapses to the same thing inside transformers, SURVEY.md K3).  With ``document_masking``
        and ``position_ids``, attention and targets stay inside each packed document."""
        B, S = input_ids.shape
        m = self.model
        if position_ids is None:
            cos, sin = m.rotary_emb.tables(S, input_ids.device)
        else:
            cos, sin = m.rotary_emb(position_ids)
        if self.tp is not None:
            return self.tp.model_forward(self, input_ids, labels, cos, sin)
        doc_start = None
        if self.document_masking and position_ids is not None:
            doc_start = ops.document_starts(position_ids)
        aux = self.router_aux_loss_coef > 0 and labels is not None
        if aux and self.activation_checkpointing and torch.is_grad_enabled():
            raise ValueError("the router aux loss needs the router probabilities' graph, which activation "
                             "checkpointing drops: train with --router-aux-loss-coef 0 or without "
                             "--checkpoint-activations")
        y = self.decoder(input_ids, cos, sin, doc_start)
        # the router statistics are read here and nowhere else: a layer must not keep them past its forward, because
        # their autograd graph reaches the engine's boundaries, whose callbacks hold the engine and so the model, and
        # that cycle runs through autograd nodes the garbage collector cannot see (the model would never be freed)
        stats = [layer.router_stats for layer in m.layers] if self.config.moe else None
        if stats is not None:
            for layer in m.layers:
                layer.router_stats = None
        logits = self.lm_head(y.reshape(B * S, -1))  # [T, V], a fresh tensor the loss may consume
        loss = aux_loss = None
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
            if aux:
                aux_loss = ref.router_aux_loss([c for c, _ in stats], [p for _, p in stats], B * S,
                                               self.config.num_experts)
                loss = loss + self.router_aux_loss_coef * aux_loss
        if logits is not None:
            logits = logits.view(B, S, -1)
        if aux_loss is not None:
            return SimpleNamespace(loss=loss, logits=logits, aux_loss=aux_loss)
        return SimpleNamespace(loss=loss, logits=logits)


def build_llama(config: ModelConfig, dtype=torch.bfloat16, device=None, tp_size=1, init=True, seed=None):
    if seed is not None:
        torch.manual_seed(seed)
    model = LlamaForCausalLM(config, dtype=dtype, device=device, tp_size=tp_size)
    if init and (device is None or torch.device(device).type != "meta"):
        model.init_weights()
    return model
