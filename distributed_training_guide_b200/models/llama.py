"""Llama-family causal LM built on the sm_90a op layer (Llama, and Mistral: Llama plus a sliding attention window).

Same module tree and parameter names as ``transformers``' ``LlamaForCausalLM`` (what
the reference instantiates at e.g. ``02-distributed-data-parallel/train_llm.py:57-58``)
so checkpoints keep meaningful keys: ``model.embed_tokens.weight``,
``model.layers.{i}.self_attn.{q,k,v,o}_proj.weight``, ``model.layers.{i}.mlp.
{gate,up,down}_proj.weight``, ``...{input,post_attention}_layernorm.weight``,
``model.norm.weight``, ``lm_head.weight``.

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
    gen = torch.Generator(device=p.device)
    gen.manual_seed(_name_seed(seed, name))
    shape = tuple(full_shape) if full_shape is not None else tuple(p.shape)
    full = torch.empty(shape, dtype=torch.float32, device=p.device).normal_(0.0, std, generator=gen)
    if shard_dim is not None and shard_count > 1:
        full = full.chunk(shard_count, dim=shard_dim)[shard_index]
    p.copy_(full.to(p.dtype))


#: which dimension of each parameter tensor parallelism splits (None = replicated)
TP_SHARD_DIM = {"q_proj": 0, "k_proj": 0, "v_proj": 0, "gate_proj": 0, "up_proj": 0, "o_proj": 1, "down_proj": 1,
                "embed_tokens": 1, "lm_head": 0}


def tp_shard_spec(name: str, p, tp_size: int, tp_rank: int) -> dict:
    """init_parameter_ kwargs that make rank ``tp_rank`` hold its slice of the full parameter."""
    if tp_size == 1:
        return {}
    for key, dim in TP_SHARD_DIM.items():
        if f"{key}.weight" in name:
            full = list(p.shape)
            full[dim] *= tp_size
            return dict(full_shape=full, shard_dim=dim, shard_index=tp_rank, shard_count=tp_size)
    return {}


class Linear(nn.Module):
    """Bias-free projection holding ``weight`` [out, in] (HF naming)."""

    def __init__(self, in_features, out_features, dtype=None, device=None):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.weight = nn.Parameter(torch.empty(out_features, in_features, dtype=dtype, device=device))

    def forward(self, x):
        return ops.linear(x, self.weight)

    def reset_parameters(self, std=0.02):
        nn.init.normal_(self.weight, mean=0.0, std=std)


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
        self.head_dim = config.head_dim
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
        #: sliding-window attention (Mistral): None, or W >= 1 with query q seeing keys k > q - W only
        self.sliding_window = config.sliding_window
        self.q_proj = Linear(h, self.num_heads * d, dtype, device)
        self.k_proj = Linear(h, self.num_kv_heads * d, dtype, device)
        self.v_proj = Linear(h, self.num_kv_heads * d, dtype, device)
        self.o_proj = Linear(self.num_heads * d, h, dtype, device)


class LlamaMLP(nn.Module):
    def __init__(self, config: ModelConfig, dtype=None, device=None, tp_size=1):
        super().__init__()
        h, i = config.hidden_size, config.intermediate_size
        assert i % tp_size == 0
        self.gate_proj = Linear(h, i // tp_size, dtype, device)
        self.up_proj = Linear(h, i // tp_size, dtype, device)
        self.down_proj = Linear(i // tp_size, h, dtype, device)


class FusedWeight:
    """A fused [q|k|v] or [gate|up] weight: adjacent parameters of a flat buffer seen as one
    matrix, plus the matching view of the flat gradient buffer (see ops._emit_weight_grad)."""

    def __init__(self, data, grad):
        self.data = data
        self._dtg_grad = grad
        self._dtg_writes = 0
        self._dtg_ready_hook = None


class LlamaDecoderLayer(nn.Module):
    #: parameter order inside a layer's flat buffer; adjacency is what makes fusion free
    FLAT_ORDER = (
        "self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight",
        "self_attn.o_proj.weight", "mlp.gate_proj.weight", "mlp.up_proj.weight",
        "mlp.down_proj.weight", "input_layernorm.weight", "post_attention_layernorm.weight",
    )
    FUSED = {"qkv": FLAT_ORDER[0:3], "gate_up": FLAT_ORDER[4:6]}

    def __init__(self, config: ModelConfig, layer_idx: int, dtype=None, device=None, tp_size=1):
        super().__init__()
        self.layer_idx = layer_idx
        self.self_attn = LlamaAttention(config, dtype, device, tp_size)
        self.mlp = LlamaMLP(config, dtype, device, tp_size)
        self.input_layernorm = RMSNorm(config.hidden_size, config.rms_norm_eps, dtype, device)
        self.post_attention_layernorm = RMSNorm(config.hidden_size, config.rms_norm_eps, dtype, device)
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
        qkv = fused_linear(y, w, owner).view(B, S, att.num_heads + 2 * att.num_kv_heads, att.head_dim)
        qkv = ops.rope_qkv_(qkv, cos, sin, att.num_heads + att.num_kv_heads)
        a = ops.attention_qkv(qkv, att.num_heads, att.num_kv_heads, doc_start=doc_start, window=att.sliding_window)
        a = a.reshape(B, S, att.num_heads * att.head_dim)
        a = ops.fp8_linear(a, att.o_proj.weight) if self.fp8 else att.o_proj(a)
        y, h = self.post_attention_layernorm(a, h)
        w, owner = self._gate_up_weight()
        act = ops.swiglu(fused_linear(y, w, owner))
        down = ops.fp8_linear(act, self.mlp.down_proj.weight) if self.fp8 else self.mlp.down_proj(act)
        return down, h


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
