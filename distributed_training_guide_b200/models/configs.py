"""Embedded model configurations.

The GPU boxes have no network, so the handful of Hugging Face model ids the
guide uses (reference: every chapter's ``-m/--model-name`` flag, e.g.
``02-distributed-data-parallel/train_llm.py:57``) are resolved from this table
instead of the hub.  A local directory containing a ``config.json`` is also
accepted, and tiny ``debug-*`` configs exist for tests.  Families: Llama 2 / 3 / 3.1 / 3.2, Mistral, Qwen3, Qwen2.5,
OLMo 2 (``allenai/OLMo-2-*``, ``model_type: "olmo2"``), OLMoE (``allenai/OLMoE-*``, ``model_type: "olmoe"``), Qwen3-MoE
(``Qwen/Qwen3-30B-A3B``, ``Qwen/Qwen3-235B-A22B``, ``model_type: "qwen3_moe"``), StarCoder2 (``bigcode/starcoder2-*``,
``model_type: "starcoder2"``), GPT-NeoX / Pythia (``EleutherAI/pythia-*``, ``model_type: "gpt_neox"``) and GPT-2.
"""
from __future__ import annotations

import dataclasses
import json
import os
from typing import Optional


@dataclasses.dataclass
class ModelConfig:
    arch: str  # "llama" | "mistral" | "qwen3" | "qwen2" | "olmo2" | "olmoe" | "qwen3_moe" | "starcoder2" | "gpt_neox" |
    # "gpt2"; mistral is
    # llama with a sliding attention window, qwen3 llama with QK-norm and a head_dim of its own, qwen2 llama with q/k/v
    # biases, olmo2 llama with a full-width QK-norm and post-sublayer norms instead of the pre-norms (``full_qk_norm``,
    # ``post_norm``), starcoder2 llama with LayerNorms, a GELU MLP and biases on every projection (``layer_norm``,
    # ``gelu_mlp``, ``all_bias``), gpt_neox starcoder2's block with a parallel residual, partial rotary embeddings
    # and an exact GELU (``parallel_residual``, ``rotary_dim``, ``gelu_exact``), olmoe llama with OLMo 2's full-width
    # QK-norm (still pre-norm) and a mixture-of-experts MLP (``moe``), qwen3_moe qwen3 with olmoe's MLP
    # (``intermediate_size`` is then each expert's, HF's ``moe_intermediate_size``)
    vocab_size: int
    hidden_size: int
    intermediate_size: int
    num_hidden_layers: int
    num_attention_heads: int
    num_key_value_heads: int
    max_position_embeddings: int
    rms_norm_eps: float = 1e-5
    rope_theta: float = 10000.0
    rope_scaling: Optional[dict] = None
    tie_word_embeddings: bool = False
    #: sliding-window attention (Mistral): query q sees only the ``sliding_window`` most recent keys, k > q - W
    sliding_window: Optional[int] = None
    #: per-head dimension when it is not hidden_size // num_attention_heads (Qwen3: 128 at every size); None derives
    #: it from the hidden size.  Read it through ``head_dim``.
    explicit_head_dim: Optional[int] = None
    #: QK-norm (Qwen3): every q and k head is RMS-normalised and scaled by a [head_dim] gain before RoPE
    qk_norm: bool = False
    #: q/k/v projection biases (Qwen2); o_proj and the MLP stay bias-free
    qkv_bias: bool = False
    # gpt2, starcoder2 and gpt_neox (their LayerNorms' eps)
    layer_norm_epsilon: float = 1e-5
    #: share of each q/k head that RoPE rotates (GPT-NeoX's ``rotary_pct``); read it through ``rotary_dim``
    partial_rotary_factor: float = 1.0
    dropout: float = 0.0
    #: mixture of experts (OLMoE): ``num_experts`` SwiGLU experts of ``intermediate_size`` each, and the
    #: ``num_experts_per_tok`` of them with the highest router probability run on each token
    num_experts: int = 0
    num_experts_per_tok: int = 0
    #: Qwen3-MoE: each token's routing weights are its top-k probabilities divided by their sum, not the raw ones
    norm_topk_prob: bool = False
    name: str = ""

    @property
    def head_dim(self) -> int:
        if self.explicit_head_dim is not None:
            return self.explicit_head_dim
        return self.hidden_size // self.num_attention_heads

    @property
    def rotary_dim(self) -> int:
        """Leading elements of each q/k head that RoPE rotates (head_dim unless ``partial_rotary_factor`` < 1)."""
        return int(self.head_dim * self.partial_rotary_factor)

    @property
    def parallel_residual(self) -> bool:
        """GPT-NeoX's layer: h' = h + attn(ln1(h)) + mlp(ln2(h)), both norms of the same h."""
        return self.arch == "gpt_neox"

    @property
    def full_qk_norm(self) -> bool:
        """OLMo 2's QK-norm: one RMSNorm over each token's whole q (nh * head_dim) and one over its whole k (nkv *
        head_dim), with gains of those lengths.  Exclusive of Qwen3's per-head ``qk_norm``.  OLMoE has it too."""
        return self.arch in ("olmo2", "olmoe")

    @property
    def post_norm(self) -> bool:
        """OLMo 2's layer: no input_layernorm; h1 = h + norm(attn(h)), h2 = h1 + norm(mlp(h1))."""
        return self.arch == "olmo2"

    @property
    def moe(self) -> bool:
        """OLMoE's and Qwen3-MoE's MLP: a router picks each token's top ``num_experts_per_tok`` of ``num_experts``
        SwiGLU experts and sums their outputs weighted by the router probabilities, raw or renormalised
        (``norm_topk_prob``) (``ops.moe``)."""
        return self.arch in ("olmoe", "qwen3_moe")

    @property
    def layer_norm(self) -> bool:
        """StarCoder2, GPT-NeoX: LayerNorms with a gain and a bias (eps ``layer_norm_epsilon``) instead of the
        RMSNorms."""
        return self.arch in ("starcoder2", "gpt_neox")

    @property
    def gelu_mlp(self) -> bool:
        """StarCoder2's and GPT-NeoX's MLP: c_fc -> GELU -> c_proj instead of SwiGLU's three matrices; the GELU is
        the tanh approximation (StarCoder2) or exact (``gelu_exact``, GPT-NeoX)."""
        return self.arch in ("starcoder2", "gpt_neox")

    @property
    def gelu_exact(self) -> bool:
        """GPT-NeoX: the MLP's GELU is the exact erf form (``hidden_act: "gelu"``), not StarCoder2's tanh form."""
        return self.arch == "gpt_neox"

    @property
    def all_bias(self) -> bool:
        """StarCoder2, GPT-NeoX: every projection (q, k, v, o, c_fc, c_proj) has a bias; the lm_head has none."""
        return self.arch in ("starcoder2", "gpt_neox")

    def num_parameters(self) -> int:
        h, i, v, l = self.hidden_size, self.intermediate_size, self.vocab_size, self.num_hidden_layers
        if self.arch == "gpt2":
            per_layer = (3 * h * h + 3 * h) + (h * h + h) + (h * i + i) + (i * h + h) + 4 * h
            return v * h + self.max_position_embeddings * h + l * per_layer + 2 * h
        q = self.num_attention_heads * self.head_dim
        kv = self.num_key_value_heads * self.head_dim
        if self.arch in ("starcoder2", "gpt_neox"):   # the same tensors: only the forward differs
            per_layer = (h * q + q) + 2 * (kv * h + kv) + (q * h + h) + (h * i + i) + (i * h + h) + 4 * h
            n = v * h + l * per_layer + 2 * h
            return n if self.tie_word_embeddings else n + v * h
        per_layer = h * q + 2 * kv * h + q * h + 2 * h
        per_layer += self.num_experts * (h + 3 * h * i) if self.moe else 3 * h * i
        if self.qk_norm:
            per_layer += 2 * self.head_dim
        if self.qkv_bias:
            per_layer += q + 2 * kv
        if self.full_qk_norm:
            per_layer += q + kv
        n = v * h + l * per_layer + h
        if not self.tie_word_embeddings:
            n += v * h
        return n

    def to_dict(self) -> dict:
        return dataclasses.asdict(self)


_LLAMA3_SCALING = {
    "rope_type": "llama3",
    "factor": 8.0,
    "low_freq_factor": 1.0,
    "high_freq_factor": 4.0,
    "original_max_position_embeddings": 8192,
}


# Llama 3.2 (1B / 3B): the llama3 rule with a factor of 32
_LLAMA32_SCALING = {**_LLAMA3_SCALING, "factor": 32.0}


def _llama(name, v, h, i, l, nh, nkv, maxpos, theta, scaling=None, tied=False):
    return ModelConfig(
        arch="llama", vocab_size=v, hidden_size=h, intermediate_size=i, num_hidden_layers=l,
        num_attention_heads=nh, num_key_value_heads=nkv, max_position_embeddings=maxpos,
        rms_norm_eps=1e-5, rope_theta=theta, rope_scaling=scaling, tie_word_embeddings=tied, name=name,
    )


def _mistral(name, v, h, i, l, nh, nkv, maxpos, theta, window):
    return dataclasses.replace(_llama(name, v, h, i, l, nh, nkv, maxpos, theta), arch="mistral", sliding_window=window)


def _qwen3(name, h, i, l, nh, nkv, tied, v=151936, maxpos=40960):
    return ModelConfig(
        arch="qwen3", vocab_size=v, hidden_size=h, intermediate_size=i, num_hidden_layers=l,
        num_attention_heads=nh, num_key_value_heads=nkv, max_position_embeddings=maxpos,
        rms_norm_eps=1e-6, rope_theta=1e6, tie_word_embeddings=tied, explicit_head_dim=128, qk_norm=True, name=name,
    )


def _qwen2(name, h, i, l, nh, nkv, tied, v, maxpos):
    return ModelConfig(
        arch="qwen2", vocab_size=v, hidden_size=h, intermediate_size=i, num_hidden_layers=l,
        num_attention_heads=nh, num_key_value_heads=nkv, max_position_embeddings=maxpos,
        rms_norm_eps=1e-6, rope_theta=1e6, tie_word_embeddings=tied, qkv_bias=True, name=name,
    )


def _olmo2(name, h, i, l, nh, nkv, v=100352, maxpos=4096):
    return ModelConfig(
        arch="olmo2", vocab_size=v, hidden_size=h, intermediate_size=i, num_hidden_layers=l,
        num_attention_heads=nh, num_key_value_heads=nkv, max_position_embeddings=maxpos,
        rms_norm_eps=1e-6, rope_theta=5e5, tie_word_embeddings=False, name=name,
    )


def _olmoe(name, h, i, l, nh, nkv, experts, top_k, v=50304, maxpos=4096):
    return ModelConfig(
        arch="olmoe", vocab_size=v, hidden_size=h, intermediate_size=i, num_hidden_layers=l,
        num_attention_heads=nh, num_key_value_heads=nkv, max_position_embeddings=maxpos,
        rms_norm_eps=1e-5, rope_theta=1e4, tie_word_embeddings=False, num_experts=experts, num_experts_per_tok=top_k,
        name=name,
    )


def _qwen3_moe(name, h, i, l, nh, nkv, experts, top_k, v=151936, maxpos=40960, norm_topk_prob=True):
    return dataclasses.replace(_qwen3(name, h, i, l, nh, nkv, False, v=v, maxpos=maxpos), arch="qwen3_moe",
                               num_experts=experts, num_experts_per_tok=top_k, norm_topk_prob=norm_topk_prob)


def _starcoder2(name, h, i, l, nh, nkv, theta, tied, v=49152, maxpos=16384, window=4096):
    return ModelConfig(
        arch="starcoder2", vocab_size=v, hidden_size=h, intermediate_size=i, num_hidden_layers=l,
        num_attention_heads=nh, num_key_value_heads=nkv, max_position_embeddings=maxpos, rope_theta=theta,
        tie_word_embeddings=tied, sliding_window=window, layer_norm_epsilon=1e-5, name=name,
    )


def _gpt_neox(name, h, i, l, nh, v=50304, rotary=0.25, tied=False, maxpos=2048):
    return ModelConfig(
        arch="gpt_neox", vocab_size=v, hidden_size=h, intermediate_size=i, num_hidden_layers=l,
        num_attention_heads=nh, num_key_value_heads=nh, max_position_embeddings=maxpos, rope_theta=1e4,
        tie_word_embeddings=tied, layer_norm_epsilon=1e-5, partial_rotary_factor=rotary, name=name,
    )


_PYTHIA = {   # size: (hidden, intermediate, layers, heads, vocab)
    "70m": (512, 2048, 6, 8, 50304), "160m": (768, 3072, 12, 12, 50304), "410m": (1024, 4096, 24, 16, 50304),
    "1.4b": (2048, 8192, 24, 16, 50304), "6.9b": (4096, 16384, 32, 32, 50432), "12b": (5120, 20480, 36, 40, 50688),
}


_GPT2 = ModelConfig(
    arch="gpt2", vocab_size=50257, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
    num_attention_heads=12, num_key_value_heads=12, max_position_embeddings=1024,
    tie_word_embeddings=True, layer_norm_epsilon=1e-5, dropout=0.1, name="openai-community/gpt2",
)

REGISTRY = {
    "openai-community/gpt2": _GPT2,
    "gpt2": _GPT2,
    "meta-llama/Llama-2-7b-hf": _llama("meta-llama/Llama-2-7b-hf", 32000, 4096, 11008, 32, 32, 32, 4096, 1e4),
    "meta-llama/Llama-2-13b-hf": _llama("meta-llama/Llama-2-13b-hf", 32000, 5120, 13824, 40, 40, 40, 4096, 1e4),
    "meta-llama/Meta-Llama-3-8B": _llama("meta-llama/Meta-Llama-3-8B", 128256, 4096, 14336, 32, 32, 8, 8192, 5e5),
    "meta-llama/Llama-3.1-8B": _llama("meta-llama/Llama-3.1-8B", 128256, 4096, 14336, 32, 32, 8, 131072, 5e5, _LLAMA3_SCALING),
    "meta-llama/Meta-Llama-3-70B": _llama("meta-llama/Meta-Llama-3-70B", 128256, 8192, 28672, 80, 64, 8, 8192, 5e5),
    "meta-llama/Llama-3.1-70B": _llama("meta-llama/Llama-3.1-70B", 128256, 8192, 28672, 80, 64, 8, 131072, 5e5, _LLAMA3_SCALING),
    "meta-llama/Llama-3.1-405B": _llama("meta-llama/Llama-3.1-405B", 128256, 16384, 53248, 126, 128, 8, 131072, 5e5, _LLAMA3_SCALING),
    "meta-llama/Meta-Llama-3.1-405B": _llama("meta-llama/Meta-Llama-3.1-405B", 128256, 16384, 53248, 126, 128, 8, 131072, 5e5, _LLAMA3_SCALING),
    # head_dim 64 (2048 / 32) and 128 (3072 / 24), tied embeddings
    "meta-llama/Llama-3.2-1B": _llama("meta-llama/Llama-3.2-1B", 128256, 2048, 8192, 16, 32, 8, 131072, 5e5, _LLAMA32_SCALING, tied=True),
    "meta-llama/Llama-3.2-3B": _llama("meta-llama/Llama-3.2-3B", 128256, 3072, 8192, 28, 24, 8, 131072, 5e5, _LLAMA32_SCALING, tied=True),
    "mistralai/Mistral-7B-v0.1": _mistral("mistralai/Mistral-7B-v0.1", 32000, 4096, 14336, 32, 32, 8, 32768, 1e4, 4096),
    "Qwen/Qwen3-0.6B": _qwen3("Qwen/Qwen3-0.6B", 1024, 3072, 28, 16, 8, True),
    "Qwen/Qwen3-1.7B": _qwen3("Qwen/Qwen3-1.7B", 2048, 6144, 28, 16, 8, True),
    "Qwen/Qwen3-4B": _qwen3("Qwen/Qwen3-4B", 2560, 9728, 36, 32, 8, True),
    "Qwen/Qwen3-8B": _qwen3("Qwen/Qwen3-8B", 4096, 12288, 36, 32, 8, False),
    "Qwen/Qwen3-32B": _qwen3("Qwen/Qwen3-32B", 5120, 25600, 64, 64, 8, False),
    # Qwen2.5: q/k/v biases; head_dim 64 (0.5B) or 128
    "Qwen/Qwen2.5-0.5B": _qwen2("Qwen/Qwen2.5-0.5B", 896, 4864, 24, 14, 2, True, 151936, 32768),
    "Qwen/Qwen2.5-1.5B": _qwen2("Qwen/Qwen2.5-1.5B", 1536, 8960, 28, 12, 2, True, 151936, 131072),
    "Qwen/Qwen2.5-3B": _qwen2("Qwen/Qwen2.5-3B", 2048, 11008, 36, 16, 2, True, 151936, 32768),
    "Qwen/Qwen2.5-7B": _qwen2("Qwen/Qwen2.5-7B", 3584, 18944, 28, 28, 4, False, 152064, 131072),
    "Qwen/Qwen2.5-14B": _qwen2("Qwen/Qwen2.5-14B", 5120, 13824, 48, 40, 8, False, 152064, 131072),
    "Qwen/Qwen2.5-32B": _qwen2("Qwen/Qwen2.5-32B", 5120, 27648, 64, 40, 8, False, 152064, 131072),
    "Qwen/Qwen2.5-72B": _qwen2("Qwen/Qwen2.5-72B", 8192, 29568, 80, 64, 8, False, 152064, 131072),
    # OLMo 2: full-width QK-norm and post-sublayer norms; head_dim 128 at every size, untied
    "allenai/OLMo-2-0425-1B": _olmo2("allenai/OLMo-2-0425-1B", 2048, 8192, 16, 16, 16),
    "allenai/OLMo-2-1124-7B": _olmo2("allenai/OLMo-2-1124-7B", 4096, 11008, 32, 32, 32),
    "allenai/OLMo-2-1124-13B": _olmo2("allenai/OLMo-2-1124-13B", 5120, 13824, 40, 40, 40),
    "allenai/OLMo-2-0325-32B": _olmo2("allenai/OLMo-2-0325-32B", 5120, 27648, 64, 40, 8),
    # OLMoE: 64 experts of intermediate size 1024, top-8, OLMo 2's full-width QK-norm in a pre-norm layer; 6.92B
    # parameters, about 1.3B active per token.  The shapes are those of the public config.json as recalled when this
    # table was written; no copy of the file was at hand to check them against.
    "allenai/OLMoE-1B-7B-0924": _olmoe("allenai/OLMoE-1B-7B-0924", 2048, 1024, 16, 16, 16, 64, 8),
    # Qwen3-MoE: Qwen3's per-head QK-norm at head_dim 128, 128 experts, top-8 with renormalised weights, untied; the
    # intermediate size is each expert's (moe_intermediate_size).  30,532,122,624 and 235,093,634,560 parameters, as
    # transformers' Qwen3MoeForCausalLM counts them.  The shapes are those of the public config.json files as recalled
    # when this table was written; no copy of those files was at hand to check them against.
    "Qwen/Qwen3-30B-A3B": _qwen3_moe("Qwen/Qwen3-30B-A3B", 2048, 768, 48, 32, 4, 128, 8),
    "Qwen/Qwen3-30B-A3B-Base": _qwen3_moe("Qwen/Qwen3-30B-A3B-Base", 2048, 768, 48, 32, 4, 128, 8),
    "Qwen/Qwen3-235B-A22B": _qwen3_moe("Qwen/Qwen3-235B-A22B", 4096, 1536, 94, 64, 4, 128, 8),
    # StarCoder2: LayerNorms, a GELU MLP, biases on every projection, sliding window 4096; head_dim 128 at every size.
    # Shapes, RoPE theta, window, norm eps and max positions are those of the public config.json files as recalled
    # when this table was written; no copy of those files was at hand to check them against.  transformers'
    # Starcoder2Config defaults (the 3B shapes: 3072 / 12288 / 30 layers / 24:2 heads, vocab 49152, eps 1e-5, tied)
    # agree with the 3B row.  The tie flags follow the published parameter counts: 3.03B and 7.17B are the tied
    # counts of the 3B and 7B shapes, and about 16B (15.96B) the untied count of the 15B shape (tied would be 15.66B).
    "bigcode/starcoder2-3b": _starcoder2("bigcode/starcoder2-3b", 3072, 12288, 30, 24, 2, 999999.4420358813, True),
    "bigcode/starcoder2-7b": _starcoder2("bigcode/starcoder2-7b", 4608, 18432, 32, 36, 4, 1e6, True),
    "bigcode/starcoder2-15b": _starcoder2("bigcode/starcoder2-15b", 6144, 24576, 40, 48, 4, 1e5, False),
    # Pythia (GPT-NeoX): parallel residual, rotary on 25 % of each head, exact GELU, untied, max positions 2048; each
    # size also under its -deduped name (same shapes, trained on the deduplicated Pile).  Shapes and vocabularies are
    # those of the public config.json files as recalled when this table was written; no copy of those files was at
    # hand to check them against.  With them num_parameters() gives the published totals (70,426,624 ... 11,846,072,320
    # for 70m ... 12b).  Pythia-1b (head_dim 256) and -2.8b (head_dim 80) are outside the attention kernels' head dims.
    **{f"EleutherAI/pythia-{size}{suffix}": _gpt_neox(f"EleutherAI/pythia-{size}{suffix}", h, i, l, nh, v)
       for size, (h, i, l, nh, v) in _PYTHIA.items() for suffix in ("", "-deduped")},
    # tiny configs for tests / smoke runs (head_dim 128 so the sm_90a attention kernel applies)
    "debug-llama": _llama("debug-llama", 1024, 256, 512, 2, 2, 2, 2048, 1e4),
    "debug-llama-gqa": _llama("debug-llama-gqa", 1024, 512, 1024, 2, 4, 2, 2048, 5e5),
    "debug-llama-tp": _llama("debug-llama-tp", 2048, 1024, 2048, 2, 8, 8, 2048, 1e4),
    # 4 heads x 64 over a hidden size of 256: head_dim 64, as in Llama-3.2-1B
    "debug-llama-d64": _llama("debug-llama-d64", 1024, 256, 512, 2, 4, 2, 2048, 5e5),
    # a window that is not a multiple of the kernels' 128-row tiles
    "debug-mistral": _mistral("debug-mistral", 1024, 512, 1024, 2, 4, 2, 2048, 1e4, 192),
    # 4 heads x 128 = 512 over a hidden size of 256: head_dim apart from the hidden size, as in Qwen3-0.6B / 4B / 32B
    "debug-qwen3": _qwen3("debug-qwen3", 256, 512, 2, 4, 2, False, v=1024, maxpos=2048),
    # 4 heads x 64 over a hidden size of 256, with q/k/v biases: head_dim 64, as in Qwen2.5-0.5B
    "debug-qwen2": _qwen2("debug-qwen2", 256, 512, 2, 4, 2, False, 1024, 2048),
    # 4 q heads and 2 k heads x 128 over a hidden size of 512: GQA, and a k norm narrower than the q norm
    "debug-olmo2": _olmo2("debug-olmo2", 512, 1024, 2, 4, 2, v=1024, maxpos=2048),
    # 2 heads x 128 over a hidden size of 256, 8 experts of intermediate size 128, top-2
    "debug-olmoe": _olmoe("debug-olmoe", 256, 128, 2, 2, 2, 8, 2, v=1024, maxpos=2048),
    # 4 q heads and 2 kv heads x 128 = 512 over a hidden size of 256, 16 experts of intermediate size 128, top-4 with
    # renormalised weights
    "debug-qwen3-moe": _qwen3_moe("debug-qwen3-moe", 256, 128, 2, 4, 2, 16, 4, v=1024, maxpos=2048),
    # 4 q heads and 2 kv heads x 128 over a hidden size of 512, tied, with StarCoder2's block
    "debug-starcoder2": _starcoder2("debug-starcoder2", 512, 2048, 2, 4, 2, 1e5, True, v=1024, maxpos=2048),
    # 4 heads x 128 over a hidden size of 512 with rotary on 32 of them, and 4 heads x 64 over 256 with rotary on 16,
    # with GPT-NeoX's block
    "debug-gpt-neox": _gpt_neox("debug-gpt-neox", 512, 2048, 2, 4, v=1024),
    "debug-gpt-neox-d64": _gpt_neox("debug-gpt-neox-d64", 256, 1024, 2, 4, v=1024),
    "debug-gpt2": dataclasses.replace(_GPT2, vocab_size=512, hidden_size=64, intermediate_size=256,
                                      num_hidden_layers=2, num_attention_heads=2, num_key_value_heads=2,
                                      max_position_embeddings=128, name="debug-gpt2"),
}


def _from_hf_dict(d: dict, name: str) -> ModelConfig:
    mt = d.get("model_type", "llama")
    if mt == "gpt2":
        h = d.get("n_embd", 768)
        return ModelConfig(
            arch="gpt2", vocab_size=d.get("vocab_size", 50257), hidden_size=h,
            intermediate_size=d.get("n_inner") or 4 * h, num_hidden_layers=d.get("n_layer", 12),
            num_attention_heads=d.get("n_head", 12), num_key_value_heads=d.get("n_head", 12),
            max_position_embeddings=d.get("n_positions", 1024), tie_word_embeddings=True,
            layer_norm_epsilon=d.get("layer_norm_epsilon", 1e-5), dropout=d.get("resid_pdrop", 0.1), name=name,
        )
    if mt == "starcoder2":
        return _starcoder2_from_hf_dict(d, name)
    if mt == "gpt_neox":
        return _gpt_neox_from_hf_dict(d, name)
    if mt == "olmoe":
        return _olmoe_from_hf_dict(d, name)
    if mt == "qwen3_moe":
        return _qwen3_moe_from_hf_dict(d, name)
    if mt not in ("llama", "mistral", "qwen3", "qwen2", "olmo2"):
        raise ValueError(f"unsupported model_type {mt!r} in {name}")
    if mt == "olmo2":
        if d.get("attention_bias"):
            raise ValueError(f"{name}: attention_bias is true; OLMo 2 projections with a bias are not supported")
        rope = d.get("rope_parameters") if isinstance(d.get("rope_parameters"), dict) else d.get("rope_scaling")
        if rope and (rope.get("rope_type") or rope.get("type") or "default") != "default":
            key = "rope_parameters" if isinstance(d.get("rope_parameters"), dict) else "rope_scaling"
            raise ValueError(f"{name}: {key} has type {rope.get('rope_type') or rope.get('type')!r}; only the default "
                             "RoPE is supported for OLMo 2")
        if d.get("head_dim") is not None and d["head_dim"] != d["hidden_size"] // d["num_attention_heads"]:
            raise ValueError(f"{name}: head_dim {d['head_dim']} differs from hidden_size / num_attention_heads = "
                             f"{d['hidden_size'] // d['num_attention_heads']}; only head_dim = hidden / heads is supported")
    window = None
    head_dim = None
    if mt == "llama":
        for key in ("attention_bias", "mlp_bias"):
            if d.get(key):
                raise ValueError(f"{name}: {key} is true; Llama projections with a bias are not supported (Qwen2's "
                                 "q/k/v biases are: model_type 'qwen2')")
    if mt == "qwen2":
        if d.get("use_sliding_window"):
            raise ValueError(f"{name}: use_sliding_window is true; Qwen2 sliding-window layers are not supported")
        if "sliding_attention" in (d.get("layer_types") or ()):
            raise ValueError(f"{name}: layer_types contains 'sliding_attention'; Qwen2 sliding-window layers are "
                             "not supported")
        rope = d.get("rope_parameters") if isinstance(d.get("rope_parameters"), dict) else d.get("rope_scaling")
        if rope and (rope.get("rope_type") or rope.get("type") or "default") != "default":
            key = "rope_parameters" if isinstance(d.get("rope_parameters"), dict) else "rope_scaling"
            raise ValueError(f"{name}: {key} has type {rope.get('rope_type') or rope.get('type')!r}; only the default "
                             "RoPE is supported for Qwen2")
        if d.get("head_dim") is not None and d["head_dim"] != d["hidden_size"] // d["num_attention_heads"]:
            raise ValueError(f"{name}: head_dim {d['head_dim']} differs from hidden_size / num_attention_heads = "
                             f"{d['hidden_size'] // d['num_attention_heads']}; only head_dim = hidden / heads is supported")
    if mt == "qwen3":
        if d.get("use_sliding_window"):
            raise ValueError(f"{name}: use_sliding_window is true; Qwen3 sliding-window layers are not supported")
        if "sliding_attention" in (d.get("layer_types") or ()):
            raise ValueError(f"{name}: layer_types contains 'sliding_attention'; Qwen3 sliding-window layers are "
                             "not supported")
        if d.get("attention_bias"):
            raise ValueError(f"{name}: attention_bias is true; q/k/v/o projections with a bias are not supported")
        head_dim = d.get("head_dim") or d["hidden_size"] // d["num_attention_heads"]
    if mt == "llama" and d.get("head_dim") is not None and d["head_dim"] != d["hidden_size"] // d["num_attention_heads"]:
        # a head_dim of its own (as transformers' LlamaConfig allows); equal or absent derives it from the hidden size
        head_dim = d["head_dim"]
    if mt == "mistral":
        if d.get("head_dim") is not None and d["head_dim"] != d["hidden_size"] // d["num_attention_heads"]:
            raise ValueError(f"{name}: head_dim {d['head_dim']} differs from hidden_size / num_attention_heads = "
                             f"{d['hidden_size'] // d['num_attention_heads']}; only head_dim = hidden / heads is supported")
        window = d.get("sliding_window", 4096)   # MistralConfig's default; null means no window
    scaling = d.get("rope_scaling")
    theta = d.get("rope_theta", 1e4)
    if isinstance(d.get("rope_parameters"), dict):  # transformers>=5 layout
        rp = d["rope_parameters"]
        theta = rp.get("rope_theta", theta)
        if rp.get("rope_type", "default") != "default":
            scaling = rp
    return ModelConfig(
        vocab_size=d["vocab_size"], hidden_size=d["hidden_size"],
        intermediate_size=d["intermediate_size"], num_hidden_layers=d["num_hidden_layers"],
        num_attention_heads=d["num_attention_heads"],
        num_key_value_heads=d.get("num_key_value_heads", d["num_attention_heads"]),
        max_position_embeddings=d.get("max_position_embeddings", 4096),
        rms_norm_eps=d.get("rms_norm_eps", 1e-5), rope_theta=theta, rope_scaling=scaling,
        tie_word_embeddings=d.get("tie_word_embeddings", False), sliding_window=window, name=name,
        arch=mt, explicit_head_dim=head_dim, qk_norm=mt == "qwen3", qkv_bias=mt == "qwen2",
    )


def _starcoder2_from_hf_dict(d: dict, name: str) -> ModelConfig:
    """A ``Starcoder2Config`` payload.  Every setting the kernel path does not implement is refused, naming its key,
    rather than dropped."""
    if d.get("use_bias", True) is not True:
        raise ValueError(f"{name}: use_bias is {d['use_bias']!r}; only StarCoder2 with biases on every projection "
                         "is supported")
    if d.get("hidden_act", "gelu_pytorch_tanh") != "gelu_pytorch_tanh":
        raise ValueError(f"{name}: hidden_act is {d['hidden_act']!r}; only 'gelu_pytorch_tanh' is supported")
    if d.get("norm_type", "layer_norm") != "layer_norm":
        raise ValueError(f"{name}: norm_type is {d['norm_type']!r}; only 'layer_norm' is supported")
    if d.get("mlp_type", "default") != "default":
        raise ValueError(f"{name}: mlp_type is {d['mlp_type']!r}; only 'default' is supported")
    rope = d.get("rope_parameters") if isinstance(d.get("rope_parameters"), dict) else d.get("rope_scaling")
    if rope and (rope.get("rope_type") or rope.get("type") or "default") != "default":
        key = "rope_parameters" if isinstance(d.get("rope_parameters"), dict) else "rope_scaling"
        raise ValueError(f"{name}: {key} has type {rope.get('rope_type') or rope.get('type')!r}; only the default "
                         "RoPE is supported for StarCoder2")
    if d.get("head_dim") is not None and d["head_dim"] != d["hidden_size"] // d["num_attention_heads"]:
        raise ValueError(f"{name}: head_dim {d['head_dim']} differs from hidden_size / num_attention_heads = "
                         f"{d['hidden_size'] // d['num_attention_heads']}; only head_dim = hidden / heads is supported")
    for key in ("attention_dropout", "residual_dropout", "embedding_dropout"):
        if d.get(key, 0.0):
            raise ValueError(f"{name}: {key} is {d[key]!r}; the kernel path has no dropout, set {key} to 0.0 to "
                             "train without it")
    theta = d.get("rope_theta", 1e4)
    if isinstance(d.get("rope_parameters"), dict):  # transformers>=5 layout
        theta = d["rope_parameters"].get("rope_theta", theta)
    return ModelConfig(
        arch="starcoder2", vocab_size=d["vocab_size"], hidden_size=d["hidden_size"],
        intermediate_size=d["intermediate_size"], num_hidden_layers=d["num_hidden_layers"],
        num_attention_heads=d["num_attention_heads"],
        num_key_value_heads=d.get("num_key_value_heads", d["num_attention_heads"]),
        max_position_embeddings=d.get("max_position_embeddings", 4096), rope_theta=theta,
        tie_word_embeddings=d.get("tie_word_embeddings", True), sliding_window=d.get("sliding_window"),
        layer_norm_epsilon=d.get("norm_epsilon", 1e-5), name=name,
    )


def _olmoe_from_hf_dict(d: dict, name: str) -> ModelConfig:
    """An ``OlmoeConfig`` payload.  Every setting the kernel path does not implement is refused, naming its key,
    rather than dropped; ``router_aux_loss_coef`` and ``output_router_logits`` are training options
    (``--router-aux-loss-coef``), not part of the model."""
    if d.get("clip_qkv") is not None:
        raise ValueError(f"{name}: clip_qkv is {d['clip_qkv']!r}; only clip_qkv null (no clipping) is supported")
    if d.get("norm_topk_prob", False):
        raise ValueError(f"{name}: norm_topk_prob is true; only the raw top-k router probabilities are supported")
    if d.get("attention_bias"):
        raise ValueError(f"{name}: attention_bias is true; OLMoE projections with a bias are not supported")
    if d.get("hidden_act", "silu") != "silu":
        raise ValueError(f"{name}: hidden_act is {d['hidden_act']!r}; only 'silu' (SwiGLU experts) is supported")
    rp = d.get("rope_parameters") if isinstance(d.get("rope_parameters"), dict) else None
    rope = rp if rp is not None else d.get("rope_scaling")
    if rope and (rope.get("rope_type") or rope.get("type") or "default") != "default":
        key = "rope_parameters" if rp is not None else "rope_scaling"
        raise ValueError(f"{name}: {key} has type {rope.get('rope_type') or rope.get('type')!r}; only the default "
                         "RoPE is supported for OLMoE")
    for key in ("attention_dropout", "hidden_dropout", "dropout"):
        if d.get(key, 0.0):
            raise ValueError(f"{name}: {key} is {d[key]!r}; the kernel path has no dropout, set {key} to 0.0 to "
                             "train without it")
    if d.get("head_dim") is not None and d["head_dim"] != d["hidden_size"] // d["num_attention_heads"]:
        raise ValueError(f"{name}: head_dim {d['head_dim']} differs from hidden_size / num_attention_heads = "
                         f"{d['hidden_size'] // d['num_attention_heads']}; only head_dim = hidden / heads is supported")
    theta = (rp or {}).get("rope_theta", d.get("rope_theta", 1e4))
    return ModelConfig(
        arch="olmoe", vocab_size=d["vocab_size"], hidden_size=d["hidden_size"],
        intermediate_size=d["intermediate_size"], num_hidden_layers=d["num_hidden_layers"],
        num_attention_heads=d["num_attention_heads"],
        num_key_value_heads=d.get("num_key_value_heads", d["num_attention_heads"]),
        max_position_embeddings=d.get("max_position_embeddings", 4096), rms_norm_eps=d.get("rms_norm_eps", 1e-5),
        rope_theta=theta, tie_word_embeddings=d.get("tie_word_embeddings", False),
        num_experts=d.get("num_experts", 64), num_experts_per_tok=d.get("num_experts_per_tok", 8), name=name,
    )


def _qwen3_moe_from_hf_dict(d: dict, name: str) -> ModelConfig:
    """A ``Qwen3MoeConfig`` payload: every layer sparse, routing weights raw or renormalised (``norm_topk_prob``,
    false by default as in ``Qwen3MoeConfig``).  Every setting the kernel path does not implement is refused, naming
    its key, rather than dropped; ``router_aux_loss_coef`` and ``output_router_logits`` are training options
    (``--router-aux-loss-coef``), not part of the model."""
    if d.get("mlp_only_layers"):
        raise ValueError(f"{name}: mlp_only_layers is {d['mlp_only_layers']!r}; dense layers between the sparse ones "
                         "are not supported, only [] (every layer sparse)")
    if d.get("decoder_sparse_step", 1) != 1:
        raise ValueError(f"{name}: decoder_sparse_step is {d['decoder_sparse_step']!r}; dense layers between the "
                         "sparse ones are not supported, only 1 (every layer sparse)")
    if d.get("use_sliding_window"):
        raise ValueError(f"{name}: use_sliding_window is true; Qwen3-MoE sliding-window layers are not supported")
    if "sliding_attention" in (d.get("layer_types") or ()):
        raise ValueError(f"{name}: layer_types contains 'sliding_attention'; Qwen3-MoE sliding-window layers are not "
                         "supported")
    if d.get("attention_bias"):
        raise ValueError(f"{name}: attention_bias is true; q/k/v/o projections with a bias are not supported")
    if d.get("hidden_act", "silu") != "silu":
        raise ValueError(f"{name}: hidden_act is {d['hidden_act']!r}; only 'silu' (SwiGLU experts) is supported")
    rp = d.get("rope_parameters") if isinstance(d.get("rope_parameters"), dict) else None
    rope = rp if rp is not None else d.get("rope_scaling")
    if rope and (rope.get("rope_type") or rope.get("type") or "default") != "default":
        key = "rope_parameters" if rp is not None else "rope_scaling"
        raise ValueError(f"{name}: {key} has type {rope.get('rope_type') or rope.get('type')!r}; only the default "
                         "RoPE is supported for Qwen3-MoE")
    for key in ("attention_dropout", "hidden_dropout", "dropout"):
        if d.get(key, 0.0):
            raise ValueError(f"{name}: {key} is {d[key]!r}; the kernel path has no dropout, set {key} to 0.0 to "
                             "train without it")
    experts = d.get("num_experts", d.get("num_local_experts", 128))
    if experts > 256:
        raise ValueError(f"{name}: num_experts is {experts}; the routing kernels serve at most 256 experts")
    head_dim = d.get("head_dim") or d["hidden_size"] // d["num_attention_heads"]
    if head_dim != 128:
        raise ValueError(f"{name}: head_dim is {head_dim}; Qwen3-MoE's per-head QK-norm kernel serves head_dim 128")
    theta = (rp or {}).get("rope_theta", d.get("rope_theta", 1e6))
    return ModelConfig(
        arch="qwen3_moe", vocab_size=d["vocab_size"], hidden_size=d["hidden_size"],
        intermediate_size=d.get("moe_intermediate_size", 768), num_hidden_layers=d["num_hidden_layers"],
        num_attention_heads=d["num_attention_heads"],
        num_key_value_heads=d.get("num_key_value_heads", d["num_attention_heads"]),
        max_position_embeddings=d.get("max_position_embeddings", 32768), rms_norm_eps=d.get("rms_norm_eps", 1e-6),
        rope_theta=theta, tie_word_embeddings=d.get("tie_word_embeddings", False), explicit_head_dim=128,
        qk_norm=True, num_experts=experts, num_experts_per_tok=d.get("num_experts_per_tok", 8),
        norm_topk_prob=bool(d.get("norm_topk_prob", False)), name=name,
    )


def _gpt_neox_from_hf_dict(d: dict, name: str) -> ModelConfig:
    """A ``GPTNeoXConfig`` payload, with RoPE settings as ``rotary_pct`` / ``rotary_emb_base`` (the published files) or
    in transformers 5's ``rope_parameters``.  Every setting the kernel path does not implement is refused, naming its
    key, rather than dropped."""
    if d.get("use_parallel_residual", True) is not True:
        raise ValueError(f"{name}: use_parallel_residual is {d['use_parallel_residual']!r}; only GPT-NeoX's parallel "
                         "residual is supported")
    if d.get("hidden_act", "gelu") != "gelu":
        raise ValueError(f"{name}: hidden_act is {d['hidden_act']!r}; only 'gelu' (exact) is supported")
    if d.get("attention_bias", True) is not True:
        raise ValueError(f"{name}: attention_bias is {d['attention_bias']!r}; only GPT-NeoX with biases on every "
                         "projection is supported")
    for key in ("hidden_dropout", "attention_dropout"):
        if d.get(key, 0.0):
            raise ValueError(f"{name}: {key} is {d[key]!r}; the kernel path has no dropout, set {key} to 0.0 to "
                             "train without it")
    rp = d.get("rope_parameters") if isinstance(d.get("rope_parameters"), dict) else None
    rope = rp if rp is not None else d.get("rope_scaling")
    if rope and (rope.get("rope_type") or rope.get("type") or "default") != "default":
        key = "rope_parameters" if rp is not None else "rope_scaling"
        raise ValueError(f"{name}: {key} has type {rope.get('rope_type') or rope.get('type')!r}; only the default "
                         "RoPE is supported for GPT-NeoX")
    theta = d.get("rotary_emb_base", d.get("rope_theta", 1e4))
    pct = d.get("rotary_pct", d.get("partial_rotary_factor", 0.25))
    if rp is not None:   # transformers>=5 layout
        theta = rp.get("rope_theta", theta)
        pct = rp.get("partial_rotary_factor", pct)
    h, nh = d["hidden_size"], d["num_attention_heads"]
    head_dim = h // nh
    if head_dim not in (64, 128) or head_dim * nh != h:
        raise ValueError(f"{name}: head_dim (hidden_size / num_attention_heads = {h} / {nh}) is not 64 or 128; the "
                         "attention kernels serve head_dim 64 and 128")
    rot = int(head_dim * pct)
    key = "rope_parameters.partial_rotary_factor" if rp is not None and "partial_rotary_factor" in rp else "rotary_pct"
    if rot <= 0 or rot % 16:
        raise ValueError(f"{name}: {key} {pct!r} gives a rotary dim of {rot} of head_dim {head_dim}; the RoPE kernel "
                         "needs a positive multiple of 16")
    return ModelConfig(
        arch="gpt_neox", vocab_size=d["vocab_size"], hidden_size=h, intermediate_size=d["intermediate_size"],
        num_hidden_layers=d["num_hidden_layers"], num_attention_heads=nh, num_key_value_heads=nh,
        max_position_embeddings=d.get("max_position_embeddings", 2048), rope_theta=theta,
        tie_word_embeddings=d.get("tie_word_embeddings", False), layer_norm_epsilon=d.get("layer_norm_eps", 1e-5),
        partial_rotary_factor=pct, name=name,
    )


def get_config(name: str, **overrides) -> ModelConfig:
    """Resolve ``name`` (registry id, or a directory / file holding an HF ``config.json``)."""
    if name in REGISTRY:
        cfg = REGISTRY[name]
    else:
        path = name
        if os.path.isdir(path):
            path = os.path.join(path, "config.json")
        if not os.path.isfile(path):
            raise KeyError(
                f"unknown model {name!r}: not in the embedded registry ({sorted(REGISTRY)}) "
                "and not a local directory with a config.json (there is no network on the GPU box)"
            )
        with open(path) as fp:
            cfg = _from_hf_dict(json.load(fp), name)
    if overrides:
        cfg = dataclasses.replace(cfg, **overrides)
    return cfg


def to_hf_config_dict(cfg: ModelConfig) -> dict:
    """An HF-style ``config.json`` payload (used to feed the *reference* scripts offline)."""
    if cfg.arch == "gpt2":
        return {
            "model_type": "gpt2", "architectures": ["GPT2LMHeadModel"], "vocab_size": cfg.vocab_size,
            "n_embd": cfg.hidden_size, "n_inner": cfg.intermediate_size, "n_layer": cfg.num_hidden_layers,
            "n_head": cfg.num_attention_heads, "n_positions": cfg.max_position_embeddings,
            "layer_norm_epsilon": cfg.layer_norm_epsilon, "resid_pdrop": cfg.dropout,
            "embd_pdrop": cfg.dropout, "attn_pdrop": cfg.dropout, "activation_function": "gelu_new",
        }
    d = {
        "model_type": "llama", "architectures": ["LlamaForCausalLM"], "vocab_size": cfg.vocab_size,
        "hidden_size": cfg.hidden_size, "intermediate_size": cfg.intermediate_size,
        "num_hidden_layers": cfg.num_hidden_layers, "num_attention_heads": cfg.num_attention_heads,
        "num_key_value_heads": cfg.num_key_value_heads, "max_position_embeddings": cfg.max_position_embeddings,
        "rms_norm_eps": cfg.rms_norm_eps, "rope_theta": cfg.rope_theta, "hidden_act": "silu",
        "tie_word_embeddings": cfg.tie_word_embeddings, "attention_bias": False, "mlp_bias": False,
        "bos_token_id": 1, "eos_token_id": 2, "torch_dtype": "bfloat16",
    }
    if cfg.arch == "mistral":
        return {
            "model_type": "mistral", "architectures": ["MistralForCausalLM"], "vocab_size": cfg.vocab_size,
            "hidden_size": cfg.hidden_size, "intermediate_size": cfg.intermediate_size,
            "num_hidden_layers": cfg.num_hidden_layers, "num_attention_heads": cfg.num_attention_heads,
            "num_key_value_heads": cfg.num_key_value_heads, "head_dim": cfg.head_dim,
            "max_position_embeddings": cfg.max_position_embeddings, "rms_norm_eps": cfg.rms_norm_eps,
            "rope_theta": cfg.rope_theta, "sliding_window": cfg.sliding_window, "hidden_act": "silu",
            "tie_word_embeddings": cfg.tie_word_embeddings, "bos_token_id": 1, "eos_token_id": 2,
            "torch_dtype": "bfloat16",
        }
    if cfg.arch == "qwen3":
        d = {
            "model_type": "qwen3", "architectures": ["Qwen3ForCausalLM"], "vocab_size": cfg.vocab_size,
            "hidden_size": cfg.hidden_size, "intermediate_size": cfg.intermediate_size,
            "num_hidden_layers": cfg.num_hidden_layers, "num_attention_heads": cfg.num_attention_heads,
            "num_key_value_heads": cfg.num_key_value_heads, "head_dim": cfg.head_dim,
            "max_position_embeddings": cfg.max_position_embeddings, "rms_norm_eps": cfg.rms_norm_eps,
            "rope_theta": cfg.rope_theta, "hidden_act": "silu", "tie_word_embeddings": cfg.tie_word_embeddings,
            "attention_bias": False, "use_sliding_window": False, "bos_token_id": 151643, "eos_token_id": 151645,
            "torch_dtype": "bfloat16",
        }
    if cfg.arch == "qwen2":
        d = {
            "model_type": "qwen2", "architectures": ["Qwen2ForCausalLM"], "vocab_size": cfg.vocab_size,
            "hidden_size": cfg.hidden_size, "intermediate_size": cfg.intermediate_size,
            "num_hidden_layers": cfg.num_hidden_layers, "num_attention_heads": cfg.num_attention_heads,
            "num_key_value_heads": cfg.num_key_value_heads, "max_position_embeddings": cfg.max_position_embeddings,
            "rms_norm_eps": cfg.rms_norm_eps, "rope_theta": cfg.rope_theta, "hidden_act": "silu",
            "tie_word_embeddings": cfg.tie_word_embeddings, "use_sliding_window": False, "bos_token_id": 151643,
            "eos_token_id": 151643, "torch_dtype": "bfloat16",
        }
    if cfg.arch == "olmo2":
        d = {
            "model_type": "olmo2", "architectures": ["Olmo2ForCausalLM"], "vocab_size": cfg.vocab_size,
            "hidden_size": cfg.hidden_size, "intermediate_size": cfg.intermediate_size,
            "num_hidden_layers": cfg.num_hidden_layers, "num_attention_heads": cfg.num_attention_heads,
            "num_key_value_heads": cfg.num_key_value_heads, "max_position_embeddings": cfg.max_position_embeddings,
            "rms_norm_eps": cfg.rms_norm_eps, "rope_theta": cfg.rope_theta, "hidden_act": "silu",
            "tie_word_embeddings": cfg.tie_word_embeddings, "attention_bias": False, "pad_token_id": None,
            "bos_token_id": None, "eos_token_id": 100257, "torch_dtype": "bfloat16",
        }
    if cfg.arch == "starcoder2":
        d = {
            "model_type": "starcoder2", "architectures": ["Starcoder2ForCausalLM"], "vocab_size": cfg.vocab_size,
            "hidden_size": cfg.hidden_size, "intermediate_size": cfg.intermediate_size,
            "num_hidden_layers": cfg.num_hidden_layers, "num_attention_heads": cfg.num_attention_heads,
            "num_key_value_heads": cfg.num_key_value_heads, "max_position_embeddings": cfg.max_position_embeddings,
            "norm_epsilon": cfg.layer_norm_epsilon, "rope_theta": cfg.rope_theta, "sliding_window": cfg.sliding_window,
            "hidden_act": "gelu_pytorch_tanh", "use_bias": True, "tie_word_embeddings": cfg.tie_word_embeddings,
            "attention_dropout": 0.0, "residual_dropout": 0.0, "embedding_dropout": 0.0, "bos_token_id": 0,
            "eos_token_id": 0, "torch_dtype": "bfloat16",
        }
    if cfg.arch == "gpt_neox":
        d = {
            "model_type": "gpt_neox", "architectures": ["GPTNeoXForCausalLM"], "vocab_size": cfg.vocab_size,
            "hidden_size": cfg.hidden_size, "intermediate_size": cfg.intermediate_size,
            "num_hidden_layers": cfg.num_hidden_layers, "num_attention_heads": cfg.num_attention_heads,
            "max_position_embeddings": cfg.max_position_embeddings, "layer_norm_eps": cfg.layer_norm_epsilon,
            "rotary_pct": cfg.partial_rotary_factor, "rotary_emb_base": cfg.rope_theta, "hidden_act": "gelu",
            "use_parallel_residual": True, "attention_bias": True, "hidden_dropout": 0.0, "attention_dropout": 0.0,
            "tie_word_embeddings": cfg.tie_word_embeddings, "bos_token_id": 0, "eos_token_id": 0,
            "torch_dtype": "float16",
        }
    if cfg.arch == "olmoe":
        d = {
            "model_type": "olmoe", "architectures": ["OlmoeForCausalLM"], "vocab_size": cfg.vocab_size,
            "hidden_size": cfg.hidden_size, "intermediate_size": cfg.intermediate_size,
            "num_hidden_layers": cfg.num_hidden_layers, "num_attention_heads": cfg.num_attention_heads,
            "num_key_value_heads": cfg.num_key_value_heads, "max_position_embeddings": cfg.max_position_embeddings,
            "rms_norm_eps": cfg.rms_norm_eps, "rope_theta": cfg.rope_theta, "hidden_act": "silu",
            "tie_word_embeddings": cfg.tie_word_embeddings, "attention_bias": False, "attention_dropout": 0.0,
            "clip_qkv": None, "num_experts": cfg.num_experts, "num_experts_per_tok": cfg.num_experts_per_tok,
            "norm_topk_prob": False, "output_router_logits": False, "router_aux_loss_coef": 0.01,
            "pad_token_id": 1, "bos_token_id": None, "eos_token_id": 50279, "torch_dtype": "bfloat16",
        }
    if cfg.arch == "qwen3_moe":
        d = {
            "model_type": "qwen3_moe", "architectures": ["Qwen3MoeForCausalLM"], "vocab_size": cfg.vocab_size,
            "hidden_size": cfg.hidden_size, "moe_intermediate_size": cfg.intermediate_size,
            "num_hidden_layers": cfg.num_hidden_layers, "num_attention_heads": cfg.num_attention_heads,
            "num_key_value_heads": cfg.num_key_value_heads, "head_dim": cfg.head_dim,
            "max_position_embeddings": cfg.max_position_embeddings, "rms_norm_eps": cfg.rms_norm_eps,
            "rope_theta": cfg.rope_theta, "hidden_act": "silu", "tie_word_embeddings": cfg.tie_word_embeddings,
            "attention_bias": False, "attention_dropout": 0.0, "use_sliding_window": False, "decoder_sparse_step": 1,
            "mlp_only_layers": [], "num_experts": cfg.num_experts, "num_experts_per_tok": cfg.num_experts_per_tok,
            "norm_topk_prob": cfg.norm_topk_prob, "output_router_logits": False, "router_aux_loss_coef": 0.001,
            "bos_token_id": 151643, "eos_token_id": 151645, "torch_dtype": "bfloat16",
        }
    if cfg.arch == "llama" and cfg.explicit_head_dim is not None:
        d["head_dim"] = cfg.explicit_head_dim
    if cfg.rope_scaling:
        d["rope_scaling"] = cfg.rope_scaling
    return d
