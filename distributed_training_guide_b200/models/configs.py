"""Embedded model configurations.

The GPU boxes have no network, so the handful of Hugging Face model ids the
guide uses (reference: every chapter's ``-m/--model-name`` flag, e.g.
``02-distributed-data-parallel/train_llm.py:57``) are resolved from this table
instead of the hub.  A local directory containing a ``config.json`` is also
accepted, and tiny ``debug-*`` configs exist for tests.
"""
from __future__ import annotations

import dataclasses
import json
import os
from typing import Optional


@dataclasses.dataclass
class ModelConfig:
    arch: str  # "llama" | "mistral" | "qwen3" | "qwen2" | "gpt2"; mistral is llama with a sliding attention window,
    # qwen3 llama with QK-norm and a head_dim of its own, qwen2 llama with q/k/v biases
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
    # gpt2 only
    layer_norm_epsilon: float = 1e-5
    dropout: float = 0.0
    name: str = ""

    @property
    def head_dim(self) -> int:
        if self.explicit_head_dim is not None:
            return self.explicit_head_dim
        return self.hidden_size // self.num_attention_heads

    def num_parameters(self) -> int:
        h, i, v, l = self.hidden_size, self.intermediate_size, self.vocab_size, self.num_hidden_layers
        if self.arch == "gpt2":
            per_layer = (3 * h * h + 3 * h) + (h * h + h) + (h * i + i) + (i * h + h) + 4 * h
            return v * h + self.max_position_embeddings * h + l * per_layer + 2 * h
        q = self.num_attention_heads * self.head_dim
        kv = self.num_key_value_heads * self.head_dim
        per_layer = h * q + 2 * kv * h + q * h + 3 * h * i + 2 * h
        if self.qk_norm:
            per_layer += 2 * self.head_dim
        if self.qkv_bias:
            per_layer += q + 2 * kv
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
    if mt not in ("llama", "mistral", "qwen3", "qwen2"):
        raise ValueError(f"unsupported model_type {mt!r} in {name}")
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
    if cfg.arch == "llama" and cfg.explicit_head_dim is not None:
        d["head_dim"] = cfg.explicit_head_dim
    if cfg.rope_scaling:
        d["rope_scaling"] = cfg.rope_scaling
    return d
