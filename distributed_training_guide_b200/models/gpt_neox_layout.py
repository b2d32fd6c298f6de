"""GPT-NeoX's checkpoint layout, in one place.

The model trains GPT-NeoX with StarCoder2's parameter names (``models/llama.py``: ``self_attn.{q,k,v,o}_proj``,
``mlp.c_fc`` / ``c_proj``), so the flat buffers, the fused q|k|v views and FSDP's layout are the Llama family's.
Hugging Face's ``GPTNeoXForCausalLM`` names them differently and stores q, k and v as one ``query_key_value``
[3 * nh * d, H] matrix (and bias) whose rows are interleaved per head: head i's rows are ``[q_i | k_i | v_i]``, each d
rows.  This module maps between the two; ``tools/load_hf.py`` reads GPT-NeoX checkpoints through it and
``tools/consolidate.py`` writes them with it.
"""
from __future__ import annotations

import re
from typing import Callable, Dict

import torch

#: our name (after ``model.layers.{i}.``) -> HF's (after ``gpt_neox.layers.{i}.``), for the tensors kept whole
_LAYER_NAMES = {
    "input_layernorm": "input_layernorm",
    "post_attention_layernorm": "post_attention_layernorm",
    "self_attn.o_proj": "attention.dense",
    "mlp.c_fc": "mlp.dense_h_to_4h",
    "mlp.c_proj": "mlp.dense_4h_to_h",
}
_TOP_NAMES = {
    "model.embed_tokens.weight": "gpt_neox.embed_in.weight",
    "model.norm.weight": "gpt_neox.final_layer_norm.weight",
    "model.norm.bias": "gpt_neox.final_layer_norm.bias",
    "lm_head.weight": "embed_out.weight",
}
_QKV = {"q_proj": 0, "k_proj": 1, "v_proj": 2}
_LAYER_RE = re.compile(r"model\.layers\.(\d+)\.(.+)\.(weight|bias)$")


def is_gpt_neox_checkpoint(names) -> bool:
    """Whether a checkpoint's tensor names are GPT-NeoX's."""
    return "gpt_neox.embed_in.weight" in names


def _split(name: str):
    """(HF name, slot of q|k|v or None) of one of our parameter names."""
    if name in _TOP_NAMES:
        return _TOP_NAMES[name], None
    m = _LAYER_RE.match(name)
    if m is None:
        raise KeyError(f"{name!r} has no GPT-NeoX counterpart")
    i, mod, kind = m.groups()
    if mod.startswith("self_attn.") and mod.split(".", 1)[1] in _QKV:
        return f"gpt_neox.layers.{i}.attention.query_key_value.{kind}", _QKV[mod.split(".", 1)[1]]
    if mod not in _LAYER_NAMES:
        raise KeyError(f"{name!r} has no GPT-NeoX counterpart")
    return f"gpt_neox.layers.{i}.{_LAYER_NAMES[mod]}.{kind}", None


def hf_name(name: str) -> str:
    """The HF tensor that holds our parameter ``name`` (whole, or as a per-head slice of query_key_value)."""
    return _split(name)[0]


class HFReader:
    """Our parameter names over a GPT-NeoX checkpoint: ``reader(name)`` reads HF's tensor through ``get`` and, for
    q / k / v, cuts that projection's rows out of every head of ``query_key_value``.  ``lm_head.weight`` falls back to
    the embedding when the checkpoint is tied and stores it once."""

    def __init__(self, get: Callable[[str], torch.Tensor], names, num_heads: int):
        self._get, self._names, self.num_heads = get, set(names), num_heads

    def _hf(self, name):
        hf, slot = _split(name)
        if name == "lm_head.weight" and hf not in self._names:
            hf = _TOP_NAMES["model.embed_tokens.weight"]
        return hf, slot

    def __contains__(self, name) -> bool:
        try:
            return self._hf(name)[0] in self._names
        except KeyError:
            return False

    def __call__(self, name: str) -> torch.Tensor:
        hf, slot = self._hf(name)
        t = self._get(hf)
        if slot is None:
            return t
        nh = self.num_heads
        d = t.shape[0] // (3 * nh)
        return t.reshape(nh, 3, d, *t.shape[1:])[:, slot].reshape(nh * d, *t.shape[1:])


def from_hf_state_dict(hf_sd: Dict[str, torch.Tensor], our_names, num_heads: int) -> Dict[str, torch.Tensor]:
    """Our state dict (for ``our_names``) from a GPT-NeoX one."""
    reader = HFReader(hf_sd.__getitem__, hf_sd.keys(), num_heads)
    return {n: reader(n) for n in our_names}


def to_hf_state_dict(sd: Dict[str, torch.Tensor], num_heads: int) -> Dict[str, torch.Tensor]:
    """A ``GPTNeoXForCausalLM`` state dict from ours: HF names, q|k|v interleaved per head into ``query_key_value``,
    and ``embed_out.weight`` written even when tied (it is the embedding then), so ``load_state_dict(strict=True)``
    takes it."""
    out, qkv = {}, {}
    for name, t in sd.items():
        hf, slot = _split(name)
        if slot is None:
            out[hf] = t
        else:
            qkv.setdefault(hf, [None, None, None])[slot] = t
    for hf, (q, k, v) in qkv.items():
        nh = num_heads
        d = q.shape[0] // nh
        parts = [p.reshape(nh, d, *p.shape[1:]) for p in (q, k, v)]
        out[hf] = torch.stack(parts, dim=1).reshape(3 * nh * d, *q.shape[1:])
    if "embed_out.weight" not in out:
        out["embed_out.weight"] = out["gpt_neox.embed_in.weight"]
    return out
