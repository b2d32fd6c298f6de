"""The published mixture-of-experts checkpoint layout of OLMoE and Qwen3-MoE, and ours.

Published OLMoE and Qwen3-MoE checkpoints (the same expert parameter names) store one tensor per expert: ``model.layers.{i}.mlp.experts.{j}.{gate,up,down}_proj.weight``
([I, H], [I, H], [H, I]).  The model here (and transformers 5 in memory) holds each layer's experts as two 3-D
parameters, ``mlp.experts.gate_up_proj`` [E, 2I, H] (expert j's gate rows, then its up rows) and ``mlp.experts.down_proj``
[E, H, I].  Every other name is shared.  This module is the one place that knows the mapping: ``HFReader`` serves our
names from a per-expert checkpoint (``--pretrained``), ``to_hf_state_dict`` writes the per-expert layout
(``tools/consolidate.py``)."""
from __future__ import annotations

import re
from typing import Callable, Dict

import torch

_EXPERT_RE = re.compile(r"(model\.layers\.\d+\.mlp\.experts)\.(\d+)\.(gate|up|down)_proj\.weight$")
_FUSED_RE = re.compile(r"(model\.layers\.\d+\.mlp\.experts)\.(gate_up_proj|down_proj)$")


def is_per_expert_checkpoint(names) -> bool:
    return any(_EXPERT_RE.match(n) for n in names)


def _expert_name(prefix: str, j: int, proj: str) -> str:
    return f"{prefix}.{j}.{proj}_proj.weight"


class HFReader:
    """``reader(name) -> tensor`` under our parameter names over ``get`` (a per-expert checkpoint's reader)."""

    def __init__(self, get: Callable[[str], torch.Tensor], names, num_experts: int):
        self._get, self._names, self.num_experts = get, set(names), num_experts

    def __contains__(self, name) -> bool:
        m = _FUSED_RE.match(name)
        if m:
            return _expert_name(m.group(1), 0, "down") in self._names
        return name in self._names or name in self._get

    def __call__(self, name: str) -> torch.Tensor:
        m = _FUSED_RE.match(name)
        if m is None:
            return self._get(name)
        prefix, E = m.group(1), self.num_experts
        if m.group(2) == "down_proj":
            return torch.stack([self._get(_expert_name(prefix, j, "down")) for j in range(E)])
        return torch.stack([torch.cat([self._get(_expert_name(prefix, j, "gate")), self._get(_expert_name(prefix, j, "up"))])
                            for j in range(E)])


def from_hf_state_dict(hf_sd: Dict[str, torch.Tensor], our_names, num_experts: int) -> Dict[str, torch.Tensor]:
    reader = HFReader(hf_sd.__getitem__, hf_sd.keys(), num_experts)
    return {n: reader(n) for n in our_names}


def to_hf_state_dict(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Our state dict -> the published per-expert layout."""
    out = {}
    for name, t in sd.items():
        m = _FUSED_RE.match(name)
        if m is None:
            out[name] = t
            continue
        prefix = m.group(1)
        for j in range(t.shape[0]):
            if m.group(2) == "down_proj":
                out[_expert_name(prefix, j, "down")] = t[j].contiguous()
            else:
                g, u = t[j].chunk(2, dim=0)
                out[_expert_name(prefix, j, "gate")] = g.contiguous()
                out[_expert_name(prefix, j, "up")] = u.contiguous()
    return out
