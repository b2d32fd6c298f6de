"""Pretrained-weight loading for sharded engines (reference: rank-0 ``from_pretrained`` on CPU +
``set_model_state_dict(broadcast_from_rank0=True)`` + manual buffer broadcasts,
``05-training-llama-405b/train_llm.py:76-145``).

Because every group is a flat buffer, distribution is per group instead of per tensor: rank 0 copies the HF
tensors of one group into a staging flat tensor (names are identical to ours), broadcasts it, and every rank
keeps the slice it owns.  Peak host memory on rank 0 is one checkpoint file + one group; nothing like the
reference's 764 GB resident model is needed.  There are no non-persistent buffers to broadcast (RoPE tables
are recomputed from the config).
"""
from __future__ import annotations

import glob
import json
import logging
import os
from typing import Callable, Dict, Optional

import torch
import torch.distributed as dist

LOGGER = logging.getLogger("dtg_b200")


# -- locating and reading Hugging Face safetensors checkpoints ------------------------------------------------------
def find_checkpoint(model_name: str) -> Optional[str]:
    """Directory holding ``*.safetensors`` for ``model_name``: the name itself when it is a local directory,
    else an already-downloaded snapshot in the Hugging Face cache (``download.py`` puts it there).  ``None``
    when there are no local weights — nothing is ever downloaded from here."""
    if os.path.isdir(model_name):
        return model_name if glob.glob(os.path.join(model_name, "*.safetensors")) else None
    try:
        from huggingface_hub import snapshot_download

        path = snapshot_download(model_name, local_files_only=True, allow_patterns=["*.safetensors", "*.json"])
        return path if glob.glob(os.path.join(path, "*.safetensors")) else None
    except Exception:
        return None


class SafetensorsReader:
    """``reader(name) -> tensor`` over a (possibly multi-file) safetensors checkpoint; files are opened lazily
    and only the requested tensor is read, so host memory stays at one tensor, not one model."""

    def __init__(self, directory: str):
        from safetensors import safe_open

        self._open = safe_open
        self.directory = directory
        self._handles = {}
        index = os.path.join(directory, "model.safetensors.index.json")
        if os.path.isfile(index):
            with open(index) as fp:
                self.weight_map = dict(json.load(fp)["weight_map"])
        else:
            self.weight_map = {}
            for f in sorted(glob.glob(os.path.join(directory, "*.safetensors"))):
                with safe_open(f, framework="pt", device="cpu") as h:
                    for k in h.keys():
                        self.weight_map[k] = os.path.basename(f)

    def __contains__(self, name):
        return name in self.weight_map

    def __call__(self, name: str) -> torch.Tensor:
        if name not in self.weight_map and name == "lm_head.weight":  # tied embeddings are stored once
            name = "model.embed_tokens.weight"
        fname = self.weight_map[name]
        if fname not in self._handles:
            self._handles[fname] = self._open(os.path.join(self.directory, fname), framework="pt", device="cpu")
        return self._handles[fname].get_tensor(name)


def maybe_load_pretrained(args, model=None, engine=None, default="never") -> bool:
    """``--pretrained auto|require|never``: load local Hugging Face weights into a sharded (``engine``) or a
    replicated (``model``) build.  Returns True when weights were loaded."""
    mode = getattr(args, "pretrained", None) or default
    if mode == "never":
        return False
    rank = dist.get_rank() if dist.is_initialized() else 0
    path = find_checkpoint(args.model_name)
    if path is None:
        if mode == "require":
            raise FileNotFoundError(f"--pretrained require: no local safetensors for {args.model_name!r} "
                                    "(a directory with *.safetensors, or a snapshot in $HF_HOME)")
        if rank == 0:
            LOGGER.info(f"No local weights for {args.model_name}: training from random initialisation")
        return False
    if rank == 0:
        LOGGER.info(f"Loading pretrained weights from {path}")
    if engine is not None:
        load_into_fsdp(engine, open_checkpoint(path) if rank == 0 else None)
    else:
        reader = open_checkpoint(path)
        load_state_dict_into_flat(model, {k: reader(k) for k in model.state_dict().keys() if k in reader or
                                          k == "lm_head.weight"})
    return True


def open_checkpoint(path: str):
    """``reader(name) -> tensor`` under this project's parameter names: a ``SafetensorsReader``, seen through
    ``models.gpt_neox_layout`` when the checkpoint is GPT-NeoX's (other names and layout), or through
    ``models.olmoe_layout`` when it stores OLMoE's experts one tensor each."""
    from ..models import get_config, gpt_neox_layout, olmoe_layout

    reader = SafetensorsReader(path)
    if gpt_neox_layout.is_gpt_neox_checkpoint(reader.weight_map):
        return gpt_neox_layout.HFReader(reader, reader.weight_map, get_config(path).num_attention_heads)
    if olmoe_layout.is_per_expert_checkpoint(reader.weight_map):
        return olmoe_layout.HFReader(reader, reader.weight_map, get_config(path).num_experts)
    return reader


def load_into_fsdp(engine, get_tensor: Optional[Callable[[str], torch.Tensor]], src_rank: int = 0):
    """``get_tensor(name)`` is only called on ``src_rank`` (e.g. a safetensors ``get_tensor``)."""
    rank = dist.get_rank() if dist.is_initialized() else 0
    for g, sh in zip(engine.groups, engine.shards):
        staging = torch.zeros(g.padded_numel, dtype=g.param.dtype, device=g.param.device)
        if rank == src_rank:
            for name, off, shape in zip(g.names, g.offsets, g.shapes):
                t = get_tensor(name)
                staging[off:off + t.numel()].copy_(t.reshape(-1).to(staging.dtype))
        if dist.is_initialized() and dist.get_world_size() > 1:
            dist.broadcast(staging, src=src_rank)
        per = sh.padded_numel
        sh.param.copy_(staging[engine.rank * per:(engine.rank + 1) * per])
        del staging


def load_state_dict_into_flat(model, state_dict: Dict[str, torch.Tensor]):
    """Replicated engines (chapters 01/02): in-place copy into the flat views."""
    own = model.state_dict()
    with torch.no_grad():
        for k, v in state_dict.items():
            own[k].copy_(v)
