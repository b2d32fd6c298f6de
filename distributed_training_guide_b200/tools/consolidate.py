"""Turn a sharded (DCP) checkpoint of chapters 04-07 into one HF-named ``model.pt``.

    python -m distributed_training_guide_b200.tools.consolidate <exp_dir> -m meta-llama/Llama-2-7b-hf [--world N]

The sharded checkpoint stores, per flat group (``embed``, ``layer{i}``, ``head``), the concatenation of the
ranks' 1-D shards; this tool loads them in a single process, cuts the groups back into named parameters
(group layouts are derived from the model config) and writes ``<exp_dir>/model.pt``.  (The reference points to
``torch.distributed.checkpoint.format_utils.dcp_to_torch_save`` for the same job.)
"""
from __future__ import annotations

import argparse
from pathlib import Path

import torch

from ..models import build_model, get_config, gpt_neox_layout, olmoe_layout
from ..parallel.flat import build_groups


def consolidate(exp_dir: str, model_name: str, world: int) -> Path:
    import torch.distributed.checkpoint as dcp

    import json

    cfg = get_config(model_name)
    model = build_model(cfg, dtype=torch.bfloat16, device="cpu", init=False)
    out = Path(exp_dir) / "model.pt"
    layout_file = Path(exp_dir) / "layout.json"
    if layout_file.exists():
        # the writer recorded where every parameter sits in its group (padding and order depend on the engine's
        # chunk alignment): cut by that, not by a re-derived layout
        layout = json.loads(layout_file.read_text())
        state = {"model": {n: torch.zeros(d["padded_numel"], dtype=torch.bfloat16) for n, d in layout.items()}}
        dcp.load(state, checkpoint_id=str(Path(exp_dir) / "checkpoint"))
        sd = model.state_dict()
        with torch.no_grad():
            for gname, d in layout.items():
                flat = state["model"][gname]
                for name, off, shape in zip(d["names"], d["offsets"], d["shapes"]):
                    n = 1
                    for x in shape:
                        n *= x
                    sd[name].copy_(flat[off:off + n].view(shape))
            if getattr(cfg, "tie_word_embeddings", False) and "lm_head.weight" in sd:
                sd["lm_head.weight"].copy_(sd["model.embed_tokens.weight"] if "model.embed_tokens.weight" in sd
                                           else sd["lm_head.weight"])
        torch.save(_hf_layout(sd, cfg), out)
        return out
    groups = build_groups(model, "cpu", torch.bfloat16, world_size=world, with_grad=False)
    state = {"model": {g.name: torch.zeros(g.padded_numel, dtype=torch.bfloat16) for g in groups}}
    dcp.load(state, checkpoint_id=str(Path(exp_dir) / "checkpoint"))
    for g in groups:
        g.param.copy_(state["model"][g.name])
    torch.save(_hf_layout(model.state_dict(), cfg), out)
    return out


def _hf_layout(sd, cfg):
    """GPT-NeoX is written under its own HF names and q|k|v layout (``GPTNeoXForCausalLM`` loads it strictly), OLMoE
    with one tensor per expert as its published checkpoints are; every other family already has HF's names."""
    if cfg.arch == "gpt_neox":
        return gpt_neox_layout.to_hf_state_dict(sd, cfg.num_attention_heads)
    if cfg.moe:
        return olmoe_layout.to_hf_state_dict(sd)
    return sd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("exp_dir")
    ap.add_argument("-m", "--model-name", required=True)
    ap.add_argument("--world", type=int, required=True, help="number of ranks that wrote the checkpoint")
    a = ap.parse_args()
    print(f"wrote {consolidate(a.exp_dir, a.model_name, a.world)}")


if __name__ == "__main__":
    main()
