"""Llama 3.2 and head_dim 64 on the CPU: ``debug-llama-d64`` against ``transformers.LlamaForCausalLM`` with the same
weights (logits, loss and every gradient), untied and tied; the registry's Llama 3.2 configs and their parameter
counts against the meta-device model; and the HF config reader honouring a Llama ``head_dim`` of its own."""
import json

import pytest
import torch

from distributed_training_guide_b200.models import build_model, get_config, to_hf_config_dict

LLAMA32 = {   # id: (hidden, intermediate, layers, heads, kv heads, head_dim, parameters)
    "meta-llama/Llama-3.2-1B": (2048, 8192, 16, 32, 8, 64, 1_235_814_400),
    "meta-llama/Llama-3.2-3B": (3072, 8192, 28, 24, 8, 128, 3_212_749_824),
}


def _hf_llama(cfg, transformers):
    d = {k: v for k, v in to_hf_config_dict(cfg).items() if k not in ("model_type", "architectures", "torch_dtype")}
    hf_cfg = transformers.LlamaConfig(**d)
    hf_cfg._attn_implementation = "eager"
    return transformers.LlamaForCausalLM(hf_cfg).float().eval()


@pytest.mark.parametrize("tied", [False, True])
def test_debug_llama_d64_matches_transformers_fp32(tied):
    transformers = pytest.importorskip("transformers")
    cfg = get_config("debug-llama-d64", tie_word_embeddings=tied)
    assert cfg.arch == "llama" and cfg.head_dim == 64 and cfg.explicit_head_dim is None
    torch.manual_seed(0)
    mine = build_model(cfg, dtype=torch.float32, device="cpu")
    with torch.no_grad():   # larger q / k weights, so that attention is far from uniform
        for layer in mine.model.layers:
            layer.self_attn.q_proj.weight.mul_(4.0)
            layer.self_attn.k_proj.weight.mul_(4.0)
    hf = _hf_llama(cfg, transformers)
    assert hf.config.head_dim == 64
    missing, unexpected = hf.load_state_dict(mine.state_dict(), strict=False)
    assert not unexpected, unexpected
    assert all("rotary" in m or "inv_freq" in m or (tied and m == "lm_head.weight") for m in missing), missing
    if tied:
        assert hf.lm_head.weight is hf.model.embed_tokens.weight
    ids = torch.randint(0, cfg.vocab_size, (2, 96), generator=torch.Generator().manual_seed(1))
    out_mine = mine(input_ids=ids, labels=ids, return_logits=True)
    out_hf = hf(input_ids=ids, labels=ids)
    assert torch.allclose(out_mine.logits, out_hf.logits, atol=2e-4, rtol=1e-3), \
        (out_mine.logits - out_hf.logits).abs().max()
    assert abs(out_mine.loss.item() - out_hf.loss.item()) < 1e-4
    out_mine.loss.backward()
    out_hf.loss.backward()
    hf_params = dict(hf.named_parameters())
    for n, p in mine.named_parameters():
        want = hf_params[n].grad
        err = ((p.grad - want).norm() / want.norm()).item()
        assert err < 1e-4, (n, err)


@pytest.mark.parametrize("name", list(LLAMA32))
def test_registry_llama32(name):
    h, i, l, nh, nkv, d, n = LLAMA32[name]
    cfg = get_config(name)
    assert cfg.arch == "llama" and not cfg.qk_norm and cfg.head_dim == d and cfg.tie_word_embeddings
    assert (cfg.vocab_size, cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers) == (128256, h, i, l)
    assert (cfg.num_attention_heads, cfg.num_key_value_heads) == (nh, nkv)
    assert (cfg.rope_theta, cfg.max_position_embeddings) == (5e5, 131072)
    assert cfg.rope_scaling == {"rope_type": "llama3", "factor": 32.0, "low_freq_factor": 1.0,
                                "high_freq_factor": 4.0, "original_max_position_embeddings": 8192}
    assert cfg.num_parameters() == n
    assert build_model(cfg, dtype=torch.bfloat16, device="meta").num_parameters() == n


@pytest.mark.parametrize("name", list(LLAMA32))
def test_llama32_counts_match_transformers(name):
    transformers = pytest.importorskip("transformers")
    cfg = get_config(name)
    d = {k: v for k, v in to_hf_config_dict(cfg).items() if k not in ("model_type", "architectures", "torch_dtype")}
    with torch.device("meta"):
        hf = transformers.LlamaForCausalLM(transformers.LlamaConfig(**d))
    assert hf.config.head_dim == LLAMA32[name][5]
    assert sum(p.numel() for p in hf.parameters()) == cfg.num_parameters(), name


def _write_config(tmp_path, d):
    (tmp_path / "config.json").write_text(json.dumps(d))
    return str(tmp_path)


def test_hf_llama_head_dim_apart_from_hidden_size(tmp_path):
    """A Llama config.json whose head_dim differs from hidden / heads builds q/k/v/o with that head_dim."""
    base = to_hf_config_dict(get_config("debug-llama-d64"))
    assert "head_dim" not in base
    cfg = get_config(_write_config(tmp_path, {**base, "head_dim": 128}))
    assert cfg.arch == "llama" and cfg.head_dim == 128 and cfg.explicit_head_dim == 128 and not cfg.qk_norm
    model = build_model(cfg, dtype=torch.float32, device="meta")
    att = model.model.layers[0].self_attn
    assert tuple(att.q_proj.weight.shape) == (4 * 128, 256)
    assert tuple(att.k_proj.weight.shape) == (2 * 128, 256)
    assert tuple(att.o_proj.weight.shape) == (256, 4 * 128)
    assert model.num_parameters() == cfg.num_parameters()
    # the payload carries it back
    d = to_hf_config_dict(cfg)
    assert d["head_dim"] == 128
    assert get_config(_write_config(tmp_path, d)).to_dict() == cfg.to_dict()
    transformers = pytest.importorskip("transformers")
    hf_d = {k: v for k, v in d.items() if k not in ("model_type", "architectures", "torch_dtype")}
    with torch.device("meta"):
        hf = transformers.LlamaForCausalLM(transformers.LlamaConfig(**hf_d))
    assert sum(p.numel() for p in hf.parameters()) == cfg.num_parameters()


@pytest.mark.parametrize("head_dim", [None, 64, "absent"])
def test_hf_llama_equal_or_absent_head_dim_changes_nothing(tmp_path, head_dim):
    base = to_hf_config_dict(get_config("debug-llama-d64"))
    d = dict(base)
    if head_dim != "absent":
        d["head_dim"] = head_dim
    cfg = get_config(_write_config(tmp_path, d))
    assert cfg.head_dim == 64 and cfg.explicit_head_dim is None
    assert cfg.to_dict() == {**get_config("debug-llama-d64").to_dict(), "name": str(tmp_path)}
    assert "head_dim" not in to_hf_config_dict(cfg)
