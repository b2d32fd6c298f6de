"""Qwen3 on the CPU: ``debug-qwen3`` against ``transformers.Qwen3ForCausalLM`` with the same weights (logits, loss and
every gradient), the registry's parameter counts against the meta-device model, the HF config round trip and its
refusals, tied and untied HF checkpoints loaded through ``--pretrained``, the flat layout of the QK-norm gains, and
DDP / FSDP / TP over gloo against one process, with the gains compared rank by rank."""
import dataclasses
import json
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dist_utils import run_distributed
from distributed_training_guide_b200 import ops
from distributed_training_guide_b200.models import build_model, get_config, to_hf_config_dict
from distributed_training_guide_b200.ops import reference as ref

QWEN3 = {   # id: (hidden, intermediate, layers, heads, kv heads, tied, parameters)
    "Qwen/Qwen3-0.6B": (1024, 3072, 28, 16, 8, True, 596_049_920),
    "Qwen/Qwen3-1.7B": (2048, 6144, 28, 16, 8, True, 1_720_574_976),
    "Qwen/Qwen3-4B": (2560, 9728, 36, 32, 8, True, 4_022_468_096),
    "Qwen/Qwen3-8B": (4096, 12288, 36, 32, 8, False, 8_190_735_360),
    "Qwen/Qwen3-32B": (5120, 25600, 64, 64, 8, False, 32_762_123_264),
}


# ---------------------------------------------------------------------------------------------------------------
# the op's CPU path
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("per_token", [False, True])
def test_qk_norm_rope_cpu_path_composes_reference(per_token):
    g = torch.Generator().manual_seed(0)
    B, S, nh, nkv, d = 2, 12, 4, 2, 16
    qkv = torch.randn(B, S, nh + 2 * nkv, d, generator=g) * 3
    q_w, k_w = torch.randn(d, generator=g), torch.randn(d, generator=g)
    pos = torch.randint(0, 50, (B, S), generator=g) if per_token else torch.arange(S)
    cos, sin = ref.rope_tables(pos, d, 1e6)
    out = ops.qk_norm_rope_(qkv, q_w, k_w, cos, sin, nh, nkv, 1e-6)
    q = ref.rope_apply(ref.rms_norm(qkv[:, :, :nh], q_w, 1e-6), cos, sin)
    k = ref.rope_apply(ref.rms_norm(qkv[:, :, nh:nh + nkv], k_w, 1e-6), cos, sin)
    torch.testing.assert_close(out[:, :, :nh], q)
    torch.testing.assert_close(out[:, :, nh:nh + nkv], k)
    assert torch.equal(out[:, :, nh + nkv:], qkv[:, :, nh + nkv:])
    # per head: scaling a head's input does not change its output (the norm), unlike plain RoPE
    out2 = ops.qk_norm_rope_(qkv * 7.0, q_w, k_w, cos, sin, nh, nkv, 1e-6)
    torch.testing.assert_close(out2[:, :, :nh + nkv], out[:, :, :nh + nkv], rtol=1e-5, atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------
# the model against transformers
# ---------------------------------------------------------------------------------------------------------------
def _hf_qwen3(cfg, transformers):
    d = {k: v for k, v in to_hf_config_dict(cfg).items() if k not in ("model_type", "architectures", "torch_dtype")}
    hf_cfg = transformers.Qwen3Config(**d)
    hf_cfg._attn_implementation = "eager"
    return transformers.Qwen3ForCausalLM(hf_cfg).float().eval()


def _peaked_debug_qwen3(cfg):
    """fp32 model whose QK-norm gains are scaled up (with a spread) so that attention is far from uniform.  Scaling
    q_proj / k_proj would change nothing: the norm removes each head's scale."""
    torch.manual_seed(0)
    mine = build_model(cfg, dtype=torch.float32, device="cpu")
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for layer in mine.model.layers:
            for n in (layer.self_attn.q_norm, layer.self_attn.k_norm):
                n.weight.copy_(3.0 * (1 + 0.3 * torch.randn(n.weight.shape, generator=g)))
    return mine


@pytest.mark.parametrize("tied", [False, True])
def test_debug_qwen3_matches_transformers_fp32(tied):
    transformers = pytest.importorskip("transformers")
    cfg = get_config("debug-qwen3", tie_word_embeddings=tied)
    assert cfg.arch == "qwen3" and cfg.qk_norm and cfg.head_dim == 128
    assert cfg.num_attention_heads * cfg.head_dim != cfg.hidden_size
    mine = _peaked_debug_qwen3(cfg)
    hf = _hf_qwen3(cfg, transformers)
    missing, unexpected = hf.load_state_dict(mine.state_dict(), strict=False)
    assert not unexpected, unexpected
    assert all("rotary" in m or "inv_freq" in m for m in missing), missing   # names are HF's
    ids = torch.randint(0, cfg.vocab_size, (2, 96), generator=torch.Generator().manual_seed(1))
    out_mine = mine(input_ids=ids, labels=ids, return_logits=True)
    out_hf = hf(input_ids=ids, labels=ids)
    assert torch.allclose(out_mine.logits, out_hf.logits, atol=2e-4, rtol=1e-3), \
        (out_mine.logits - out_hf.logits).abs().max()
    assert abs(out_mine.loss.item() - out_hf.loss.item()) < 1e-4
    out_mine.loss.backward()
    out_hf.loss.backward()
    hf_params = dict(hf.named_parameters())
    names = [n for n, _ in mine.named_parameters()]
    assert any("q_norm" in n for n in names) and any("k_norm" in n for n in names)
    for n, p in mine.named_parameters():
        want = hf_params[n].grad
        err = ((p.grad - want).norm() / want.norm()).item()
        assert err < 1e-4, (n, err)
    # the norm matters at these weights: the same weights without it give other logits
    plain = build_model(dataclasses.replace(cfg, qk_norm=False), dtype=torch.float32, device="cpu")
    plain.load_state_dict({k: v for k, v in mine.state_dict().items() if "_norm." not in k or "layernorm" in k})
    with torch.no_grad():
        out_plain = plain(input_ids=ids, return_logits=True)
    assert (out_plain.logits - out_hf.logits).abs().max() > 1e-1


# ---------------------------------------------------------------------------------------------------------------
# configs
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(QWEN3))
def test_registry_qwen3(name):
    h, i, l, nh, nkv, tied, n = QWEN3[name]
    cfg = get_config(name)
    assert cfg.arch == "qwen3" and cfg.qk_norm and cfg.head_dim == 128
    assert (cfg.vocab_size, cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers) == (151936, h, i, l)
    assert (cfg.num_attention_heads, cfg.num_key_value_heads, cfg.tie_word_embeddings) == (nh, nkv, tied)
    assert (cfg.rope_theta, cfg.rms_norm_eps, cfg.max_position_embeddings) == (1e6, 1e-6, 40960)
    assert cfg.num_parameters() == n
    assert build_model(cfg, dtype=torch.bfloat16, device="meta").num_parameters() == n


def test_num_parameters_meta_and_transformers():
    cfg = get_config("debug-qwen3")
    assert build_model(cfg, dtype=torch.float32, device="meta").num_parameters() == cfg.num_parameters()
    transformers = pytest.importorskip("transformers")
    for name in list(QWEN3) + ["debug-qwen3"]:
        c = get_config(name)
        d = {k: v for k, v in to_hf_config_dict(c).items() if k not in ("model_type", "architectures", "torch_dtype")}
        with torch.device("meta"):
            hf = transformers.Qwen3ForCausalLM(transformers.Qwen3Config(**d))
        assert sum(p.numel() for p in hf.parameters()) == c.num_parameters(), name


def test_existing_configs_keep_head_dim_and_counts():
    """Overriding the hidden size of a Llama config still derives head_dim from it, and counts are unchanged."""
    cfg = get_config("debug-llama-gqa", hidden_size=2048, num_attention_heads=16)
    assert cfg.head_dim == 128 and not cfg.qk_norm and cfg.explicit_head_dim is None
    assert get_config("meta-llama/Llama-2-7b-hf").num_parameters() == 6_738_415_616
    assert get_config("mistralai/Mistral-7B-v0.1").num_parameters() == 7_241_732_096


def _write_config(tmp_path, d):
    (tmp_path / "config.json").write_text(json.dumps(d))
    return str(tmp_path)


@pytest.mark.parametrize("name", ["Qwen/Qwen3-8B", "Qwen/Qwen3-0.6B", "debug-qwen3"])
def test_hf_config_round_trip(tmp_path, name):
    cfg = get_config(name)
    d = to_hf_config_dict(cfg)
    assert d["model_type"] == "qwen3" and d["architectures"] == ["Qwen3ForCausalLM"] and d["head_dim"] == 128
    back = get_config(_write_config(tmp_path, d))
    assert back.to_dict() == {**cfg.to_dict(), "name": str(tmp_path)}
    transformers = pytest.importorskip("transformers")
    hf = transformers.Qwen3Config(**{k: v for k, v in d.items() if k not in ("model_type", "architectures")})
    assert hf.head_dim == 128 and hf.tie_word_embeddings == cfg.tie_word_embeddings


def test_hf_config_transformers_layout_and_refusals(tmp_path):
    d = to_hf_config_dict(get_config("debug-qwen3"))
    # transformers>=5 writes rope_parameters instead of rope_theta
    v5 = {k: v for k, v in d.items() if k != "rope_theta"}
    v5["rope_parameters"] = {"rope_theta": 1e6, "rope_type": "default"}
    v5["layer_types"] = ["full_attention", "full_attention"]
    assert get_config(_write_config(tmp_path, v5)).rope_theta == 1e6
    for bad, key in (({"use_sliding_window": True}, "use_sliding_window"),
                     ({"layer_types": ["full_attention", "sliding_attention"]}, "layer_types"),
                     ({"attention_bias": True}, "attention_bias")):
        with pytest.raises(ValueError, match=key):
            get_config(_write_config(tmp_path, {**d, **bad}))
    # without head_dim the head dimension is hidden / heads
    nohd = {k: v for k, v in d.items() if k != "head_dim"}
    assert get_config(_write_config(tmp_path, nohd)).head_dim == 256 // 4


def test_other_payloads_and_mistral_refusal_unchanged(tmp_path):
    assert "head_dim" not in to_hf_config_dict(get_config("debug-llama-gqa"))
    assert "use_sliding_window" not in to_hf_config_dict(get_config("debug-mistral"))
    d = to_hf_config_dict(get_config("debug-mistral"))
    with pytest.raises(ValueError, match="head_dim"):
        get_config(_write_config(tmp_path, {**d, "head_dim": 64}))
    assert not get_config("debug-mistral").qk_norm


@pytest.mark.parametrize("tied", [False, True])
def test_pretrained_hf_qwen3_checkpoint_loads(tmp_path, tied):
    transformers = pytest.importorskip("transformers")
    pytest.importorskip("safetensors")
    from distributed_training_guide_b200.tools.load_hf import maybe_load_pretrained

    cfg = get_config("debug-qwen3", tie_word_embeddings=tied)
    torch.manual_seed(5)
    hf = _hf_qwen3(cfg, transformers)
    with torch.no_grad():   # gains other than 1, so that loading them is visible
        for n, p in hf.named_parameters():
            if "norm" in n:
                p.uniform_(0.5, 2.0)
    hf.save_pretrained(str(tmp_path / "m"), safe_serialization=True)
    loaded_cfg = get_config(str(tmp_path / "m"))
    assert loaded_cfg.arch == "qwen3" and loaded_cfg.head_dim == 128 and loaded_cfg.tie_word_embeddings == tied
    model = build_model(loaded_cfg, dtype=torch.float32, device="cpu")
    assert maybe_load_pretrained(SimpleNamespace(model_name=str(tmp_path / "m"), pretrained="require"), model=model)
    hf_sd = hf.state_dict()
    for k, v in model.state_dict().items():
        assert torch.equal(v, hf_sd[k]), k
    ids = torch.randint(0, cfg.vocab_size, (1, 64), generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        assert torch.allclose(model(input_ids=ids, return_logits=True).logits, hf(input_ids=ids).logits,
                              atol=2e-4, rtol=1e-3)


# ---------------------------------------------------------------------------------------------------------------
# flat layout
# ---------------------------------------------------------------------------------------------------------------
def test_flat_groups_hold_the_qk_norm_gains_after_the_layer_norms():
    from distributed_training_guide_b200.parallel.flat import build_groups

    model = build_model(get_config("debug-qwen3"), dtype=torch.bfloat16, device="cpu")
    groups = build_groups(model, "cpu", torch.bfloat16)
    layer = groups[1]
    tail = [n.split(".", 3)[-1] for n in layer.names[-4:]]
    assert tail == ["input_layernorm.weight", "post_attention_layernorm.weight", "self_attn.q_norm.weight",
                    "self_attn.k_norm.weight"]
    # every gain ends with "norm.weight" and the four are one contiguous run (TP sums their gradients in one launch)
    offs = layer.offsets[-4:]
    sizes = [int(np.prod(s)) for s in layer.shapes[-4:]]
    assert all(offs[j + 1] == offs[j] + sizes[j] for j in range(3))
    assert len({id(p) for g in groups for p in g.params}) == len(list(model.parameters()))
    # a Llama layer's order is unchanged
    llama = build_model(get_config("debug-llama-gqa"), dtype=torch.bfloat16, device="meta")
    llama_order = ("self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight",
                   "self_attn.o_proj.weight", "mlp.gate_proj.weight", "mlp.up_proj.weight", "mlp.down_proj.weight",
                   "input_layernorm.weight", "post_attention_layernorm.weight")
    assert llama.model.layers[0].flat_order == llama_order
    assert llama.model.layers[0].fused == {"qkv": llama_order[:3], "gate_up": llama_order[4:6]}
    l0 = model.model.layers[0]
    assert l0.flat_order == llama_order + ("self_attn.q_norm.weight", "self_attn.k_norm.weight")
    assert l0.fused == {"qkv": llama_order[:3], "gate_up": llama_order[4:6]}


# ---------------------------------------------------------------------------------------------------------------
# DDP, FSDP and TP over gloo against one process
# ---------------------------------------------------------------------------------------------------------------
S_DIST, LR_DIST = 256, 5e-3   # an lr at which every step moves the bf16 gains by whole ulps


def _batch(vocab, step, rank, B=1):
    g = torch.Generator().manual_seed(1000 * step + rank)
    ids = torch.randint(0, vocab, (B, S_DIST), generator=g)
    return {"input_ids": ids, "labels": ids.clone()}


def _gains(model):
    return [torch.stack([l.self_attn.q_norm.weight.detach().float(), l.self_attn.k_norm.weight.detach().float()])
            for l in model.model.layers]


def _train_dist(rank, world, parallelism, steps):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    kw = {"tensor_parallel": world} if parallelism == "tp" else {}
    eng = TrainEngine.create("debug-qwen3", parallelism=parallelism, batch_size=1, seq_length=S_DIST, device="cpu",
                             lr=LR_DIST, **kw)
    dp_rank = eng.strategy.dp_rank
    losses, gains = [], []
    for i in range(steps):
        losses.append(float(eng.step(_batch(eng.config.vocab_size, i, dp_rank))))
        if parallelism != "fsdp":   # FSDP holds shards; its gains are checked through the loss
            gains.append(_gains(eng.model))
    return losses, gains, eng.strategy.dp_size


def _single(steps, dp):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-qwen3", parallelism="single", batch_size=dp, seq_length=S_DIST, device="cpu",
                             lr=LR_DIST)
    losses, gains = [], []
    for i in range(steps):
        parts = [_batch(eng.config.vocab_size, i, r) for r in range(dp)]
        losses.append(float(eng.step({k: torch.cat([p[k] for p in parts]) for k in parts[0]})))
        gains.append(_gains(eng.model))
    return losses, gains


@pytest.mark.parametrize("parallelism", ["ddp", "fsdp", "tp"])
def test_distributed_qwen3_matches_single_process(parallelism):
    steps, world = 3, 2
    res = run_distributed(_train_dist, world=world, args=(parallelism, steps), timeout=600)
    dp = res[0][2]
    ref_losses, ref_gains = _single(steps, dp)
    for i in range(steps):
        mean = float(np.mean([r[0][i] for r in res]))
        assert abs(mean - ref_losses[i]) < 2e-2, (parallelism, i, [r[0][i] for r in res], ref_losses[i])
    if parallelism == "fsdp":
        return
    for i in range(steps):
        moved = 0
        for layer in range(len(ref_gains[i])):
            a, b = res[0][1][i][layer], res[1][1][i][layer]
            assert np.array_equal(a, b), (parallelism, i, layer, "gains differ between ranks")
            want = ref_gains[i][layer].numpy()
            # bf16 tolerance: two ulps at the gains' magnitude (about 1)
            assert np.abs(a - want).max() <= 2 * 2.0 ** -7, (parallelism, i, layer, np.abs(a - want).max())
            moved += int((a != 1.0).sum())
        assert moved > 0, "the gains never moved: the comparison is vacuous"
    if parallelism == "tp":
        assert np.allclose(res[0][0], res[1][0], atol=1e-5)


@pytest.mark.parametrize("flags", [dict(fp8=True), dict(max_grad_norm=1.0), dict(checkpoint_activations=True),
                                   dict(document_masking=True)])
def test_single_engine_flags_train_qwen3(flags):
    """The flags a Llama run takes also train debug-qwen3: finite losses, and the gains get their updates."""
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-qwen3", parallelism="single", batch_size=1, seq_length=128, device="cpu",
                             lr=LR_DIST, **flags)
    g0 = _gains(eng.model)
    for i in range(2):
        b = _batch(eng.config.vocab_size, i, 0)
        b = {k: v[:, :128] for k, v in b.items()}
        if flags.get("document_masking"):
            b["position_ids"] = torch.cat([torch.arange(50), torch.arange(78)])[None]
        assert math.isfinite(float(eng.step(b)))
    assert any(not torch.equal(a, b) for a, b in zip(g0, _gains(eng.model)))
