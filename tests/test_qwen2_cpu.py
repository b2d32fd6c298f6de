"""Qwen2 on the CPU: ``debug-qwen2`` (head_dim 64, and a head_dim 128 variant), tied and untied, against
``transformers.Qwen2ForCausalLM`` with the same weights and random q/k/v biases (logits, loss and every gradient), the
registry's parameter counts against the meta-device model, the HF config round trip and its refusals (the Llama
``attention_bias`` / ``mlp_bias`` ones included), tied and untied HF checkpoints loaded through ``--pretrained``, the
flat layout of the biases, DDP / FSDP / TP over gloo against one process with the biases compared rank by rank, and
the single-GPU chapter flags."""
import dataclasses
import json
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from dist_utils import run_distributed
from distributed_training_guide_b200.models import build_model, get_config, to_hf_config_dict

QWEN2 = {   # id: (hidden, intermediate, layers, heads, kv heads, head_dim, vocab, tied, max positions, parameters)
    "Qwen/Qwen2.5-0.5B": (896, 4864, 24, 14, 2, 64, 151936, True, 32768, 494_032_768),
    "Qwen/Qwen2.5-1.5B": (1536, 8960, 28, 12, 2, 128, 151936, True, 131072, 1_543_714_304),
    "Qwen/Qwen2.5-3B": (2048, 11008, 36, 16, 2, 128, 151936, True, 32768, 3_085_938_688),
    "Qwen/Qwen2.5-7B": (3584, 18944, 28, 28, 4, 128, 152064, False, 131072, 7_615_616_512),
    "Qwen/Qwen2.5-14B": (5120, 13824, 48, 40, 8, 128, 152064, False, 131072, 14_770_033_664),
    "Qwen/Qwen2.5-32B": (5120, 27648, 64, 40, 8, 128, 152064, False, 131072, 32_763_876_352),
    "Qwen/Qwen2.5-72B": (8192, 29568, 80, 64, 8, 128, 152064, False, 131072, 72_706_203_648),
}
D128 = dict(num_attention_heads=2, num_key_value_heads=1)   # 2 heads x 128 over a hidden size of 256


def _hf_qwen2(cfg, transformers):
    d = {k: v for k, v in to_hf_config_dict(cfg).items() if k not in ("model_type", "architectures", "torch_dtype")}
    hf_cfg = transformers.Qwen2Config(**d)
    hf_cfg._attn_implementation = "eager"
    return transformers.Qwen2ForCausalLM(hf_cfg).float().eval()


def _biased_debug_qwen2(cfg):
    """fp32 model with random q/k/v biases; the k biases are far larger than the k projections' outputs and the q
    biases of layer 0 cancel the q projection of one token (b = -acc), so the bias add is exercised at both ends."""
    torch.manual_seed(0)
    mine = build_model(cfg, dtype=torch.float32, device="cpu")
    g = torch.Generator().manual_seed(3)
    with torch.no_grad():
        for layer in mine.model.layers:
            a = layer.self_attn
            a.q_proj.bias.copy_(torch.randn(a.q_proj.bias.shape, generator=g) * 0.5)
            a.k_proj.bias.copy_(torch.randn(a.k_proj.bias.shape, generator=g) * 20.0)
            a.v_proj.bias.copy_(torch.randn(a.v_proj.bias.shape, generator=g) * 0.5)
    return mine


@pytest.mark.parametrize("d128", [False, True])
@pytest.mark.parametrize("tied", [False, True])
def test_debug_qwen2_matches_transformers_fp32(tied, d128):
    transformers = pytest.importorskip("transformers")
    cfg = get_config("debug-qwen2", tie_word_embeddings=tied, **(D128 if d128 else {}))
    assert cfg.arch == "qwen2" and cfg.qkv_bias and cfg.head_dim == (128 if d128 else 64)
    mine = _biased_debug_qwen2(cfg)
    hf = _hf_qwen2(cfg, transformers)
    missing, unexpected = hf.load_state_dict(mine.state_dict(), strict=False)
    assert not unexpected, unexpected
    assert all("rotary" in m or "inv_freq" in m for m in missing), missing
    ids = torch.randint(0, cfg.vocab_size, (2, 96), generator=torch.Generator().manual_seed(1))
    # cancellation: the q bias of layer 0 is minus the q projection of token (0, 0)'s normed input
    with torch.no_grad():
        l0 = mine.model.layers[0]
        y = l0.input_layernorm(mine.model.embed_tokens(ids[:1, :1]))[0]
        l0.self_attn.q_proj.bias.copy_(-(y @ l0.self_attn.q_proj.weight.t()).reshape(-1))
        hf.model.layers[0].self_attn.q_proj.bias.copy_(l0.self_attn.q_proj.bias)
    out_mine = mine(input_ids=ids, labels=ids, return_logits=True)
    out_hf = hf(input_ids=ids, labels=ids)
    assert torch.allclose(out_mine.logits, out_hf.logits, atol=2e-4, rtol=1e-3), \
        (out_mine.logits - out_hf.logits).abs().max()
    assert abs(out_mine.loss.item() - out_hf.loss.item()) < 1e-4
    out_mine.loss.backward()
    out_hf.loss.backward()
    hf_params = dict(hf.named_parameters())
    names = [n for n, _ in mine.named_parameters()]
    assert sum(n.endswith("_proj.bias") for n in names) == 3 * cfg.num_hidden_layers
    for n, p in mine.named_parameters():
        want = hf_params[n].grad
        err = ((p.grad - want).norm() / want.norm()).item()
        assert err < 1e-4, (n, err)
    # the biases matter at these weights: the same weights without them give other logits
    plain = build_model(dataclasses.replace(cfg, qkv_bias=False, arch="llama"), dtype=torch.float32, device="cpu")
    plain.load_state_dict({k: v for k, v in mine.state_dict().items() if not k.endswith(".bias")})
    with torch.no_grad():
        assert (plain(input_ids=ids, return_logits=True).logits - out_hf.logits).abs().max() > 1e-1


def test_linear_bias_op_cpu_path():
    from distributed_training_guide_b200 import ops

    g = torch.Generator().manual_seed(0)
    x, w, b = torch.randn(3, 5, 16, generator=g), torch.randn(24, 16, generator=g), torch.randn(24, generator=g)
    torch.testing.assert_close(ops.linear(x, w, b), torch.nn.functional.linear(x, w, b))
    torch.testing.assert_close(ops.linear(x, w, b, owner=w, bias_owner=b), torch.nn.functional.linear(x, w, b))
    torch.testing.assert_close(ops.bias_grad(x.reshape(-1, 16)), x.reshape(-1, 16).sum(0))
    out = torch.zeros(15, 24)
    ops.gemm(x.reshape(-1, 16), w, out=out, trans_b=True, bias=b)
    torch.testing.assert_close(out, torch.nn.functional.linear(x.reshape(-1, 16), w, b))


# ---------------------------------------------------------------------------------------------------------------
# configs
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(QWEN2))
def test_registry_qwen2(name):
    h, i, l, nh, nkv, d, v, tied, maxpos, n = QWEN2[name]
    cfg = get_config(name)
    assert cfg.arch == "qwen2" and cfg.qkv_bias and not cfg.qk_norm and cfg.head_dim == d
    assert (cfg.vocab_size, cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers) == (v, h, i, l)
    assert (cfg.num_attention_heads, cfg.num_key_value_heads, cfg.tie_word_embeddings) == (nh, nkv, tied)
    assert (cfg.rope_theta, cfg.rms_norm_eps, cfg.max_position_embeddings) == (1e6, 1e-6, maxpos)
    assert cfg.num_parameters() == n
    assert build_model(cfg, dtype=torch.bfloat16, device="meta").num_parameters() == n


def test_num_parameters_against_transformers_and_existing_counts():
    transformers = pytest.importorskip("transformers")
    for name in list(QWEN2) + ["debug-qwen2"]:
        c = get_config(name)
        d = {k: v for k, v in to_hf_config_dict(c).items() if k not in ("model_type", "architectures", "torch_dtype")}
        with torch.device("meta"):
            hf = transformers.Qwen2ForCausalLM(transformers.Qwen2Config(**d))
        assert sum(p.numel() for p in hf.parameters()) == c.num_parameters(), name
    assert get_config("meta-llama/Llama-2-7b-hf").num_parameters() == 6_738_415_616
    assert get_config("Qwen/Qwen3-8B").num_parameters() == 8_190_735_360
    assert not get_config("meta-llama/Llama-2-7b-hf").qkv_bias


def _write_config(tmp_path, d):
    (tmp_path / "config.json").write_text(json.dumps(d))
    return str(tmp_path)


@pytest.mark.parametrize("name", ["Qwen/Qwen2.5-7B", "Qwen/Qwen2.5-0.5B", "debug-qwen2"])
def test_hf_config_round_trip(tmp_path, name):
    cfg = get_config(name)
    d = to_hf_config_dict(cfg)
    assert d["model_type"] == "qwen2" and d["architectures"] == ["Qwen2ForCausalLM"]
    assert (d["bos_token_id"], d["eos_token_id"], d["use_sliding_window"]) == (151643, 151643, False)
    back = get_config(_write_config(tmp_path, d))
    assert back.to_dict() == {**cfg.to_dict(), "name": str(tmp_path)}
    transformers = pytest.importorskip("transformers")
    hf = transformers.Qwen2Config(**{k: v for k, v in d.items() if k not in ("model_type", "architectures")})
    assert hf.tie_word_embeddings == cfg.tie_word_embeddings and hf.num_key_value_heads == cfg.num_key_value_heads


def test_hf_config_layouts_and_refusals(tmp_path):
    d = to_hf_config_dict(get_config("debug-qwen2"))
    v5 = {k: v for k, v in d.items() if k != "rope_theta"}
    v5["rope_parameters"] = {"rope_theta": 1e6, "rope_type": "default"}
    v5["layer_types"] = ["full_attention", "full_attention"]
    v5["sliding_window"] = 4096   # ignored while use_sliding_window is false, as in transformers
    assert get_config(_write_config(tmp_path, v5)).rope_theta == 1e6
    assert get_config(_write_config(tmp_path, {**d, "head_dim": 64})).head_dim == 64
    yarn = {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768}
    for bad, key in (({"use_sliding_window": True}, "use_sliding_window"),
                     ({"layer_types": ["full_attention", "sliding_attention"]}, "layer_types"),
                     ({"rope_scaling": yarn}, "rope_scaling"),
                     ({"rope_parameters": {**yarn, "rope_theta": 1e6}}, "rope_parameters"),
                     ({"head_dim": 128}, "head_dim")):
        with pytest.raises(ValueError, match=key):
            get_config(_write_config(tmp_path, {**d, **bad}))


def test_llama_bias_keys_are_refused(tmp_path):
    d = to_hf_config_dict(get_config("debug-llama-gqa"))
    assert d["attention_bias"] is False and d["mlp_bias"] is False
    for key in ("attention_bias", "mlp_bias"):
        with pytest.raises(ValueError, match=key):
            get_config(_write_config(tmp_path, {**d, key: True}))
    for d2 in ({**d, "attention_bias": False}, {k: v for k, v in d.items() if k not in ("attention_bias", "mlp_bias")}):
        cfg = get_config(_write_config(tmp_path, d2))
        assert cfg.arch == "llama" and not cfg.qkv_bias
    q3 = to_hf_config_dict(get_config("debug-qwen3"))
    with pytest.raises(ValueError, match="attention_bias"):
        get_config(_write_config(tmp_path, {**q3, "attention_bias": True}))


@pytest.mark.parametrize("tied", [False, True])
def test_pretrained_hf_qwen2_checkpoint_loads(tmp_path, tied):
    transformers = pytest.importorskip("transformers")
    pytest.importorskip("safetensors")
    from distributed_training_guide_b200.tools.load_hf import maybe_load_pretrained

    cfg = get_config("debug-qwen2", tie_word_embeddings=tied)
    torch.manual_seed(5)
    hf = _hf_qwen2(cfg, transformers)
    with torch.no_grad():   # biases other than 0, so that loading them is visible
        for n, p in hf.named_parameters():
            if n.endswith(".bias"):
                p.uniform_(-1.0, 1.0)
    hf.save_pretrained(str(tmp_path / "m"), safe_serialization=True)
    loaded_cfg = get_config(str(tmp_path / "m"))
    assert loaded_cfg.arch == "qwen2" and loaded_cfg.qkv_bias and loaded_cfg.tie_word_embeddings == tied
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
def test_flat_groups_hold_one_qkv_bias_view_after_the_layer_norms():
    from distributed_training_guide_b200.models.llama import init_parameter_
    from distributed_training_guide_b200.parallel.flat import build_groups

    cfg = get_config("debug-qwen2")
    model = build_model(cfg, dtype=torch.bfloat16, device="cpu")
    assert all(float(p.detach().abs().max()) == 0 for n, p in model.named_parameters() if n.endswith(".bias"))
    groups = build_groups(model, "cpu", torch.bfloat16)
    layer = groups[1]
    tail = [n.split(".", 3)[-1] for n in layer.names[-5:]]
    assert tail == ["input_layernorm.weight", "post_attention_layernorm.weight", "self_attn.q_proj.bias",
                    "self_attn.k_proj.bias", "self_attn.v_proj.bias"]
    l0 = model.model.layers[0]
    assert l0.flat_order == ("self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight",
                             "self_attn.o_proj.weight", "mlp.gate_proj.weight", "mlp.up_proj.weight",
                             "mlp.down_proj.weight", "input_layernorm.weight", "post_attention_layernorm.weight",
                             "self_attn.q_proj.bias", "self_attn.k_proj.bias", "self_attn.v_proj.bias")
    assert l0.fused == {"qkv": l0.flat_order[:3], "gate_up": l0.flat_order[4:6], "qkv_bias": l0.flat_order[9:]}
    fw = l0._fused["qkv_bias"]
    nq, nkv = cfg.num_attention_heads * cfg.head_dim, cfg.num_key_value_heads * cfg.head_dim
    assert fw.data.shape == (nq + 2 * nkv,) and fw._dtg_grad.shape == (nq + 2 * nkv,)
    a = model.model.layers[0].self_attn
    with torch.no_grad():
        for p in (a.q_proj.bias, a.k_proj.bias, a.v_proj.bias):
            init_parameter_(p, "x.weight", 1)   # random values through the parameters...
    assert torch.equal(fw.data, torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias]))   # ...seen by the view
    assert fw.data.data_ptr() == a.q_proj.bias.data_ptr()
    assert len({id(p) for g in groups for p in g.params}) == len(list(model.parameters()))
    for name in ("debug-llama-gqa", "debug-mistral", "debug-qwen3"):
        other = build_model(get_config(name), dtype=torch.bfloat16, device="meta")
        l0 = other.model.layers[0]
        assert l0.flat_order[:9] == ("self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight",
                                     "self_attn.o_proj.weight", "mlp.gate_proj.weight", "mlp.up_proj.weight",
                                     "mlp.down_proj.weight", "input_layernorm.weight",
                                     "post_attention_layernorm.weight")
        assert not any(n.endswith(".bias") for n in l0.flat_order)
        assert "qkv_bias" not in l0.fused


def test_tp_shard_spec_splits_the_biases_with_their_heads():
    from distributed_training_guide_b200.models.llama import tp_shard_spec

    p = torch.empty(128)
    assert tp_shard_spec("model.layers.0.self_attn.k_proj.bias", p, 2, 1) == dict(
        full_shape=[256], shard_dim=0, shard_index=1, shard_count=2)
    assert tp_shard_spec("model.layers.0.input_layernorm.weight", p, 2, 1) == {}


# ---------------------------------------------------------------------------------------------------------------
# DDP, FSDP and TP over gloo against one process
# ---------------------------------------------------------------------------------------------------------------
S_DIST, LR_DIST = 256, 5e-3


def _batch(vocab, step, rank, B=1):
    g = torch.Generator().manual_seed(1000 * step + rank)
    ids = torch.randint(0, vocab, (B, S_DIST), generator=g)
    return {"input_ids": ids, "labels": ids.clone()}


def _biases(model):
    return [torch.cat([l.self_attn.q_proj.bias.detach().float(), l.self_attn.k_proj.bias.detach().float(),
                       l.self_attn.v_proj.bias.detach().float()]) for l in model.model.layers]


def _train_dist(rank, world, parallelism, steps):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    kw = {"tensor_parallel": world} if parallelism == "tp" else {}
    eng = TrainEngine.create("debug-qwen2", parallelism=parallelism, batch_size=1, seq_length=S_DIST, device="cpu",
                             lr=LR_DIST, **kw)
    dp_rank = eng.strategy.dp_rank
    losses, biases = [], []
    for i in range(steps):
        losses.append(float(eng.step(_batch(eng.config.vocab_size, i, dp_rank))))
        if parallelism != "fsdp":   # FSDP holds shards; its biases are checked through the loss
            biases.append([b.numpy() for b in _biases(eng.model)])
    return losses, biases, eng.strategy.dp_size


def _single(steps, dp):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-qwen2", parallelism="single", batch_size=dp, seq_length=S_DIST, device="cpu",
                             lr=LR_DIST)
    losses, biases = [], []
    for i in range(steps):
        parts = [_batch(eng.config.vocab_size, i, r) for r in range(dp)]
        losses.append(float(eng.step({k: torch.cat([p[k] for p in parts]) for k in parts[0]})))
        biases.append([b.numpy() for b in _biases(eng.model)])
    return losses, biases


@pytest.mark.parametrize("parallelism", ["ddp", "fsdp", "tp"])
def test_distributed_qwen2_matches_single_process(parallelism):
    steps, world = 3, 2
    res = run_distributed(_train_dist, world=world, args=(parallelism, steps), timeout=600)
    dp = res[0][2]
    ref_losses, ref_biases = _single(steps, dp)
    for i in range(steps):
        mean = float(np.mean([r[0][i] for r in res]))
        assert abs(mean - ref_losses[i]) < 2e-2, (parallelism, i, [r[0][i] for r in res], ref_losses[i])
    if parallelism == "fsdp":
        return
    for i in range(steps):
        moved = 0
        for layer in range(len(ref_biases[i])):
            want = ref_biases[i][layer]
            if parallelism == "tp":   # each rank holds the q, k and v slices of its heads
                got = _tp_gather_biases(res, i, layer)
            else:
                a, b = res[0][1][i][layer], res[1][1][i][layer]
                assert np.array_equal(a, b), (parallelism, i, layer, "biases differ between ranks")
                got = a
            # AdamW moves each bias element by about lr a step whatever its gradient's size.  The k bias gradient
            # nearly cancels (a k bias shifts every score of a query by the same amount, up to RoPE), so its elements
            # step either way when the gradient is summed in another order: compare the q and v biases, as whole
            # vectors (a bias left untrained, or TP slices put back in the wrong place, are off by ~100 %)
            cfg = get_config("debug-qwen2")
            nq, nkv = cfg.num_attention_heads * cfg.head_dim, cfg.num_key_value_heads * cfg.head_dim
            qv = np.r_[0:nq, nq + nkv:nq + 2 * nkv]
            rel = np.linalg.norm(got[qv] - want[qv]) / max(np.linalg.norm(want[qv]), 1e-30)
            assert rel < 0.25, (parallelism, i, layer, rel)
            moved += int((got != 0).sum())
        assert moved > 0, "the biases never moved: the comparison is vacuous"


def _tp_gather_biases(res, i, layer):
    """Concatenate the ranks' q, k and v bias slices back into the full q | k | v bias."""
    cfg = get_config("debug-qwen2")
    t = len(res)
    nq, nkv = cfg.num_attention_heads * cfg.head_dim // t, cfg.num_key_value_heads * cfg.head_dim // t
    parts = [r[1][i][layer] for r in res]
    q = np.concatenate([p[:nq] for p in parts])
    k = np.concatenate([p[nq:nq + nkv] for p in parts])
    v = np.concatenate([p[nq + nkv:] for p in parts])
    return np.concatenate([q, k, v])


@pytest.mark.parametrize("flags", [dict(fp8=True), dict(max_grad_norm=1.0), dict(checkpoint_activations=True),
                                   dict(document_masking=True)])
def test_single_engine_flags_train_qwen2(flags):
    from distributed_training_guide_b200.engine import TrainEngine

    torch.manual_seed(0)
    eng = TrainEngine.create("debug-qwen2", parallelism="single", batch_size=1, seq_length=128, device="cpu",
                             lr=LR_DIST, **flags)
    b0 = _biases(eng.model)
    for i in range(2):
        b = _batch(eng.config.vocab_size, i, 0)
        b = {k: v[:, :128] for k, v in b.items()}
        if flags.get("document_masking"):
            b["position_ids"] = torch.cat([torch.arange(50), torch.arange(78)])[None]
        assert math.isfinite(float(eng.step(b)))
    assert any(not torch.equal(a, b) for a, b in zip(b0, _biases(eng.model)))
